"""CPU: the chunk planner of the materialised-p[] path (csrc/wva_scratch_plan.h) compiles without CUDA and lays out
each chunk's scratch rows as the pair and queue calls need them: prefix sums in list order, one chunk when the list
fits, a split where the next item would overflow, and an empty chunk when one item alone does not fit.  Its equal-row
form, for the sweep's and the blocking plane's lists, covers the list once in order under the same capacity rule:
the larger of half the free memory and the scratch already held."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "inferno-autoscaler_b200", "csrc")

DRIVER = r"""
#include "wva_scratch_plan.h"
#include <cstdio>
#include <vector>
// stdin: capacity, n, n lengths.  stdout: one line per chunk, "end doubles offs...", as the runner walks the list
int main() {
    long long cap = 0;
    size_t n = 0;
    if (std::scanf("%lld %zu", &cap, &n) != 2) return 2;
    std::vector<long long> len(n);
    for (long long& x : len)
        if (std::scanf("%lld", &x) != 1) return 2;
    std::vector<long long> offs;
    for (size_t i0 = 0; i0 < n;) {
        const wva::ScratchChunk c = wva::scratch_chunk(len, i0, cap, offs);
        std::printf("%zu %lld", c.end, c.doubles);
        for (long long o : offs) std::printf(" %lld", o);
        std::printf("\n");
        if (c.end == i0) break;
        i0 = c.end;
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def planner():
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "plan.cpp"), os.path.join(tmp, "plan")
        with open(src, "w") as f:
            f.write(DRIVER)
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + CSRC,
                               "-o", exe, src])

        def run(lengths, cap):
            inp = "%d %d\n%s\n" % (cap, len(lengths), " ".join(str(int(x)) for x in lengths))
            out = subprocess.run([exe], input=inp, capture_output=True, text=True, check=True).stdout
            chunks = []
            for line in out.splitlines():
                v = [int(x) for x in line.split()]
                chunks.append((v[0], v[1], v[2:]))
            return chunks
        yield run


def parent_offsets(lengths):
    """The whole-list layout the pair and queue calls computed inline: offs[i] = total so far, then total += len[i]."""
    offs, total = [], 0
    for n in lengths:
        offs.append(total)
        total += n
    return offs, total


def pair_lengths(rng, n):
    return [11 * int(N) + 1 for N in rng.integers(1, 8193, n)]


def test_offsets_are_prefix_sums_in_list_order(planner):
    rng = np.random.default_rng(3)
    lengths = [int(x) for x in rng.integers(1, 10 ** 6, 500)]
    (end, doubles, offs), = planner(lengths, 1 << 60)
    assert end == len(lengths) and doubles == sum(lengths)
    assert offs == [0] + list(np.cumsum(lengths)[:-1])


@pytest.mark.parametrize("slack", [0, 1, 10 ** 9])
def test_list_under_capacity_is_one_chunk_with_parent_offsets(planner, slack):
    rng = np.random.default_rng(5)
    for lengths in (pair_lengths(rng, 1), pair_lengths(rng, 37), [2 * 64 + 1, 2 * 1 + 1, 8192 + 8192 * 4 + 1]):
        offs, total = parent_offsets(lengths)
        assert planner(lengths, total + slack) == [(len(lengths), total, offs)]


def test_capacity_splits_where_the_next_item_would_overflow(planner):
    rng = np.random.default_rng(11)
    lengths = pair_lengths(rng, 400)
    cap = 3 * max(lengths) + 17
    chunks = planner(lengths, cap)
    assert len(chunks) > 1
    start = 0
    for end, doubles, offs in chunks:
        assert end > start
        part = lengths[start:end]
        assert (offs, doubles) == parent_offsets(part)
        assert doubles <= cap
        if end < len(lengths):
            assert doubles + lengths[end] > cap
        start = end
    assert start == len(lengths)
    # at exactly the capacity an item still fits
    assert planner([4, 6, 5], 10) == [(2, 10, [0, 4]), (3, 5, [0])]


def test_item_larger_than_capacity_gives_an_empty_chunk(planner):
    assert planner([11 * 4096 + 1], 11 * 4096) == [(0, 0, [])]
    # in the middle of a list: the items before it run, then the chunk at it is empty
    assert planner([5, 5, 100, 5], 12) == [(2, 10, [0, 5]), (2, 0, [])]


def test_empty_list_gives_no_chunks(planner):
    assert planner([], 1 << 30) == []
    assert planner([], 0) == []


ROWS_DRIVER = r"""
#include "wva_scratch_plan.h"
#include <cstdio>
// stdin: free bytes, held bytes, n, row doubles.  stdout: one line per chunk, "end doubles", as the runner walks the list
int main() {
    size_t freeB = 0, heldB = 0, n = 0;
    long long row = 0;
    if (std::scanf("%zu %zu %zu %lld", &freeB, &heldB, &n, &row) != 4) return 2;
    const long long cap = wva::scratch_cap_doubles(freeB, heldB);
    for (size_t i0 = 0; i0 < n;) {
        const wva::ScratchChunk c = wva::scratch_chunk_rows(n, i0, row, cap);
        std::printf("%zu %lld\n", c.end, c.doubles);
        if (c.end == i0) break;
        i0 = c.end;
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def rows_planner():
    """The equal-row planner of the sweep's and the blocking plane's literal lists, under the scratch rule."""
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "rows.cpp"), os.path.join(tmp, "rows")
        with open(src, "w") as f:
            f.write(ROWS_DRIVER)
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + CSRC,
                               "-o", exe, src])

        def run(n, row, free, held):
            out = subprocess.run([exe], input="%d %d %d %d\n" % (free, held, n, row), capture_output=True, text=True,
                                 check=True).stdout
            return [tuple(int(x) for x in line.split()) for line in out.splitlines()]
        yield run


def check_rows_cover(chunks, n, row, cap_doubles):
    start = 0
    for end, doubles in chunks:
        assert start < end <= n
        assert doubles == (end - start) * row <= cap_doubles
        if end < n:
            assert doubles + row > cap_doubles
        start = end
    assert start == n


@pytest.mark.parametrize("n", [1, 7, 1000, 123457])
def test_equal_rows_cover_the_list_once_in_order(rows_planner, n):
    row = 11 * 8192 + 1
    for free in (row * 8 * 2 * 3 + 5, row * 8 * 2 * 1000, 80 << 30):
        chunks = rows_planner(n, row, free, 0)
        check_rows_cover(chunks, n, row, (free // 2) // 8)
        # the parent's rule when nothing is held: (free / 2) / (8 * row) items per chunk
        assert chunks[0][0] == min(n, (free // 2) // (8 * row))


def test_equal_rows_held_scratch_above_half_the_free_memory_gives_the_larger_chunk(rows_planner):
    row, n = 11 * 512 + 1, 10000
    free = 2 * 8 * row * 10                    # half the free memory holds 10 rows
    held = 8 * row * 300                       # the buffer already held holds 300
    chunks = rows_planner(n, row, free, held)
    assert chunks[0] == (300, 300 * row)
    check_rows_cover(chunks, n, row, held // 8)
    assert len(chunks) == (n + 299) // 300
    # held memory below half the free memory changes nothing
    assert rows_planner(n, row, free, 8 * row * 3) == rows_planner(n, row, free, 0)
    # held memory alone is enough when the free memory is gone
    assert rows_planner(5, row, 0, 8 * row * 5) == [(5, 5 * row)]


def test_equal_row_larger_than_the_capacity_gives_an_empty_chunk(rows_planner):
    row = 11 * 8192 + 1
    assert rows_planner(4, row, 2 * 8 * row - 2, 8 * row - 8) == [(0, 0)]
    assert rows_planner(4, row, 0, 0) == [(0, 0)]
    assert rows_planner(4, row, 2 * 8 * row, 0) == [(1, row), (2, row), (3, row), (4, row)]
