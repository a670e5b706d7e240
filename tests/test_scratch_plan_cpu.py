"""CPU: the chunk planner of the materialised-p[] path (csrc/wva_scratch_plan.h) compiles without CUDA and lays out
each chunk's scratch rows as the pair and queue calls need them: prefix sums in list order, one chunk when the list
fits, a split where the next item would overflow, and an empty chunk when one item alone does not fit."""
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
