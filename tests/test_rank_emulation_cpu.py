"""CPU: the inputs of tests/test_rank_emulation_gpu.py can tell summation orders apart.

The GPU tests compare the sharded cost totals with the oracle bit for bit.  That only means something if a different
order gives different bits on these images: folding the ranks in another order, or summing one shard as a tree instead
of in ascending server order, must change some type's total.  Checked here on P1's unlimited decisions for every plan,
with the oracle alone, together with the shapes the plans are meant to have and the order-independence of the counts.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rank_emulation as re_


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def p1():
    return re_.reference("P1")


def test_partials_are_ascending_sums(oracle, p1):
    """the restated per-server contributions, summed in ascending order, are the oracle's shard partials: the tree-sum
    check below works on the same numbers the oracle adds"""
    img = p1.img
    for G in re_.PLANS["P1"]:
        parts = re_.partials(oracle, img, p1.acc, p1.chosen, G)
        for (f, c), (_, cost) in zip(re_.plan(img.S, G), parts):
            for t in range(img.T):
                v = re_.contributions(img, p1.acc, p1.chosen, t)[f:f + c]
                assert _bits(re_.ascending_sum(v)) == _bits(cost[t]), (G, f, t)


@pytest.mark.parametrize("G", re_.PLANS["P1"])
def test_rank_order_fold_differs_from_one_rank(oracle, p1, G):
    """(a) the rank-order fold of the partials differs in bits from one rank's ascending sum, for some type"""
    img = p1.img
    parts = re_.partials(oracle, img, p1.acc, p1.chosen, G)
    _, whole = oracle.allocate_by_type(img, p1.acc, p1.chosen)
    folded = re_.fold_cost(parts)
    assert (_bits(folded) != _bits(whole)).any(), G
    # and the two are the same sum up to rounding
    assert np.allclose(folded, whole, rtol=1e-5)


@pytest.mark.parametrize("G", re_.PLANS["P1"])
def test_reverse_rank_fold_differs(oracle, p1, G):
    """(b) folding the ranks in reverse order gives other bits, for some type.  Not at G = 2: float32 addition commutes,
    so (+0 + a) + b and (+0 + b) + a are the same bits and the order of two ranks cannot show (nor matter)."""
    parts = re_.partials(oracle, p1.img, p1.acc, p1.chosen, G)
    fwd = re_.fold_cost(parts)
    rev = re_.fold_cost(parts, order=range(G - 1, -1, -1))
    assert (_bits(fwd) != _bits(rev)).any() == (G > 2), G


@pytest.mark.parametrize("G", re_.PLANS["P1"])
def test_tree_sum_inside_a_shard_differs(p1, G):
    """(c) in every shard of more than 1 024 servers (G = 5 has none: there, in every 1 000-server shard), a pairwise sum
    differs in bits from the ascending sum for some type: a k_totals that reduced cost as a tree would be seen"""
    img = p1.img
    shards = [(f, c) for f, c in re_.plan(img.S, G) if c > re_.STAGE] or re_.plan(img.S, G)
    assert (G == 5) == all(c <= re_.STAGE for _, c in shards)
    for f, c in shards:
        vs = [re_.contributions(img, p1.acc, p1.chosen, t)[f:f + c] for t in range(img.T)]
        assert any(_bits(re_.pairwise_sum(v)) != _bits(re_.ascending_sum(v)) for v in vs), (G, f, c)


def test_plans_have_the_claimed_shapes():
    """(d) P1: shards of 1 000 - 2 500 servers, a start that is not a multiple of 1 024 in every plan, one to three staging
    blocks; P2: sizes differing by one; P3: empty shards; P4: one rank holding everything"""
    S1 = re_.reference("P1").img.S
    blocks = set()
    for G in re_.PLANS["P1"]:
        p = re_.plan(S1, G)
        assert sum(c for _, c in p) == S1 and p[0][0] == 0
        assert all(1000 <= c <= 2500 for _, c in p), p
        assert any(f % re_.STAGE for f, _ in p), p
        blocks |= {-(-c // re_.STAGE) for _, c in p}
    assert blocks == {1, 2, 3}
    S2 = re_.reference("P2").img.S
    for G in re_.PLANS["P2"]:
        sizes = {c for _, c in re_.plan(S2, G)}
        assert len(sizes) == 2 and max(sizes) - min(sizes) == 1, (G, sizes)
    p3 = re_.plan(re_.reference("P3").img.S, 8)
    assert sum(1 for _, c in p3 if c == 0) >= 2 and sum(c for _, c in p3) == 5
    assert re_.plan(S2, 1) == [(0, S2)]


@pytest.mark.parametrize("name,G", re_.cases(), ids=["%s-G%d" % c for c in re_.cases()])
def test_counts_are_order_free(oracle, name, G):
    """(e) the integer counts sum to the whole image's counts in any rank order"""
    ref = re_.reference(name)
    parts = re_.partials(oracle, ref.img, ref.acc, ref.chosen, G)
    whole, _ = oracle.allocate_by_type(ref.img, ref.acc, ref.chosen)
    assert np.array_equal(re_.sum_count(parts), whole)
    assert np.array_equal(re_.sum_count(parts[::-1]), whole)
    count, cost = re_.expected_totals(oracle, ref.img, ref.acc, ref.chosen, G)
    assert np.array_equal(count, whole) and cost.dtype == np.float32


def test_limited_capacities_bind(oracle):
    """the capacities make a limited solve hand out less than the unlimited demand on every image"""
    for name in ("P1", "P2", "P3"):
        ref = re_.reference(name)
        acc, chosen = oracle.solve(ref.img, ref.pairs, ref.feasible, unlimited=False)
        count, _ = oracle.allocate_by_type(ref.img, acc, chosen)
        u_count, _ = oracle.allocate_by_type(ref.img, ref.acc, ref.chosen)
        assert (count <= ref.img.type_capacity).all() and count.sum() < u_count.sum(), name
