"""GPU: the sharded Analyze -> Optimize exchange on one device, several contexts standing in for the ranks.

Each context is sharded like one rank (`distributed.shard_range`) and runs what a rank runs; the collective is replaced by
device-to-device copies on the receiving context's stream, so everything else of the multi-GPU flow -- shard-local pair
sizing and sweep, k_totals at s0 > 0 and across its staging blocks, wva_pairs_device / wva_pairs_commit with rows another
shard produced, wva_type_totals_merge -- is checked bit for bit against the oracle, on the images and plans of
tests/rank_emulation.py:

  * unlimited mode: each rank's pair rows, sweep winners and decisions against the oracle over the whole image, its local
    totals against its shard's oracle partial, and after the exchange every rank's totals against the rank-order fold
    (the same bytes on every rank);
  * limited mode: every rank receives the other shards' rows, commits them and runs the limited solve; decisions and
    scaled records are the same on every rank and equal oracle.solve on the full arrays, totals as above;
  * a negative control (one rank's rows withheld) and the state errors of the exchange calls.
"""
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rank_emulation as re_

pytestmark = pytest.mark.gpu

abi = re_.abi
NONE, PEXH, PRR, RR = abi.POLICY_NONE, abi.POLICY_PRIORITY_EXHAUSTIVE, abi.POLICY_PRIORITY_ROUND_ROBIN, abi.POLICY_ROUND_ROBIN
PATH = {2: 3, 1: 2, 0: 1}                       # wva_solve_set_ranked setting -> path at A <= 32: scan, ranked queue, heap

# (policy, delayed best effort, solver setting) of the limited solves of each plan
_FULL = [(p, d, 2) for p in (NONE, PEXH, PRR, RR) for d in (False, True)] + \
        [(PEXH, False, 1), (RR, True, 1), (PEXH, False, 0), (RR, True, 0)]
LIMITED = {
    ("P1", 3): _FULL,
    ("P1", 5): [(PEXH, False, 2)],
    ("P2", 2): [(NONE, False, 2), (PRR, True, 2), (PEXH, False, 1)],
    ("P2", 5): [(RR, True, 2), (RR, True, 0), (PEXH, False, 2)],
    ("P3", 8): [(NONE, False, 2), (PRR, False, 2), (PEXH, True, 0)],
    ("P4", 1): [(PEXH, False, 2), (RR, True, 1)],
}
CASES = re_.cases()
IDS = ["%s-G%d" % c for c in CASES]


@pytest.fixture(scope="module")
def ranks(wva):
    """eight contexts on device 0 (a G-rank plan uses the first G), all closed at the end"""
    from inferno_autoscaler_b200 import binding
    ctxs = []
    try:
        for _ in range(max(G for _, G in CASES)):
            ctxs.append(binding.Context(0))
        yield ctxs
    finally:
        for c in ctxs:
            c.close()


@functools.lru_cache(maxsize=None)
def _winners(name):
    import oracle
    ref = re_.reference(name)
    r_max, b_max = re_.SWEEP[name]
    return oracle.analyze_grid(ref.img, r_max, b_max, want_cube=False, threads=oracle.hardware_threads())[0]


def _torch():
    import torch
    return torch


def _dev(ctx):
    return _torch().device("cuda", ctx.device)


def _view(ctx, ptr, n, dt):
    from inferno_autoscaler_b200 import distributed
    return distributed.device_tensor(ptr, n, dt, _dev(ctx))


def _on_stream(ctx):
    torch = _torch()
    return torch.cuda.stream(torch.cuda.ExternalStream(ctx.stream(), device=_dev(ctx)))


def _bytes(count, cost):
    return np.asarray(count, dtype=np.int64).tobytes() + np.asarray(cost, dtype=np.float32).tobytes()


def setup_ranks(ctxs, img, G):
    shards = re_.plan(img.S, G)
    for c, (f, n) in zip(ctxs[:G], shards):
        c.upload(img)
        c.set_shard(f, n)
    return ctxs[:G], shards


def gather_rows(ctxs, shards, img, withhold=None):
    """every context receives the other ranks' candidate rows (the nine record fields and `feasible`) from their contexts'
    device arrays, copied on its own stream; rank `withhold`'s rows are replaced by feasible = 0 on every context, its own
    included.  Then wva_pairs_commit on each."""
    A, n = img.A, img.S * img.A
    views = [c.pairs_device() for c in ctxs]
    for r, c in enumerate(ctxs):
        with _on_stream(c):
            for name, (ptr, dt) in views[r].items():
                dst = _view(c, ptr, n, dt)
                for q, (f, k) in enumerate(shards):
                    lo, hi = f * A, (f + k) * A
                    if k == 0:
                        continue
                    if q == withhold:
                        if name == "feasible":
                            dst[lo:hi].zero_()
                    elif q != r:
                        dst[lo:hi].copy_(_view(ctxs[q], views[q][name][0], n, dt)[lo:hi])
    for c in ctxs:
        c.pairs_commit()                       # waits for the device: every copy above has landed


def exchange_totals(ctxs, T):
    """the totals exchange of a G-rank run: each context concatenates the G blocks of wva_type_totals_device in rank order
    (on its own stream), then wva_type_totals_merge; returns each context's totals read back through the device view"""
    torch = _torch()
    G, nbytes = len(ctxs), 12 * T
    blocks = []
    for c in ctxs:
        ptr, nb = c.type_totals_device()
        assert nb == nbytes
        blocks.append(_view(c, ptr, nbytes, np.uint8))
    bufs = []
    for c in ctxs:
        with _on_stream(c):
            buf = torch.empty(G * nbytes, dtype=torch.uint8, device=_dev(c))
            for r, b in enumerate(blocks):
                buf[r * nbytes:(r + 1) * nbytes].copy_(b)
        bufs.append(buf)
    torch.cuda.synchronize()                   # every block is copied before a merge overwrites its source
    for c, buf in zip(ctxs, bufs):
        c.type_totals_merge(buf.data_ptr(), G)
    torch.cuda.synchronize()
    return [read_totals(c, T) for c in ctxs]


def read_totals(ctx, T):
    """(count, cost) of the context's totals buffer, read through its device view"""
    ptr, _ = ctx.type_totals_device()
    return _view(ctx, ptr, T, np.int64).cpu().numpy(), _view(ctx, ptr + 8 * T, T, np.float32).cpu().numpy()


def check_totals(oracle, img, acc, chosen, shards, local, merged):
    """local totals = each shard's oracle partial; merged totals = the rank-order fold, the same bytes on every rank"""
    G = len(shards)
    parts = re_.partials(oracle, img, acc, chosen, G)
    for r, ((count, cost), (w_count, w_cost)) in enumerate(zip(local, parts)):
        assert _bytes(count, cost) == _bytes(w_count, w_cost), ("local", r, shards[r])
    w_count, w_cost = re_.sum_count(parts), re_.fold_cost(parts)
    whole, _ = oracle.allocate_by_type(img, acc, chosen)
    assert np.array_equal(w_count, whole)
    for r, (count, cost) in enumerate(merged):
        assert _bytes(count, cost) == _bytes(w_count, w_cost), ("merged", r, count, cost, w_count, w_cost)


@pytest.mark.parametrize("name,G", CASES, ids=IDS)
def test_unlimited_ranks(oracle, ranks, name, G):
    ref = re_.reference(name)
    img, A = ref.img, ref.img.A
    ctxs, shards = setup_ranks(ranks, img, G)
    r_max, b_max = re_.SWEEP[name]
    o_best = _winners(name)
    local = []
    for r, (c, (f, n)) in enumerate(zip(ctxs, shards)):
        c.analyze(r_max, b_max)                # pair sizing and the sweep, overlapped
        pairs, feas = c.pairs_fetch()
        m = slice(f * A, (f + n) * A)
        assert np.array_equal(feas[m], ref.feasible[m]), (r, f, n)
        ok, field = pairs.equal_bits(ref.pairs, mask=m)
        assert ok, (r, f, n, field)
        assert c.grid_fetch().tobytes() == o_best[f:f + n].tobytes(), (r, f, n)
        acc, chosen = c.solve(unlimited=True)
        assert np.array_equal(acc[f:f + n], ref.acc[f:f + n]), (r, f, n)
        ok, field = chosen.equal_bits(ref.chosen, mask=slice(f, f + n))
        assert ok, (r, f, n, field)
        local.append(c.allocate_by_type())
    merged = exchange_totals(ctxs, img.T)
    check_totals(oracle, img, ref.acc, ref.chosen, shards, local, merged)


def limited_round(ctxs, shards, img, policy, delayed, ranked, withhold=None):
    """one limited solve on every rank: shard-local pair sizing, the gather, the solve, local totals, the exchange"""
    for c in ctxs:
        c.analyze_pairs(download=False)        # a limited solve scales the records in place: size them afresh
    gather_rows(ctxs, shards, img, withhold=withhold)
    out, local = [], []
    for c in ctxs:
        c.solve_set_ranked(ranked)
        try:
            acc, chosen = c.solve(unlimited=False, delayed_best_effort=delayed, policy=policy)
            path = c.solve_greedy_path()
        finally:
            c.solve_set_ranked(2)
        out.append((acc, chosen, path))
        local.append(c.allocate_by_type())
    return out, local, exchange_totals(ctxs, img.T)


@pytest.mark.parametrize("name,G", list(LIMITED), ids=["%s-G%d" % c for c in LIMITED])
def test_limited_ranks(oracle, ranks, name, G):
    ref = re_.reference(name)
    img = ref.img
    ctxs, shards = setup_ranks(ranks, img, G)
    for policy, delayed, ranked in LIMITED[(name, G)]:
        what = (policy, delayed, ranked)
        w_acc, w_chosen = oracle.solve(img, ref.pairs, ref.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
        out, local, merged = limited_round(ctxs, shards, img, policy, delayed, ranked)
        for r, (acc, chosen, path) in enumerate(out):
            assert path == PATH[ranked], what + (r,)
            assert np.array_equal(acc, w_acc), what + (r, np.nonzero(acc != w_acc)[0][:8])
            ok, field = chosen.equal_bits(w_chosen)
            assert ok, what + (r, field)
        check_totals(oracle, img, w_acc, w_chosen, shards, local, merged)


@pytest.mark.parametrize("name,G,withheld", [("P2", 5, 2), ("P1", 3, 1)], ids=["P2-G5-rank2", "P1-G3-rank1"])
def test_withheld_rows(oracle, ranks, name, G, withheld):
    """negative control: one rank's rows are not gathered (feasible = 0 over them instead).  The decisions follow the
    oracle on those inputs and differ from the full gather's, so the gather is what the limited tests see."""
    ref = re_.reference(name)
    img = ref.img
    ctxs, shards = setup_ranks(ranks, img, G)
    f, n = shards[withheld]
    assert n > 0
    feas = ref.feasible.copy()
    feas[f * img.A:(f + n) * img.A] = 0
    policy = abi.POLICY_PRIORITY_EXHAUSTIVE
    w_acc, w_chosen = oracle.solve(img, ref.pairs, feas, unlimited=False, policy=policy)
    full_acc, full_chosen = oracle.solve(img, ref.pairs, ref.feasible, unlimited=False, policy=policy)
    assert not (np.array_equal(w_acc, full_acc) and w_chosen.equal_bits(full_chosen)[0])
    out, local, merged = limited_round(ctxs, shards, img, policy, False, 2, withhold=withheld)
    for r, (acc, chosen, _) in enumerate(out):
        assert np.array_equal(acc, w_acc), r
        assert chosen.equal_bits(w_chosen)[0], r
        assert not (np.array_equal(acc, full_acc) and chosen.equal_bits(full_chosen)[0]), r
    check_totals(oracle, img, w_acc, w_chosen, shards, local, merged)


def test_exchange_state_errors(wva, oracle, ranks):
    """the exchange calls refuse to run out of order, and each context goes on working after the refusal"""
    from inferno_autoscaler_b200 import binding
    ref = re_.reference("P2")
    img, G = ref.img, 2
    policy = abi.POLICY_PRIORITY_ROUND_ROBIN
    w_acc, w_chosen = oracle.solve(img, ref.pairs, ref.feasible, unlimited=False, policy=policy)

    def refused(code, call, *args):
        with pytest.raises(binding.WvaError) as e:
            call(*args)
        assert e.value.code == code, (call, e.value)

    def limited_ok(ctxs, shards):
        out, local, merged = limited_round(ctxs, shards, img, policy, False, 2)
        for acc, chosen, _ in out:
            assert np.array_equal(acc, w_acc) and chosen.equal_bits(w_chosen)[0]
        check_totals(oracle, img, w_acc, w_chosen, shards, local, merged)

    # wva_type_totals_merge before any wva_allocate_by_type on the context, and with n_ranks = 0
    fresh = binding.Context(0)
    try:
        fresh.upload(img)
        fresh.analyze_pairs(download=False)
        fresh.solve(unlimited=True)
        buf = _torch().zeros(12 * img.T * G, dtype=_torch().uint8, device=_dev(fresh))
        refused(wva.abi.ESTATE, fresh.type_totals_merge, buf.data_ptr(), G)
        fresh.allocate_by_type()
        refused(wva.abi.EINVAL, fresh.type_totals_merge, buf.data_ptr(), 0)
        count, cost = fresh.allocate_by_type()
        w = oracle.allocate_by_type(img, ref.acc, ref.chosen)
        assert _bytes(count, cost) == _bytes(*w)
    finally:
        fresh.close()

    ctxs, shards = setup_ranks(ranks, img, G)
    # wva_pairs_commit before wva_analyze_pairs (set_shard has dropped the rows)
    for c in ctxs:
        refused(wva.abi.ESTATE, c.pairs_commit)
    # a limited solve on a partial shard without the gather and the commit
    for c in ctxs:
        c.analyze_pairs(download=False)
        refused(wva.abi.ESTATE, c.solve, False, False, policy)
    limited_ok(ctxs, shards)
    # the records a limited solve has scaled in place cannot be fetched
    for c in ctxs:
        refused(wva.abi.ESTATE, c.pairs_fetch)
    # n_ranks = 0 on contexts that hold merged totals: refused, the totals stay as they were
    before = [read_totals(c, img.T) for c in ctxs]
    for c in ctxs:
        refused(wva.abi.EINVAL, c.type_totals_merge, c.type_totals_device()[0], 0)
    _torch().cuda.synchronize()
    assert [_bytes(*read_totals(c, img.T)) for c in ctxs] == [_bytes(*x) for x in before]
    limited_ok(ctxs, shards)
