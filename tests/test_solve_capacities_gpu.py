"""GPU: the limited-capacity solve over a list of capacity vectors (wva_solve_capacities) against the oracle and against
the library's own one-vector loop (wva_system_set_capacity -> wva_analyze_pairs -> wva_solve -> wva_solution_fetch ->
wva_allocate_by_type), on a generated image, on the injected tables of tests/solve_inject_tables.py on every solver
path, across chunk boundaries, and around the state the call must leave alone.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solve_capacities_cases as sc
import solve_inject_tables as st
from test_solve_inject_gpu import _inject, expected_path

pytestmark = pytest.mark.gpu
abi = st.abi


def _generated(wva, ctx, S=1000, A=8, T=3, seed=3):
    img = wva.synth.make_system(S, A, seed=seed, n_types=T)
    ctx.upload(img)
    ctx.analyze_pairs(download=False)
    pairs, feasible = ctx.pairs_fetch()
    return img, pairs, feasible


def _loop(ctx, caps, delayed, policy):
    """the public loop, one vector at a time"""
    img = ctx.image
    n, S, T = len(caps), img.S, img.T
    acc = np.zeros((n, S), dtype=np.int32)
    recs = np.zeros((n, S), dtype=abi.PAIR_REC_DTYPE)
    count = np.zeros((n, T), dtype=np.int64)
    cost = np.zeros((n, T), dtype=np.float32)
    saved = img.type_capacity.copy()
    for j, cap in enumerate(caps):
        ctx.set_capacity(cap)
        ctx.analyze_pairs(download=False)
        ctx.solve(unlimited=False, delayed_best_effort=delayed, policy=policy, download=False)
        a, ch = ctx.solution_fetch()
        acc[j], recs[j] = a, sc.to_recs(a, ch)
        count[j], cost[j] = ctx.allocate_by_type()
    ctx.set_capacity(saved)
    ctx.analyze_pairs(download=False)
    return acc, recs, count, cost


def _bytes_equal(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


@pytest.mark.parametrize("delayed", [False, True])
@pytest.mark.parametrize("policy", st.POLICIES)
def test_generated_image_against_oracle(wva, oracle, ctx, policy, delayed):
    """config-3 shape (1 000 x 8, 3 types), 64 vectors: zero, fractions 0.05 ... 1.2 of the demand, the first candidates'
    demand and +-1, negative, 2^62, each type starved"""
    img, pairs, feasible = _generated(wva, ctx)
    caps = sc.ladder(img, pairs, feasible, oracle, round_robin=policy in st.ROUND_ROBIN)
    got = ctx.solve_capacities(caps, delayed_best_effort=delayed, policy=policy)
    c = ctx.solve_capacities_counters()
    assert c["path"] == 3 and c["chunks"] == 1 and c["events"] > 0 and c["max_cycles"] > 0
    sc.check(got, sc.expected(oracle, img, pairs, feasible, caps, delayed, policy), (policy, delayed))
    acc = got[0]
    placed = (acc >= 0).sum(axis=1)
    assert placed.min() == 0 and placed.max() > placed.min()                  # nobody placed at zero, more further up
    assert len({a.tobytes() for a in acc}) > 20                               # placements change along the ladder


@pytest.mark.parametrize("policy", [abi.POLICY_NONE, abi.POLICY_PRIORITY_EXHAUSTIVE, abi.POLICY_PRIORITY_ROUND_ROBIN])
def test_equals_the_library_loop(wva, oracle, ctx, policy):
    """byte-equal to the public loop on a subset of the ladder; the uploaded capacity gives a plain wva_solve's result"""
    img, pairs, feasible = _generated(wva, ctx, S=300, A=6, T=3, seed=11)
    caps = sc.ladder(img, pairs, feasible, oracle, round_robin=policy in st.ROUND_ROBIN)[::8]
    caps = np.concatenate([caps, img.type_capacity[None, :].astype(np.int64)])
    for delayed in (False, True):
        got = ctx.solve_capacities(caps, delayed_best_effort=delayed, policy=policy)
        assert _bytes_equal(got, _loop(ctx, caps, delayed, policy)), (policy, delayed)
        a, ch = ctx.solve(unlimited=False, delayed_best_effort=delayed, policy=policy)
        assert got[0][-1].tobytes() == a.tobytes() and got[1][-1].tobytes() == sc.to_recs(a, ch).tobytes()
        ctx.analyze_pairs(download=False)


INJECTED = ["accels-A8", "accels-A16", "accels-A32", "accels-A33", "accels-A64", "types-A32-T256-high", "capacities-400",
            "wrap-500", "wrap-huge-500", "values-600", "values-A32", "dropped-700"]


def _table_caps(t, n):
    """n vectors around the table's own: the first candidates' demand scaled, one unit more or less, nothing, negative"""
    dem, one = st.first_counts(t)
    dem, one = np.array(dem, dtype=np.int64), np.array(one, dtype=np.int64)
    rng = np.random.default_rng(len(t.kind) + t.img.S)
    rows = [t.img.type_capacity.astype(np.int64), np.zeros(t.img.T, dtype=np.int64), np.full(t.img.T, -5, dtype=np.int64), one, one - 1]
    while len(rows) < n:
        rows.append((rng.choice([0.0, 0.1, 0.3, 0.5, 0.8, 1.0, 1.5], t.img.T) * dem).astype(np.int64))
    caps = np.array(rows[:n], dtype=np.int64)
    return caps if t.huge else np.minimum(caps, st.ROUND_ROBIN_ROUNDS)


@pytest.mark.parametrize("name", INJECTED)
def test_injected_tables_every_path(oracle, ctx, name):
    case = next(c for c in st.CASES if c[0] == name)
    t = st.case_table(case)
    caps = _table_caps(t, 4 + (case[2] % 13))
    ctx.upload(t.img)
    _inject(ctx, t)
    seen = set()
    try:
        for policy in t.policies():
            for delayed in (False, True):
                want = sc.expected(oracle, t.img, t.pairs, t.feasible, caps, delayed, policy)
                for ranked in (2, 1, 0):
                    ctx.solve_set_ranked(ranked)
                    got = ctx.solve_capacities(caps, delayed_best_effort=delayed, policy=policy)
                    path = ctx.solve_capacities_counters()["path"]
                    assert path == expected_path(t, ranked), (name, ranked)
                    sc.check(got, want, (name, policy, delayed, ranked))
                    seen.add(path)
    finally:
        ctx.solve_set_ranked(2)
    assert seen == ({3, 2, 1} if t.img.A <= 32 else {2, 1})


def test_more_than_256_types_is_rejected(wva, oracle, ctx):
    from inferno_autoscaler_b200 import binding
    rng = np.random.Generator(np.random.PCG64(42))
    t = st.make_table(rng, 30, 8, 257, "types", type_map="scatter")
    ctx.upload(t.img)
    _inject(ctx, t)
    before = _state(ctx, totals=False)
    with pytest.raises(binding.WvaError) as e:
        ctx.solve_capacities(np.zeros((2, 257), dtype=np.int64))
    assert e.value.code == wva.abi.EINVAL
    assert _state(ctx, totals=False) == before and before[0][0] != "error"
    t2 = st.make_table(rng, 30, 8, 256, "types", type_map="scatter")
    ctx.upload(t2.img)
    _inject(ctx, t2)
    caps = _table_caps(t2, 6)
    got = ctx.solve_capacities(caps, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
    sc.check(got, sc.expected(oracle, t2.img, t2.pairs, t2.feasible, caps, False, abi.POLICY_PRIORITY_EXHAUSTIVE), "T=256")


def _device_bytes(ptr, n):
    import torch
    from inferno_autoscaler_b200 import distributed
    torch.cuda.synchronize()
    return distributed.device_tensor(ptr, n, np.dtype(np.uint8), torch.device("cuda", 0)).cpu().numpy().tobytes()


def _state(ctx, totals=True):
    """what other calls read: pair records and feasible flags, the last decisions, the totals buffer (when the image's T
    is the one wva_allocate_by_type last ran with), the sweep winners (a part that its own call refuses is recorded as
    that call's error code)"""
    from inferno_autoscaler_b200 import binding

    def get(fn):
        try:
            return fn()
        except binding.WvaError as e:
            return ("error", e.code)

    def pairs():
        p, fe = ctx.pairs_fetch()
        return b"".join(getattr(p, n).tobytes() for n, _ in abi.ALLOC_FIELDS) + fe.tobytes()

    def decisions():
        acc, chosen = ctx.solution_fetch()
        return acc.tobytes() + b"".join(getattr(chosen, n).tobytes() for n, _ in abi.ALLOC_FIELDS)

    def totals_bytes():
        tp, tn = ctx.type_totals_device()
        return _device_bytes(tp, tn)

    return get(pairs), get(decisions), get(totals_bytes) if totals else None, get(lambda: ctx.grid_fetch().tobytes())


def _capacity_is(ctx, oracle, img, pairs, feasible):
    """the image's capacity, read through limited solves: every policy and schedule equals the oracle at img.type_capacity
    (the ladder's vectors around it give other decisions); re-sizes the pairs after each solve"""
    for policy in st.POLICIES:
        for delayed in (False, True):
            acc, ch = ctx.solve(unlimited=False, delayed_best_effort=delayed, policy=policy)
            w_acc, w_ch = oracle.solve(img, pairs, feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
            assert np.array_equal(acc, w_acc) and ch.equal_bits(w_ch)[0], (policy, delayed)
            ctx.analyze_pairs(download=False)


def test_residency_and_errors(wva, oracle, ctx):
    """pair records, feasible flags, the last decisions, totals, sweep winners and the image's capacity stay as they were,
    around the call and around each error; a limited wva_solve right after works; after it the call needs new records"""
    from inferno_autoscaler_b200 import binding
    L = binding.lib()
    img = wva.synth.make_system(120, 4, seed=21, n_types=2)
    ctx.upload(img)
    ctx.analyze(8, 16)
    ctx.solve(unlimited=True)
    ctx.allocate_by_type()
    pairs, feasible = ctx.pairs_fetch()
    caps = sc.ladder(img, pairs, feasible, oracle, n=16)
    before = _state(ctx)
    ctx.solve_capacities(caps, policy=abi.POLICY_ROUND_ROBIN)
    assert _state(ctx) == before
    cap = np.ascontiguousarray(caps)
    for spec, n_c, ptr in ((abi.OptimizerSpec(1, 0, 0), 4, abi.ptr(cap, C.c_int64)), (abi.OptimizerSpec(0, 0, 0), 0, abi.ptr(cap, C.c_int64)),
                           (abi.OptimizerSpec(0, 0, 0), abi.SOLVE_MAX_CAPACITIES + 1, abi.ptr(cap, C.c_int64)),
                           (abi.OptimizerSpec(0, 0, 0), 4, None)):
        assert L.wva_solve_capacities(ctx._h, C.byref(spec), n_c, ptr, None, None, None, None) == abi.EINVAL
        assert _state(ctx) == before
    assert L.wva_solve_capacities(ctx._h, None, 4, abi.ptr(cap, C.c_int64), None, None, None, None) == abi.EINVAL
    assert _state(ctx) == before
    # a limited solve right after the call works, without re-analysis, and equals the oracle at the uploaded capacity
    acc, ch = ctx.solve(unlimited=False, policy=abi.POLICY_ROUND_ROBIN)
    w_acc, w_ch = oracle.solve(img, pairs, feasible, unlimited=False, policy=abi.POLICY_ROUND_ROBIN)
    assert np.array_equal(acc, w_acc) and ch.equal_bits(w_ch)[0]
    ctx.allocate_by_type()
    # the records are scaled now: refused with WVA_ESTATE, and nothing changes around the refusal
    before = _state(ctx)
    assert before[0] == ("error", abi.ESTATE)
    with pytest.raises(binding.WvaError) as e:
        ctx.solve_capacities(caps)
    assert e.value.code == abi.ESTATE
    assert _state(ctx) == before
    ctx.analyze_pairs(download=False)
    # the image's capacity is the uploaded one after the successful call and after every refusal
    _capacity_is(ctx, oracle, img, pairs, feasible)
    got = ctx.solve_capacities(caps)
    sc.check(got, sc.expected(oracle, img, pairs, feasible, caps, False, abi.POLICY_NONE), "after re-analysis")


def test_chunks(wva, oracle, ctx):
    """a budget that splits 8 192 vectors at 61 x 4 into several chunks gives the unchunked call's bytes"""
    img, pairs, feasible = _generated(wva, ctx, S=61, A=4, T=2, seed=31)
    base = sc.ladder(img, pairs, feasible, oracle, n=64)
    rng = np.random.default_rng(7)
    caps = base[rng.integers(0, len(base), 8192)]
    caps[::7] = (caps[::7] * rng.uniform(0.5, 1.5, caps[::7].shape)).astype(np.int64)
    for policy in (abi.POLICY_NONE, abi.POLICY_PRIORITY_EXHAUSTIVE):
        whole = ctx.solve_capacities(caps, policy=policy)
        assert ctx.solve_capacities_counters()["chunks"] == 1
        try:
            ctx.solve_capacities_set_budget(1 << 20)
            parts = ctx.solve_capacities(caps, policy=policy)
            chunks = ctx.solve_capacities_counters()["chunks"]
        finally:
            ctx.solve_capacities_set_budget(0)
        assert chunks >= 3, chunks
        assert _bytes_equal(whole, parts), policy
        pick = np.arange(0, 8192, 401)
        sc.check(tuple(x[pick] for x in whole), sc.expected(oracle, img, pairs, feasible, caps[pick], False, policy), policy)
    # small lists over a tiny budget: one vector per chunk
    try:
        ctx.solve_capacities_set_budget(1)
        got = ctx.solve_capacities(caps[:5])
        assert ctx.solve_capacities_counters()["chunks"] == 5
    finally:
        ctx.solve_capacities_set_budget(0)
    assert _bytes_equal(got, ctx.solve_capacities(caps[:5]))


# ---- sharded runs ------------------------------------------------------------------------------------------------
SHARDED_IMAGE = "P2"          # tests/rank_emulation.py: 61 x 4, 2 types, capacities at 0.55 of the demand
LOOPBACK_DRIVER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "solve_capacities_loopback_driver.py")


def _sharded_reference(oracle):
    import rank_emulation as re_
    ref = re_.reference(SHARDED_IMAGE)
    caps = sc.ladder(ref.img, ref.pairs, ref.feasible, oracle, n=16)
    return ref, caps


@pytest.mark.parametrize("G", [2, 3])
def test_rank_emulation(wva, oracle, G):
    """G contexts on one device, each sizing its shard; rows exchanged through wva_pairs_device / wva_pairs_commit.  Before
    the exchange the call is refused (incomplete rows, no communicator); after it every rank returns the same bytes, equal
    to the oracle's (totals: the ascending sum over all S servers)"""
    from inferno_autoscaler_b200 import binding
    from test_rank_emulation_gpu import gather_rows, setup_ranks
    ref, caps = _sharded_reference(oracle)
    policy = abi.POLICY_PRIORITY_EXHAUSTIVE
    all_ctxs = [binding.Context(0) for _ in range(G)]
    try:
        ctxs, shards = setup_ranks(all_ctxs, ref.img, G)
        for c in ctxs:
            c.analyze_pairs(download=False)
        for c in ctxs:
            with pytest.raises(binding.WvaError) as e:
                c.solve_capacities(caps, policy=policy)
            assert e.value.code == abi.ESTATE
        gather_rows(ctxs, shards, ref.img)
        want = sc.expected(oracle, ref.img, ref.pairs, ref.feasible, caps, True, policy)
        outs = [c.solve_capacities(caps, delayed_best_effort=True, policy=policy) for c in ctxs]
        for r, got in enumerate(outs):
            sc.check(got, want, (G, r))
            assert _bytes_equal(got, outs[0]), (G, r)
            assert ctxs[r].solve_capacities_counters()["path"] == 3
    finally:
        for c in all_ctxs:
            c.close()


def _drive(case, cfg, img, caps):
    """one case of tests/solve_capacities_loopback_driver.py in a torch-free subprocess (the loopback NCCL stand-in)"""
    import json
    import subprocess
    import tempfile
    from test_nccl_loopback_gpu import image_arrays
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.npz"), os.path.join(d, "out.npz")
        np.savez(src, cfg=np.array(json.dumps(cfg)), caps=caps, **image_arrays("img", img))
        p = subprocess.run([sys.executable, LOOPBACK_DRIVER, case, src, dst], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           timeout=600)
        assert p.returncode == 0, p.stdout.decode(errors="replace")[-4000:]
        return dict(np.load(dst, allow_pickle=False))


def _res(out, key):
    return out[key + ".acc"], out[key + ".recs"], out[key + ".count"], out[key + ".cost"]


@pytest.mark.parametrize("G", [2, 3])
def test_loopback_comm_gathers_once(oracle, G):
    """wva_comm_init ranks that sized only their shard: the first call makes exactly one pair all-gather on every rank, the
    second none; every rank's results equal the oracle's"""
    ref, caps = _sharded_reference(oracle)
    policy = abi.POLICY_ROUND_ROBIN
    caps = np.minimum(caps, st.ROUND_ROBIN_ROUNDS)
    out = _drive("comm", dict(G=G, policy=policy, delayed=False), ref.img, caps)
    want = sc.expected(oracle, ref.img, ref.pairs, ref.feasible, caps, False, policy)
    for r in range(G):
        p = "r%d" % r
        assert out[p + ".shard"][1] < ref.img.S, (G, r)                    # a proper shard: the rows were incomplete
        assert out[p + ".gathers"].tolist() == [1, 0], (G, r)
        assert int(out[p + ".path"]) == 3
        sc.check(_res(out, p + ".first"), want, (G, r))
        assert _bytes_equal(_res(out, p + ".first"), _res(out, p + ".second")), (G, r)


@pytest.mark.parametrize("G", [2, 3])
def test_group_equals_plain_context(oracle, G):
    """wva_group_solve_capacities over [0] * G: one all-gather per member on the first call, none on the second, member
    0's results equal a plain context's and the oracle's; a member without valid records refuses the call before any
    member gathers"""
    ref, caps = _sharded_reference(oracle)
    policy = abi.POLICY_PRIORITY_ROUND_ROBIN
    caps = np.minimum(caps, st.ROUND_ROBIN_ROUNDS)
    out = _drive("group", dict(G=G, policy=policy, delayed=True), ref.img, caps)
    assert len(out["shards"]) == G and (out["shards"][:, 1] < ref.img.S).all()
    assert out["gathers"].tolist() == [[1] * G, [0] * G]
    single = _res(out, "single")
    assert _bytes_equal(_res(out, "group"), single) and _bytes_equal(_res(out, "again"), single)
    sc.check(single, sc.expected(oracle, ref.img, ref.pairs, ref.feasible, caps, True, policy), G)
    assert int(out["refused"]) == abi.ESTATE and "device" in str(out["refused.msg"])
    assert out["refused.gathers"].tolist() == [0] * G
