"""GPU: the limited-capacity solve over a matrix of arrival-rate scenarios (wva_solve_loads) against the oracle (one
analyze_pairs -> limited solve -> allocate_by_type per column) and against the library's own per-scenario loop
(wva_system_update_servers -> wva_analyze_pairs -> wva_solve -> wva_solution_fetch -> wva_allocate_by_type), on a
config-3-shaped image, across chunk boundaries, on every solver path, on images whose pairs take the materialised-p[]
path, and around the state the call must leave alone."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solve_capacities_cases as sc
import solve_inject_tables as st
import solve_loads_cases as lc
from test_pairs_loads_cpu import with_rates
from test_pairs_loads_gpu import _finishing
from test_profile_edges_gpu import FAMILIES, pairs_image
from test_solve_capacities_gpu import _state

pytestmark = pytest.mark.gpu
abi = st.abi
F = np.float32


def _with_capacity(img, cap):
    out = img.shard(0, img.S)
    out.type_capacity[:] = cap
    return out


def _loop(ctx, rpm, delayed, policy):
    """the public loop, one scenario at a time; the uploaded rates are restored afterwards"""
    img = ctx.image
    base = img.shard(0, img.S)
    n, S, T = rpm.shape[1], img.S, img.T
    acc = np.zeros((n, S), dtype=np.int32)
    recs = np.zeros((n, S), dtype=abi.PAIR_REC_DTYPE)
    count = np.zeros((n, T), dtype=np.int64)
    cost = np.zeros((n, T), dtype=np.float32)
    for j in range(n):
        ctx.update_servers(0, with_rates(base, rpm[:, j]))
        ctx.analyze_pairs(download=False)
        ctx.solve(unlimited=False, delayed_best_effort=delayed, policy=policy, download=False)
        a, ch = ctx.solution_fetch()
        acc[j], recs[j] = a, sc.to_recs(a, ch)
        count[j], cost[j] = ctx.allocate_by_type()
    ctx.update_servers(0, base)
    return acc, recs, count, cost


def _bytes_equal(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


_C3 = {}


def _config3(wva, oracle):
    """config 3 (1 000 x 8, 3 types), 47 forecast multipliers 0.2 ... 2.0 and a zero column, sized by the oracle once"""
    if not _C3:
        img, _ = wva.synth.baseline_config(3)
        rpm = lc.forecast(img, 48)
        _C3.update(img=img, rpm=rpm, cols=lc.oracle_columns(oracle, img, rpm))
    return _C3["img"], _C3["rpm"], _C3["cols"]


@pytest.mark.parametrize("delayed", [False, True])
@pytest.mark.parametrize("policy", st.POLICIES)
def test_config3_against_oracle(wva, oracle, ctx, policy, delayed):
    img, rpm, cols = _config3(wva, oracle)
    cap = lc.binding(img, oracle, cols, round_robin=policy in st.ROUND_ROBIN)
    ctx.upload(_with_capacity(img, cap))
    got = ctx.solve_loads(rpm, delayed_best_effort=delayed, policy=policy)
    c = ctx.solve_loads_counters()
    assert c["path"] == 3 and c["chunks"] == 1 and c["max_cycles"] > 0 and c["sized_pairs"] > 0 and c["analyzed"] > 0
    want = lc.expected(oracle, cols, cap, delayed, policy)
    sc.check(got, want, (policy, delayed))
    acc = got[0]
    assert len({a.tobytes() for a in acc}) > 20                               # decisions follow the load
    has_cand = np.array([f.reshape(img.S, img.A).any(axis=1) for _, _, f in cols])
    assert ((acc < 0) & has_cand).any()                                       # the capacities bind somewhere


@pytest.mark.parametrize("policy", [abi.POLICY_NONE, abi.POLICY_PRIORITY_EXHAUSTIVE, abi.POLICY_PRIORITY_ROUND_ROBIN])
def test_equals_the_library_loop(wva, oracle, ctx, policy):
    """byte-equal to the public loop; the column of the uploaded rates gives a plain wva_solve + wva_allocate_by_type"""
    img = wva.synth.make_system(300, 6, seed=21, n_types=3, zero_load_fraction=0.1)
    rpm = lc.mixed(img)
    cap = lc.binding(img, oracle, lc.oracle_columns(oracle, img, rpm[:, :3]), round_robin=policy in st.ROUND_ROBIN)
    ctx.upload(_with_capacity(img, cap))
    for delayed in (False, True):
        got = ctx.solve_loads(rpm, delayed_best_effort=delayed, policy=policy)
        assert _bytes_equal(got, _loop(ctx, rpm, delayed, policy)), (policy, delayed)
        ctx.analyze_pairs(download=False)
        a, ch = ctx.solve(unlimited=False, delayed_best_effort=delayed, policy=policy)
        count, cost = ctx.allocate_by_type()
        assert got[0][0].tobytes() == a.tobytes() and got[1][0].tobytes() == sc.to_recs(a, ch).tobytes()
        assert got[2][0].tobytes() == count.tobytes() and got[3][0].tobytes() == cost.tobytes()


def test_chunks(wva, oracle, ctx):
    img = wva.synth.make_system(300, 6, seed=21, n_types=3, zero_load_fraction=0.1)
    rpm = lc.mixed(img)
    cap = lc.binding(img, oracle, lc.oracle_columns(oracle, img, rpm[:, :3]))
    ctx.upload(_with_capacity(img, cap))
    whole = ctx.solve_loads(rpm, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
    assert ctx.solve_loads_counters()["chunks"] == 1
    # a scenario stages at least its plane, slow list and records (48 + 8 + 45 bytes a pair): a budget of three times
    # that holds at most three scenarios
    low = img.S * img.A * (48 + 8 + 45)
    try:
        for budget, chunks in ((1, rpm.shape[1]), (3 * low, None), (2 * low, None)):
            ctx.solve_loads_set_budget(budget)
            got = ctx.solve_loads(rpm, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
            c = ctx.solve_loads_counters()["chunks"]
            assert c == chunks if chunks else c >= 4, (budget, c)
            assert _bytes_equal(got, whole), budget
    finally:
        ctx.solve_loads_set_budget(0)


def test_every_solver_path(wva, oracle, ctx):
    img = wva.synth.make_system(200, 8, seed=23, n_types=3, zero_load_fraction=0.1)
    rpm = lc.mixed(img)
    cols = lc.oracle_columns(oracle, img, rpm)
    cap = lc.binding(img, oracle, cols)
    ctx.upload(_with_capacity(img, cap))
    want = lc.expected(oracle, cols, cap, True, abi.POLICY_PRIORITY_EXHAUSTIVE)
    try:
        for ranked, path in ((2, 3), (1, 2), (0, 1)):
            ctx.solve_set_ranked(ranked)
            got = ctx.solve_loads(rpm, delayed_best_effort=True, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
            c = ctx.solve_loads_counters()
            assert c["path"] == path and (c["max_cycles"] > 0) == (path == 3), ranked
            sc.check(got, want, ranked)
    finally:
        ctx.solve_set_ranked(2)
    # more than 32 accelerators: the ranked queue by itself
    img = wva.synth.make_system(60, 33, seed=24, n_types=4, zero_load_fraction=0.1)
    rpm = lc.mixed(img)[:, :6]
    cols = lc.oracle_columns(oracle, img, rpm)
    cap = lc.binding(img, oracle, cols)
    ctx.upload(_with_capacity(img, cap))
    got = ctx.solve_loads(rpm, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
    assert ctx.solve_loads_counters()["path"] == 2
    sc.check(got, lc.expected(oracle, cols, cap, False, abi.POLICY_PRIORITY_EXHAUSTIVE), "A=33")


def test_round_robin_tickets_in_hbm(wva, oracle, ctx):
    """S = 8 000: the stopped bits and the ticket pool (36 bytes a server) no longer fit shared memory together"""
    img = wva.synth.make_system(8000, 2, seed=25, n_types=2)
    assert (8000 + 31) // 32 * 4 + 8000 * 36 > 220 * 1024
    rpm = lc.forecast(img, 4, lo=0.5, hi=1.5)
    cols = lc.oracle_columns(oracle, img, rpm)
    cap = lc.binding(img, oracle, cols, round_robin=True)
    ctx.upload(_with_capacity(img, cap))
    for policy in st.ROUND_ROBIN:
        got = ctx.solve_loads(rpm, policy=policy)
        assert ctx.solve_loads_counters()["path"] == 3
        sc.check(got, lc.expected(oracle, cols, cap, False, policy), policy)


def _overflow_image(wva):
    """tests/test_pairs_loads_gpu.py's overflow image: chains that need the materialised p[] path"""
    img = wva.synth.make_system(6, 2, seed=5, max_pair_batch=0)
    img.perf_alpha[:] = 20.0; img.perf_beta[:] = 1e-4; img.perf_gamma[:] = 10.0; img.perf_delta[:] = 1e-7  # noqa: E702
    img.perf_valid[:] = 1; img.srv_target_valid[:] = 1  # noqa: E702
    img.srv_max_batch[:] = [900, 1500, 2500, 1200, 3000, 2000]
    img.srv_arrival_rpm[:] = [3e5, 6e5, 2e6, 1e3, 5e6, 9e5]
    img.srv_in_tokens[:] = 64; img.srv_out_tokens[:] = 8  # noqa: E702
    img.srv_slo_itl[:] = 200.0; img.srv_slo_ttft[:] = 2000.0; img.srv_slo_tps[:] = 0.0  # noqa: E702
    img.srv_keep_acc[:] = 0
    return img


def test_materialised_path_images(wva, oracle, ctx):
    img = _overflow_image(wva)
    rpm = (img.srv_arrival_rpm.astype(F)[:, None] * np.array([0.5, 1.0, 2.0, 0.0], dtype=F)[None, :]).astype(F)
    cases = [(img, rpm)]
    for name in FAMILIES:
        im = pairs_image(wva, name)
        base = im.srv_arrival_rpm.astype(F)
        cases.append((im, _finishing(im, np.stack([F(f) * base for f in (0.0, 0.5, 1.0, 4.0)], axis=1).astype(F))))
    for k, (im, r) in enumerate(cases):
        cols = lc.oracle_columns(oracle, im, r)
        cap = lc.binding(im, oracle, cols)
        ctx.upload(_with_capacity(im, cap))
        got = ctx.solve_loads(r, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
        if k == 0:
            assert ctx.solve_loads_counters()["materialised"] > 0
        sc.check(got, lc.expected(oracle, cols, cap, False, abi.POLICY_PRIORITY_EXHAUSTIVE), k)


def test_nothing_else_moves_and_errors_change_nothing(wva, oracle, ctx):
    from inferno_autoscaler_b200 import binding
    fresh = binding.Context(0)
    fresh.image = wva.synth.config1()
    try:
        with pytest.raises(binding.WvaError) as e:
            fresh.solve_loads(np.ones((1, 2), dtype=F))
        assert e.value.code == abi.ESTATE
    finally:
        fresh.close()
    img = wva.synth.make_system(80, 4, seed=26, n_types=2, zero_load_fraction=0.1)
    rpm = lc.mixed(img)
    cap = lc.binding(img, oracle, lc.oracle_columns(oracle, img, rpm[:, :3]))
    ctx.upload(_with_capacity(img, cap))
    ctx.analyze(8, 64)
    ctx.analyze_pairs(download=False)
    ctx.solve(unlimited=True)
    ctx.allocate_by_type()
    ctx.analyze_pairs_loads(rpm[:, :2])
    ctx.solve_capacities(np.array([cap], dtype=np.int64))

    def snapshot():
        return (_state(ctx), ctx.solve_greedy_path(), tuple(ctx.solve_stats()), ctx.dims(), ctx.pairs_loads_counters(),
                ctx.solve_capacities_counters())

    before = snapshot()
    want = ctx.solve_loads(rpm, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
    assert snapshot() == before
    nan = rpm.copy()
    nan[7, 3] = np.nan
    spec_l = abi.OptimizerSpec(0, 0, abi.POLICY_NONE)
    spec_u = abi.OptimizerSpec(1, 0, abi.POLICY_NONE)
    L, C = binding.lib(), binding.C
    for bad in (rpm[:, :0], np.ones((img.S, 8193), dtype=F), nan):
        with pytest.raises(binding.WvaError) as e:
            ctx.solve_loads(bad)
        assert e.value.code == abi.EINVAL
    r = np.ascontiguousarray(rpm)
    assert L.wva_solve_loads(ctx._h, None, 2, abi.ptr(r, C.c_float), None, None, None, None) == abi.EINVAL
    assert L.wva_solve_loads(ctx._h, C.byref(spec_u), 2, abi.ptr(r, C.c_float), None, None, None, None) == abi.EINVAL
    assert L.wva_solve_loads(ctx._h, C.byref(spec_l), 2, None, None, None, None, None) == abi.EINVAL
    assert snapshot() == before
    # a limited solve right after the call runs on the untouched records; the call then works on the consumed records
    a0, ch0 = ctx.solve(unlimited=False, policy=abi.POLICY_PRIORITY_EXHAUSTIVE)
    assert want[0][0].tobytes() == a0.tobytes() and want[1][0].tobytes() == sc.to_recs(a0, ch0).tobytes()
    assert _bytes_equal(ctx.solve_loads(rpm, policy=abi.POLICY_PRIORITY_EXHAUSTIVE), want)
    # right after an upload, with no pair records at all
    ctx.upload(_with_capacity(img, cap))
    assert _bytes_equal(ctx.solve_loads(rpm, policy=abi.POLICY_PRIORITY_EXHAUSTIVE), want)
    # a shard that is not every server
    ctx.set_shard(0, img.S - 1)
    with pytest.raises(binding.WvaError) as e:
        ctx.solve_loads(rpm)
    assert e.value.code == abi.ESTATE
    # T > 256 and S = 0
    rng = np.random.Generator(np.random.PCG64(42))
    t = st.make_table(rng, 30, 8, 257, "types", type_map="scatter")
    ctx.upload(t.img)
    with pytest.raises(binding.WvaError) as e:
        ctx.solve_loads(np.ones((30, 2), dtype=F))
    assert e.value.code == abi.EINVAL
    empty = img.take(np.array([], dtype=np.int64))
    ctx.upload(empty)
    acc, recs, count, cost = ctx.solve_loads(np.zeros((0, 3), dtype=F))
    assert acc.shape == (3, 0) and (count == 0).all() and (cost.view(np.uint32) == 0).all()
    assert ctx.solve_loads_counters()["path"] == 0
