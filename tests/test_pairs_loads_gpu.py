"""GPU: pair sizing over arrival-rate scenarios (wva_analyze_pairs_loads).  Every record of scenario column j is compared
bit for bit with two witnesses -- the oracle's analyze_pairs on the image with srv_arrival_rpm = column j, and this
library's own wva_analyze_pairs after uploading that image -- and each (server, scenario)'s best record with the numpy
restatement of SolveUnlimited, the oracle's solve and wva_solve on the same image."""
import numpy as np
import pytest

from test_pairs_loads_cpu import boundary_rates, num_replicas, oracle_loads, rate_star, with_rates
from test_pairs_plane_cpu import choose, rec_bytes, to_recs
from test_profile_edges_gpu import FAMILIES, pairs_image

pytestmark = pytest.mark.gpu
F = np.float32


def empty_where(wva, acc, chosen):
    """wva_solve / oracle solve decisions -> wva_pair_rec: the chosen record with feasible = 1, the empty record where
    the server received none"""
    r = to_recs(wva, chosen, (acc >= 0).astype(np.uint8))
    r[acc < 0] = np.zeros(1, dtype=r.dtype)
    r["acc"][acc < 0] = -1
    return r


def gpu_loads(wva, ctx, img, rpm):
    """the second witness: wva_analyze_pairs after uploading each column, and wva_solve(unlimited)'s choice"""
    cols, best = [], []
    for j in range(rpm.shape[1]):
        ctx.upload(with_rates(img, rpm[:, j]))
        allocs, fe = ctx.analyze_pairs()
        cols.append(to_recs(wva, allocs, fe).reshape(img.S, img.A))
        acc, chosen = ctx.solve(unlimited=True)
        best.append(empty_where(wva, acc, chosen))
    return np.stack(cols, axis=1), np.stack(best, axis=1)


def oracle_best(wva, oracle, img, rpm):
    out = []
    for j in range(rpm.shape[1]):
        im = with_rates(img, rpm[:, j])
        allocs, fe, _ = oracle.analyze_pairs(im, threads=oracle.hardware_threads())
        acc, chosen = oracle.solve(im, allocs, fe, unlimited=True)
        out.append(empty_where(wva, acc, chosen))
    return np.stack(out, axis=1)


def choose_rows(plane):
    """numpy SolveUnlimited over each (server, scenario)'s A records: [S, n_l, A] -> [S, n_l]"""
    S, n_l, A = plane.shape
    return choose(plane.reshape(-1, 1), A).reshape(S, n_l)


def assert_loads(got, want):
    assert got.shape == want.shape
    bad = [j for j in range(got.shape[1]) if rec_bytes(got[:, j]) != rec_bytes(want[:, j])]
    assert not bad, "scenario columns %s differ" % bad


def sizing_pairs(img, rpm):
    """pairs that reach the queue analyzer under at least one positive scenario, from the image alone"""
    A = img.A
    valid = img.perf_valid.reshape(img.M, A)[img.srv_model] == 1
    ok = (img.srv_out_tokens > 0) & (img.srv_in_tokens >= 0) & (img.srv_target_valid == 1) & (rpm > 0).any(axis=1)
    cand = np.ones((img.S, A), bool)
    keep = (img.srv_keep_acc == 1) & (img.srv_cur_acc != -1)
    cand[keep] = np.arange(A)[None, :] == img.srv_cur_acc[keep][:, None]
    return int((valid & ok[:, None] & cand).sum())


def test_known_answers_config1(wva, oracle, ctx):
    img = wva.synth.config1()
    ctx.upload(img)
    own = img.srv_arrival_rpm[0]
    rpm = np.array([[own, 0.0, -1.0]], dtype=F)
    plane, best = ctx.analyze_pairs_loads(rpm)
    r = plane[0, 0, 0]
    assert r["feasible"] == 1 and r["num_replicas"] == 5
    assert r["itl"] == F(23.991173) and r["ttft"] == F(243.6568)
    allocs, fe = ctx.analyze_pairs()
    assert rec_bytes(plane[:, 0]) == rec_bytes(to_recs(wva, allocs, fe).reshape(1, 1))
    assert_loads(plane, oracle_loads(wva, oracle, img, rpm))
    z = plane[0, 1, 0]
    assert z["feasible"] == 1 and z["rho"] == 0 and z["num_replicas"] == img.srv_min_replicas[0]
    assert plane[0, 2, 0]["feasible"] == 0 and plane[0, 2, 0]["acc"] == -1
    assert rec_bytes(best) == rec_bytes(choose_rows(plane))


def _witness_images(wva):
    a = wva.synth.make_system(24, 4, seed=81, n_types=2, max_pair_batch=512, tps_fraction=0.2, keep_fraction=0.2)
    assert 0 < (a.srv_max_batch > 0).sum() < a.S and (a.srv_slo_tps > 0).any() and (a.srv_keep_acc == 1).any()
    b = wva.synth.make_system(16, 3, seed=82, n_types=3, max_pair_batch=0, zero_load_fraction=0.2)
    return [a, b]


def _witness_columns(img):
    base = img.srv_arrival_rpm.astype(F)
    cols = [F(f) * base for f in (0.0, 0.25, 1.0, 3.0, 40.0)]
    cols += [np.full(img.S, v, dtype=F) for v in (-0.0, -1.0, -np.inf, np.inf, 3e38, 1e15)]
    # the next float above the uploaded rate; a zero-load server keeps 0 (the float above 0 is a rate the reference
    # never finishes on, test_tiny_rates_give_the_empty_record)
    cols.append(np.where(base > 0, np.nextafter(base, F(np.inf)), base))
    return np.stack(cols, axis=1).astype(F)


@pytest.mark.parametrize("which", [0, 1])
def test_two_witnesses(wva, oracle, ctx, which):
    img = _witness_images(wva)[which]
    rpm = _witness_columns(img)
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    cnt = ctx.pairs_loads_counters()
    want = oracle_loads(wva, oracle, img, rpm)
    assert_loads(plane, want)
    g_plane, g_best = gpu_loads(wva, ctx, img, rpm)
    assert_loads(plane, g_plane)
    assert rec_bytes(best) == rec_bytes(choose_rows(want))
    assert rec_bytes(best) == rec_bytes(oracle_best(wva, oracle, img, rpm))
    assert rec_bytes(best) == rec_bytes(g_best)
    assert cnt["slices"] == 1 and cnt["sized_pairs"] == sizing_pairs(img, rpm) and cnt["analyzed"] > 0
    assert (plane["feasible"] == 1).sum() > plane.size // 8
    # a TPS-target server's record does not depend on the rate: every positive scenario gives the same one
    for s in np.nonzero(img.srv_slo_tps > 0)[0]:
        pos = np.nonzero(rpm[s] > 0)[0]
        assert all(rec_bytes(plane[s, j]) == rec_bytes(plane[s, pos[0]]) for j in pos[1:])
    # replica counts above 2^31 at 1e15 req/min
    assert (plane[:, 10]["num_replicas"][plane[:, 10]["feasible"] == 1] > 2 ** 31).any()


def test_replica_count_boundaries(wva, oracle, ctx):
    img = wva.synth.make_system(40, 3, seed=91, n_types=2, tps_fraction=0.0, zero_load_fraction=0.0)
    img.srv_keep_acc[:] = 0
    picks = []
    for s in range(img.S):
        a = s % img.A
        rs = rate_star(wva, oracle, img, s, a)
        if rs is not None and len(boundary_rates(rs)):
            picks.append((s, a, rs, boundary_rates(rs)))
    assert len(picks) >= 10
    n_l = max(len(p[3]) for p in picks)
    rpm = np.full((img.S, n_l), -1.0, dtype=F)
    for s, _, _, rates in picks:
        rpm[s, :len(rates)] = rates
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    want = oracle_loads(wva, oracle, img, rpm)
    assert_loads(plane, want)
    steps = 0
    for s, a, rs, rates in picks:
        got = plane[s, :len(rates), a]
        ok = got["feasible"] == 1
        assert list(got["num_replicas"][ok]) == [num_replicas(r, rs, img.srv_min_replicas[s]) for r in rates[ok]]
        steps += int((np.diff(got["num_replicas"][ok]) != 0).sum())
    assert steps > 0
    assert rec_bytes(best) == rec_bytes(choose_rows(want))


def test_config3_96_scenarios(wva, oracle, ctx):
    img, _ = wva.synth.baseline_config(3)
    A, n_l = img.A, 96
    rng = np.random.default_rng(93)
    fac = rng.uniform(0.0, 4.0, n_l).astype(F)
    fac[[7, 40, 88]] = 0.0
    rpm = (img.srv_arrival_rpm.astype(F)[:, None] * fac[None, :]).astype(F)
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    cnt = ctx.pairs_loads_counters()
    assert cnt["slices"] == 1
    assert cnt["sized_pairs"] == sizing_pairs(img, rpm)          # Size ran once per pair, not once per scenario
    assert cnt["analyzed"] > cnt["sized_pairs"] * 8
    assert rec_bytes(best) == rec_bytes(choose_rows(plane))
    servers = np.sort(rng.choice(img.S, 40, replace=False))
    sub = img.take(servers)
    want = oracle_loads(wva, oracle, sub, rpm[servers])
    assert_loads(plane[servers], want)
    assert rec_bytes(best[servers]) == rec_bytes(choose_rows(want))
    # 10^5 random (pair, scenario) records: per scenario the oracle sizes only the sampled pairs (config 3 has one model
    # per server, so a perf row is one pair)
    items = rng.choice(img.S * A * n_l, 100_000, replace=False)
    srv, col, acc = items // (A * n_l), (items // A) % n_l, items % A
    for j in np.unique(col):
        m = col == j
        ss, aa = srv[m], acc[m]
        us = np.unique(ss)
        sub = with_rates(img.take(us), rpm[us, j])
        keep = np.zeros(sub.M * A, np.uint8)
        pos = np.searchsorted(us, ss)
        keep[sub.srv_model[pos].astype(np.int64) * A + aa] = 1
        sub.perf_valid[:] &= keep
        allocs, fe, _ = oracle.analyze_pairs(sub, threads=oracle.hardware_threads())
        w = to_recs(wva, allocs, fe).reshape(len(us), A)[pos, aa]
        assert rec_bytes(plane[ss, j, aa]) == rec_bytes(w), int(j)
    _, best_only = ctx.analyze_pairs_loads(rpm, plane=False)
    assert rec_bytes(best_only) == rec_bytes(best)


def test_materialised_path_overflow_image(wva, oracle, ctx):
    img = wva.synth.make_system(6, 2, seed=5, max_pair_batch=0)
    img.perf_alpha[:] = 20.0; img.perf_beta[:] = 1e-4; img.perf_gamma[:] = 10.0; img.perf_delta[:] = 1e-7
    img.perf_valid[:] = 1; img.srv_target_valid[:] = 1
    img.srv_max_batch[:] = [900, 1500, 2500, 1200, 3000, 2000]
    img.srv_arrival_rpm[:] = [3e5, 6e5, 2e6, 1e3, 5e6, 9e5]
    img.srv_in_tokens[:] = 64; img.srv_out_tokens[:] = 8
    img.srv_slo_itl[:] = 200.0; img.srv_slo_ttft[:] = 2000.0; img.srv_slo_tps[:] = 0.0
    img.srv_keep_acc[:] = 0
    rpm = (img.srv_arrival_rpm.astype(F)[:, None] * np.array([0.5, 1.0, 2.0, 0.0], dtype=F)[None, :]).astype(F)
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    assert ctx.pairs_loads_counters()["materialised"] > 0
    want = oracle_loads(wva, oracle, img, rpm)
    assert_loads(plane, want)
    assert rec_bytes(best) == rec_bytes(choose_rows(want))


def _finishing(img, rpm):
    """rpm with every positive rate the reference never finishes on (numReplicas 0 at totalRate 0) made negative"""
    with np.errstate(under="ignore"):
        tiny = (rpm > 0) & (rpm / F(60) == 0) & (img.srv_slo_tps == 0)[:, None] & (img.srv_min_replicas == 0)[:, None]
    out = rpm.copy()
    out[tiny] = -1.0
    return out


@pytest.mark.parametrize("name", FAMILIES)
def test_materialised_path_profile_families(wva, oracle, ctx, name):
    """pairs whose RateRange.Max is +Inf cannot be sized by the reference at any load: they lose their perf row"""
    img = pairs_image(wva, name)
    base = img.srv_arrival_rpm.astype(F)
    rpm = _finishing(img, np.stack([F(f) * base for f in (0.0, 0.5, 1.0, 4.0)], axis=1).astype(F))
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    want = oracle_loads(wva, oracle, img, rpm)
    assert_loads(plane, want)
    assert rec_bytes(best) == rec_bytes(choose_rows(want))
    assert (plane["feasible"] == 1).any()


def test_tiny_rates_give_the_empty_record(wva, ctx):
    img = wva.synth.make_system(12, 3, seed=94, n_types=2, tps_fraction=0.0, zero_load_fraction=0.0)
    img.srv_min_replicas[:] = np.arange(img.S) % 3 - 1           # a negative floor too: numReplicas is then 0 as well
    tiny = np.array([1.4e-45, 2.8e-45, 4.2e-44], dtype=F)
    assert (tiny > 0).all() and (tiny / F(60) == 0).all()
    rpm = np.repeat(tiny[None, :], img.S, axis=0)
    rpm = np.concatenate([rpm, img.srv_arrival_rpm.astype(F)[:, None]], axis=1)
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    cnt = ctx.pairs_loads_counters()
    assert (plane[:, :3]["feasible"] == 0).all() and (plane[:, :3]["acc"] == -1).all()
    assert (plane[:, :3]["num_replicas"] == 0).all() and (best[:, :3]["acc"] == -1).all()
    assert cnt["materialised"] == 0
    allocs, fe = ctx.analyze_pairs()
    assert rec_bytes(plane[:, 3]) == rec_bytes(to_recs(wva, allocs, fe).reshape(img.S, img.A))


def test_slices_shards_and_groups(wva, oracle, ctx):
    A, n_l = 256, 16
    per_slice = (1 << 28) // (A * n_l * 48)
    S = 2 * per_slice + 270
    img = wva.synth.make_system(S, A, seed=95, n_types=4, max_pair_batch=512)
    rng = np.random.default_rng(96)
    edges = sorted({s for b in (0, per_slice, 2 * per_slice, S) for s in range(b - 2, b + 3) if 0 <= s < S})
    img.perf_valid[:] = 0
    for s in range(S):
        k = 4 if s in edges else int(rng.uniform() < 0.02)
        img.perf_valid[int(img.srv_model[s]) * A + rng.choice(A, k, replace=False)] = 1
    rpm = (img.srv_arrival_rpm.astype(F)[:, None] * rng.uniform(0.0, 3.0, n_l).astype(F)[None, :]).astype(F)
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_loads(rpm)
    cnt = ctx.pairs_loads_counters()
    assert cnt["slices"] == 3 and cnt["sized_pairs"] == sizing_pairs(img, rpm)
    want = oracle_loads(wva, oracle, img.take(edges), rpm[edges])
    assert_loads(plane[edges], want)
    assert rec_bytes(best[edges]) == rec_bytes(choose_rows(want))
    assert (plane[edges]["feasible"] == 1).any()
    # a shard is its rows of the full call; a one-device group equals the context
    small = _witness_images(wva)[0]
    srpm = _witness_columns(small)
    ctx.upload(small)
    full, fbest = ctx.analyze_pairs_loads(srpm)
    ctx.set_shard(5, 11)
    part, pbest = ctx.analyze_pairs_loads(srpm[5:16])
    assert rec_bytes(part) == rec_bytes(full[5:16]) and rec_bytes(pbest) == rec_bytes(fbest[5:16])
    from inferno_autoscaler_b200 import binding
    g = binding.Group([0])
    try:
        g.upload(small)
        gp, gb = g.analyze_pairs_loads(srpm)
    finally:
        g.close()
    assert rec_bytes(gp) == rec_bytes(full) and rec_bytes(gb) == rec_bytes(fbest)


def test_two_device_group_equals_one_context(wva, ctx):
    from inferno_autoscaler_b200 import binding
    try:
        g = binding.Group([0, 1])
    except binding.WvaError as e:
        if e.code not in (wva.abi.EINVAL, wva.abi.ECUDA):       # no device 1
            raise
        pytest.skip("needs 2 GPUs")
    small = _witness_images(wva)[0]
    srpm = _witness_columns(small)
    ctx.upload(small)
    full, fbest = ctx.analyze_pairs_loads(srpm)
    try:
        g.upload(small)
        gp, gb = g.analyze_pairs_loads(srpm)
        # a NaN in the second device's rows fails the call before the first device writes or counts anything
        before = [c.pairs_loads_counters() for c in g.ctxs]
        bad = srpm.copy()
        bad[-1, 2] = np.nan                                     # the last server is the second device's
        with pytest.raises(binding.WvaError) as e:
            g.analyze_pairs_loads(bad)
        assert e.value.code == wva.abi.EINVAL
        assert [c.pairs_loads_counters() for c in g.ctxs] == before
    finally:
        g.close()
    assert rec_bytes(gp) == rec_bytes(full) and rec_bytes(gb) == rec_bytes(fbest)


def test_certified_tails_do_not_change_the_plane(wva, ctx):
    img = wva.synth.make_system(40, 4, seed=97, n_types=2)
    rpm = _witness_columns(img)
    ctx.upload(img)
    got = [ctx.analyze_pairs_loads(rpm)]
    ctx.set_certified_tails(0)
    try:
        got.append(ctx.analyze_pairs_loads(rpm))
    finally:
        ctx.set_certified_tails(1)
    assert rec_bytes(got[0][0]) == rec_bytes(got[1][0]) and rec_bytes(got[0][1]) == rec_bytes(got[1][1])


def _state(wva, ctx):
    """every result the other calls read back"""
    pairs, fe = ctx.pairs_fetch()
    acc, chosen = ctx.solution_fetch()
    count, cost = ctx.allocate_by_type()
    return [rec_bytes(to_recs(wva, pairs, fe)), acc.tobytes(), rec_bytes(to_recs(wva, chosen, np.zeros(len(acc), np.uint8))),
            count.tobytes(), cost.tobytes(), ctx.grid_fetch().tobytes(), ctx.grid_best_blocking().tobytes()]


def test_nothing_else_moves_and_errors_change_nothing(wva, ctx):
    from inferno_autoscaler_b200 import binding
    fresh = binding.Context(0)
    fresh.image, fresh.count = wva.synth.config1(), 1
    try:
        with pytest.raises(binding.WvaError) as e:
            fresh.analyze_pairs_loads(np.ones((1, 2), dtype=F))
        assert e.value.code == wva.abi.ESTATE
    finally:
        fresh.close()
    img = wva.synth.make_system(50, 4, seed=98, n_types=2)
    rpm = _witness_columns(img)
    ctx.upload(img)
    ctx.analyze(8, 64)
    ctx.solve(unlimited=True)
    before = _state(wva, ctx)
    _, ok_best = ctx.analyze_pairs_loads(rpm)
    assert _state(wva, ctx) == before
    nan = rpm.copy()
    nan[7, 3] = np.nan
    for bad in (rpm[:, :0], np.ones((img.S, 8193), dtype=F), nan):
        with pytest.raises(binding.WvaError) as e:
            ctx.analyze_pairs_loads(bad)
        assert e.value.code == wva.abi.EINVAL
    assert binding.lib().wva_analyze_pairs_loads(ctx._h, 2, None, None, None) == wva.abi.EINVAL
    assert _state(wva, ctx) == before
    acc, _ = ctx.solve(unlimited=True)
    assert acc.tobytes() == before[1]
    # the resident rates were not touched: a later analyze_pairs gives the records of before
    allocs, fe = ctx.analyze_pairs()
    assert rec_bytes(to_recs(wva, allocs, fe)) == before[0]
    assert rec_bytes(ctx.analyze_pairs_loads(rpm)[1]) == rec_bytes(ok_best)


def test_follows_updates(wva, oracle, ctx):
    img = wva.synth.make_system(30, 3, seed=99, n_types=2)
    ctx.upload(img.shard(0, img.S))
    rows = img.shard(4, 3)
    rows.srv_arrival_rpm[:] *= F(5.0)
    rows.srv_min_replicas[:] = 2
    rows.srv_slo_itl[:] *= F(0.7)
    ctx.update_servers(4, rows)
    ctx.remove_server(9)
    cur = ctx.image.shard(0, ctx.image.S)
    rpm = _witness_columns(cur)
    plane, best = ctx.analyze_pairs_loads(rpm)
    want = oracle_loads(wva, oracle, cur, rpm)
    assert_loads(plane, want)
    assert rec_bytes(best) == rec_bytes(choose_rows(want))
