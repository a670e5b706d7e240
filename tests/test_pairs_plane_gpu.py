"""GPU: pair sizing over a batch-size list (wva_analyze_pairs_batches), every record compared bit for bit with two
witnesses -- the oracle's analyze_pairs on the image with srv_max_batch[:] = b, and this library's own
wva_analyze_pairs after uploading that image -- and each server's choice with the numpy restatement of
SolveUnlimited."""
import numpy as np
import pytest

from test_pairs_plane_cpu import choose, oracle_plane, override, rec_bytes, to_recs
from test_profile_edges_gpu import FAMILIES, family, rate_max, rate_table

pytestmark = pytest.mark.gpu
F = np.float32
WITNESS_LIST = [1, 2, 3, 31, 32, 33, 100, 512, 3072, 3073, 8192]


def gpu_override_plane(wva, ctx, img, batch):
    """the second witness: wva_analyze_pairs after uploading the image under each override"""
    cols = []
    for b in batch:
        ctx.upload(override(img, int(b)))
        allocs, fe = ctx.analyze_pairs()
        cols.append(to_recs(wva, allocs, fe))
    return np.stack(cols, axis=1)


def assert_plane(got, want):
    assert got.shape == want.shape
    bad = [k for k in range(got.shape[1]) if rec_bytes(got[:, k]) != rec_bytes(want[:, k])]
    assert not bad, "batch columns %s differ" % bad


def test_known_answers_config1(wva, oracle, ctx):
    img = wva.synth.config1()
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_batches([1, 8, 64, 256, 512])
    r = plane[0]
    assert r["feasible"][0] == 0 and r["acc"][0] == -1
    assert list(r["num_replicas"][1:4]) == [7, 5, 5] and r["feasible"][1:].all()
    assert list(r["batch_size"][1:]) == [8, 64, 256, 512]
    assert r["num_replicas"][4] == 5 and r["cost"][4] == F(160.0)
    assert r["itl"][4] == F(23.991173) and r["ttft"][4] == F(243.6568) and r["rho"][4] == F(0.012853656)
    assert rec_bytes(best) == rec_bytes(choose(plane, 1))
    # the iteration-budget image (a bisection that runs all 100 iterations: 122 Solves at its own batch size)
    c1 = wva.synth.config1()
    c1.srv_slo_itl[0] = 10.0; c1.srv_slo_ttft[0] = 1000.0
    c1.perf_alpha[0], c1.perf_beta[0], c1.perf_gamma[0], c1.perf_delta[0] = 7.470, 0.044, 15.415, 0.000337
    c1.acc_cost[0] = 100.0; c1.srv_arrival_rpm[0] = 6000.0
    batch = [1, 16, 100, 256, 512, 1024]
    want = oracle_plane(wva, oracle, c1, batch)
    for warp_max in (0, 1 << 22):
        ctx.pairs_set_warp_max(warp_max)
        ctx.upload(c1)
        plane, best = ctx.analyze_pairs_batches(batch)
        assert_plane(plane, want)
    ctx.pairs_set_warp_max(1 << 22)
    assert plane[0]["num_replicas"][4] == 3


def _witness_images(wva):
    a = wva.synth.make_system(24, 4, seed=71, n_types=2, max_pair_batch=512)     # mixed server overrides
    assert 0 < (a.srv_max_batch > 0).sum() < a.S
    b = wva.synth.make_system(16, 3, seed=72, n_types=3, max_pair_batch=0, zero_load_fraction=0.2)
    return [a, b]


@pytest.mark.parametrize("which", [0, 1])
def test_two_witnesses(wva, oracle, ctx, which):
    img = _witness_images(wva)[which]
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_batches(WITNESS_LIST)
    cnt = ctx.pairs_batches_counters()
    want = oracle_plane(wva, oracle, img, WITNESS_LIST)
    assert_plane(plane, want)
    assert_plane(plane, gpu_override_plane(wva, ctx, img, WITNESS_LIST))
    assert rec_bytes(best) == rec_bytes(choose(want, img.A))
    assert cnt["slices"] == 1 and cnt["sized"] > 0 and cnt["steps"] > 0
    assert (plane["feasible"] == 1).sum() > plane.size // 4
    # zero-load servers with minNumReplicas 1 carry the listed batch size
    zl = np.repeat((img.srv_arrival_rpm == 0) & (img.srv_min_replicas == 1), img.A) & (plane["feasible"][:, 0] == 1)
    if zl.any():
        assert (plane["batch_size"][zl] == np.array(WITNESS_LIST)).all()


def test_config3_full_list(wva, oracle, ctx):
    img, _ = wva.synth.baseline_config(3)
    batch = np.arange(1, 513)
    A, nB = img.A, len(batch)
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_batches(batch)
    cnt = ctx.pairs_batches_counters()
    assert cnt["slices"] == 1 and cnt["sized"] > img.S * A * 256
    assert rec_bytes(best) == rec_bytes(choose(plane, A))
    rng = np.random.default_rng(73)
    # 40 whole servers and their choice
    servers = np.sort(rng.choice(img.S, 40, replace=False))
    want = oracle_plane(wva, oracle, img.take(servers), batch)
    rows = (servers[:, None] * A + np.arange(A)).reshape(-1)
    assert_plane(plane[rows], want)
    assert rec_bytes(best[servers]) == rec_bytes(choose(want, A))
    # 10^5 random (pair, b) records: per b, the oracle sizes only the sampled pairs (every other perf row switched off;
    # config 3 has one model per server, so a perf row is one pair)
    items = rng.choice(img.S * A * nB, 100_000, replace=False)
    pair, col = items // nB, items % nB
    for j in np.unique(col):
        pj = np.sort(pair[col == j])
        srv = np.unique(pj // A)
        sub = override(img.take(srv), int(batch[j]))
        keep = np.zeros(sub.M * A, np.uint8)
        pos = np.searchsorted(srv, pj // A)
        keep[sub.srv_model[pos].astype(np.int64) * A + pj % A] = 1
        sub.perf_valid[:] &= keep
        allocs, fe, _ = oracle.analyze_pairs(sub, threads=oracle.hardware_threads())
        got = plane[pj, j]
        assert rec_bytes(got) == rec_bytes(to_recs(wva, allocs, fe)[pos * A + pj % A]), int(batch[j])
    _, best_only = ctx.analyze_pairs_batches(batch, plane=False)
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
    batch = [900, 1200, 1500, 2000, 2500, 3000]
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_batches(batch)
    assert ctx.pairs_batches_counters()["materialised"] > 0
    want = oracle_plane(wva, oracle, img, batch)
    assert_plane(plane, want)
    assert rec_bytes(best) == rec_bytes(choose(want, img.A))


def _sizing_ends(img, s, a, batch):
    """for each listed b: whether the reference's sizing of the item terminates -- it does not when RateRange.Max is
    +Inf at b (Size's bisection then evaluates lambda = +Inf, test_profile_edges_gpu.unsizable_pairs)"""
    with np.errstate(all="ignore"):
        tab = rate_table(img, s, a, batch[-1])
        return np.array([not np.isposinf(rate_max(tab[:b])[-1]) for b in batch])


def _family_case(wva, name):
    """the family's pair image, a list on both sides of its pairs' first bad table entries, and which items
    ([S * A, n_b]) the reference can size"""
    img = family(wva, name)[0]
    firsts = {}
    with np.errstate(all="ignore"):
        for s in range(img.S):
            for a in range(img.A):
                tab = rate_table(img, s, a, 8192)
                bad = np.nonzero(~((tab > 0) & np.isfinite(tab)))[0]
                if len(bad):
                    firsts[(s, a)] = int(bad[0]) + 1          # the first batch size whose table holds it
    fb = sorted(set(firsts.values()))
    picks = fb[:3] + fb[-2:]
    batch = sorted({1, 2, 64} | {b + d for b in picks for d in (-1, 0, 1) if 1 <= b + d <= 2048})
    ends = np.array([_sizing_ends(img, s, a, batch) for s in range(img.S) for a in range(img.A)])
    return img, batch, ends, firsts


@pytest.mark.parametrize("name", FAMILIES)
def test_materialised_path_profile_families(wva, oracle, ctx, name):
    """Items the reference cannot size are left out item by item: for each distinct first such batch index u, the
    pairs that end up to it are sized over batch[:u] (the others lose their perf row in that call only), and their
    items below u are compared."""
    img, batch, ends, firsts = _family_case(wva, name)
    A = img.A
    # the number of leading listed batch sizes each pair can be sized at
    upto = np.where(ends.all(axis=1), len(batch), np.argmin(ends, axis=1))
    compared = feasible = materialised = 0
    for u in sorted(set(upto.tolist()) - {0}):
        sub = img.shard(0, img.S)
        for p in np.nonzero(upto < u)[0]:
            sub.perf_valid[int(img.srv_model[p // A]) * A + p % A] = 0
        ctx.upload(sub)
        plane, best = ctx.analyze_pairs_batches(batch[:u])
        materialised += ctx.pairs_batches_counters()["materialised"]
        want = oracle_plane(wva, oracle, sub, batch[:u])
        mine = np.nonzero(upto == u)[0]
        assert rec_bytes(plane[mine]) == rec_bytes(want[mine])
        assert rec_bytes(best) == rec_bytes(choose(want, A))
        compared += mine.size * u
        feasible += int((plane[mine]["feasible"] == 1).sum())
    assert compared > 0 and feasible > 0
    # every item whose table prefix holds a bad entry goes to the materialised path, and the items of the same pairs at
    # smaller b mostly do not (a chain that rescales goes there too): the entry is compared with each item's b, not with
    # the call's largest
    def sized(s, a):
        return (img.perf_valid[int(img.srv_model[s]) * A + a] and img.srv_target_valid[s] and img.srv_arrival_rpm[s] > 0
                and img.srv_out_tokens[s] > 0 and img.srv_in_tokens[s] >= 0
                and not (img.srv_keep_acc[s] and img.srv_cur_acc[s] != -1 and img.srv_cur_acc[s] != a))
    prefix_bad = sum(sum(1 for b in batch[:upto[s * A + a]] if f <= b) for (s, a), f in firsts.items() if sized(s, a))
    whole_table = sum(upto[s * A + a] for (s, a), f in firsts.items() if sized(s, a) and f <= batch[upto[s * A + a] - 1])
    assert prefix_bad <= materialised
    if whole_table > prefix_bad:
        assert materialised < whole_table


def test_certified_tails_do_not_change_the_plane(wva, ctx):
    img = wva.synth.make_system(40, 4, seed=74, n_types=2)
    batch = [1, 7, 64, 300, 512, 2000]
    ctx.upload(img)
    got = [ctx.analyze_pairs_batches(batch)]
    ctx.set_certified_tails(0)
    try:
        got.append(ctx.analyze_pairs_batches(batch))
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


def test_nothing_else_moves(wva, ctx):
    img = wva.synth.make_system(50, 4, seed=75, n_types=2)
    ctx.upload(img)
    ctx.analyze(8, 64)
    ctx.solve(unlimited=True)
    before = _state(wva, ctx)
    ctx.analyze_pairs_batches([1, 5, 128, 600])
    after = _state(wva, ctx)
    assert before == after
    acc, chosen = ctx.solve(unlimited=True)
    assert acc.tobytes() == before[1]


def test_slices_and_shards(wva, oracle, ctx):
    A, batch = 256, [1, 2, 4, 8, 16, 24, 32, 48, 64, 96, 128, 160, 192, 224, 256, 320]
    per_slice = (1 << 28) // (A * len(batch) * 48)
    S = 2 * per_slice + 270
    img = wva.synth.make_system(S, A, seed=76, n_types=4, max_pair_batch=512)
    rng = np.random.default_rng(77)
    edges = sorted({s for b in (0, per_slice, 2 * per_slice, S) for s in range(b - 2, b + 3) if 0 <= s < S})
    img.perf_valid[:] = 0
    for s in range(S):
        k = 4 if s in edges else int(rng.uniform() < 0.02)
        img.perf_valid[int(img.srv_model[s]) * A + rng.choice(A, k, replace=False)] = 1
    ctx.upload(img)
    plane, best = ctx.analyze_pairs_batches(batch)
    cnt = ctx.pairs_batches_counters()
    assert cnt["slices"] == 3
    # every item that reaches the queue analyzer is sized: the count follows from the image alone
    m = img.srv_model
    valid = img.perf_valid.reshape(img.M, A)[m] == 1
    load = (img.srv_arrival_rpm > 0) & (img.srv_out_tokens > 0) & (img.srv_in_tokens >= 0) & (img.srv_target_valid == 1)
    cand = np.ones((S, A), bool)
    keep = (img.srv_keep_acc == 1) & (img.srv_cur_acc != -1)
    cand[keep] = np.arange(A)[None, :] == img.srv_cur_acc[keep][:, None]
    assert cnt["sized"] == len(batch) * int((valid & load[:, None] & cand).sum())
    want = oracle_plane(wva, oracle, img.take(edges), batch)
    rows = (np.array(edges)[:, None] * A + np.arange(A)).reshape(-1)
    assert_plane(plane[rows], want)
    assert rec_bytes(best[edges]) == rec_bytes(choose(want, A))
    assert (plane[rows]["feasible"] == 1).sum() > 0
    # a shard is the same servers of the full plane; a one-device group equals the context
    small = _witness_images(wva)[0]
    ctx.upload(small)
    full, fbest = ctx.analyze_pairs_batches(WITNESS_LIST[:8])
    ctx.set_shard(5, 11)
    part, pbest = ctx.analyze_pairs_batches(WITNESS_LIST[:8])
    assert rec_bytes(part) == rec_bytes(full[5 * small.A:16 * small.A]) and rec_bytes(pbest) == rec_bytes(fbest[5:16])
    from inferno_autoscaler_b200 import binding
    g = binding.Group([0])
    try:
        g.upload(small)
        gp, gb = g.analyze_pairs_batches(WITNESS_LIST[:8])
    finally:
        g.close()
    assert rec_bytes(gp) == rec_bytes(full) and rec_bytes(gb) == rec_bytes(fbest)


def test_errors_leave_state_untouched(wva, ctx):
    from inferno_autoscaler_b200 import binding
    fresh = binding.Context(0)
    fresh.image, fresh.count = wva.synth.config1(), 1
    try:
        with pytest.raises(binding.WvaError) as e:
            fresh.analyze_pairs_batches([1, 2])
        assert e.value.code == wva.abi.ESTATE
    finally:
        fresh.close()
    img = wva.synth.make_system(20, 3, seed=78, n_types=2)
    ctx.upload(img)
    ctx.analyze(4, 32)
    ctx.solve(unlimited=True)
    before = ctx.pairs_fetch()
    _, ok_best = ctx.analyze_pairs_batches([4, 8])
    for bad in ([2, 1], [3, 3], [0, 5], [1, 8193], [], list(range(1, 8194))):
        with pytest.raises(binding.WvaError) as e:
            ctx.analyze_pairs_batches(bad)
        assert e.value.code == wva.abi.EINVAL, bad
    after = ctx.pairs_fetch()
    assert rec_bytes(to_recs(wva, *before)) == rec_bytes(to_recs(wva, *after))
    ctx.solve(unlimited=True)
    ctx.grid_fetch()
    assert rec_bytes(ctx.analyze_pairs_batches([4, 8])[1]) == rec_bytes(ok_best)
