"""GPU: the blocking probability of sweep candidates (wva_grid_blocking, wva_grid_best_blocking) against the oracle,
bit for bit, a NaN on both sides counting as equal.

  * config 2: the whole 4 194 304-candidate plane, and cube.throughput == f32(f32(lambda f32(1 - p_block)) 1000) on the
    cube of the same sweep;
  * config 3 (bench.py's default workload, default path): >= 1e6 random candidates, every candidate the plane ran as an
    exact chain, and every server's winner;
  * the performance-profile families of test_profile_edges_gpu, whole planes, plus a fixture whose rates sit a few ulps
    under RateRange.Max at b = 1..4 (p_block of a few percent, decided by the closed form);
  * the new calls change nothing the sweep, the pair sizing or the solver produced, and refuse to run on stale state;
  * a server slice, a one-device group and (with two GPUs) a two-device group.
"""
import numpy as np
import pytest

from test_blocking_cpu import check_throughput_identity
from test_profile_edges_gpu import FAMILIES, family, rate_max, rate_table

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


def _threads(oracle):
    return max(1, oracle.hardware_threads())


def _decode(idx, A, R, B):
    idx = np.asarray(idx, dtype=np.int64)
    b = (idx % B + 1).astype(np.int32)
    r = ((idx // B) % R + 1).astype(np.int32)
    pair = idx // (B * R)
    return (pair // A).astype(np.int32), (pair % A).astype(np.int32), r, b


def _mismatch(got, want):
    """first index whose float differs bit for bit (NaN == NaN), or None"""
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    bad = np.flatnonzero(~same)
    return None if len(bad) == 0 else int(bad[0])


def _check_ids(ob, oracle, img, p, ids, R, B, first=0):
    s, a, r, b = _decode(ids, img.A, R, B)
    _, _, want = ob.grid_candidates_blocking(img, s + first, a, r, b, threads=_threads(oracle))
    bad = _mismatch(p[ids], want)
    assert bad is None, (int(ids[bad]), float(p[ids][bad]), float(want[bad]))


def test_config2_whole_plane(wva, oracle, ob, ctx):
    img, c = wva.synth.baseline_config(2)
    R, B = c["r_max"], c["b_max"]
    ctx.upload(img)
    _, cube, status = ctx.analyze_grid(R, B, want_cube=True)
    p = ctx.grid_blocking()
    counts = ctx.grid_blocking_counts()
    _, w_status, want = ob.grid_plane_blocking(img, R, B, threads=_threads(oracle))
    assert np.array_equal(status, w_status)
    bad = _mismatch(p, want)
    assert bad is None, (bad, float(p[bad]), float(want[bad]))
    s, _, r, _ = _decode(np.arange(len(p)), img.A, R, B)
    n_ok = check_throughput_identity(img, s, r, cube, status, p)
    assert counts["zero"] + counts["closed_form"] + counts["exact"] >= n_ok
    assert counts["zero"] > 0 and counts["closed_form"] > 0
    print("config 2 blocking counts: %s, %d analysed of %d" % (counts, n_ok, len(p)))


def test_config3_random_exact_and_winners(wva, oracle, ob, ctx):
    img, c = wva.synth.baseline_config(3)
    R, B = c["r_max"], c["b_max"]
    ctx.upload(img)
    ctx.analyze(R, B, want_cube=False)
    p = ctx.grid_blocking()
    counts = ctx.grid_blocking_counts()
    exact, n_exact = ctx.grid_blocking_exact()
    assert len(exact) > 0 and n_exact >= len(exact)
    rng = np.random.default_rng(3)
    ids = np.sort(rng.choice(len(p), 1_000_000, replace=False))
    _check_ids(ob, oracle, img, p, ids, R, B)
    _check_ids(ob, oracle, img, p, exact.astype(np.int64), R, B)
    best = ctx.grid_fetch()
    wb = ctx.grid_best_blocking()
    has = best["acc"] >= 0
    assert has.any() and np.isnan(wb[~has]).all()
    srv = np.flatnonzero(has).astype(np.int32)
    _, st, want = ob.grid_candidates_blocking(img, srv, best["acc"][has], best["replicas"][has], best["batch"][has],
                                              threads=_threads(oracle))
    assert (st & 1).all()
    assert _mismatch(wb[has], want) is None
    widx = ((srv.astype(np.int64) * img.A + best["acc"][has]) * R + best["replicas"][has] - 1) * B + best["batch"][has] - 1
    assert _mismatch(p[widx], wb[has]) is None
    print("config 3 blocking counts: %s; %d random + %d exact-chain candidates and %d winners checked" %
          (counts, len(ids), len(exact), int(has.sum())))


def _near_max(wva):
    """rows whose rate is k ulps under RateRange.Max at b = 1..4 (r = 1): heavily loaded, p_block of a few percent"""
    img = wva.synth.make_system(8, 2, seed=23, n_types=2, zero_load_fraction=0.0)
    img.srv_slo_tps[:] = 0
    targets = []
    for s in range(img.S):
        bstar, k = 1 + s % 4, s // 4
        target = rate_max(rate_table(img, s, 0, bstar))[bstar - 1]
        for _ in range(k):
            target = np.nextafter(target, F(0))
        arr = F(float(target) * 60.0)
        while F(arr / F(60)) > target:
            arr = np.nextafter(arr, F(0))
        img.srv_arrival_rpm[s] = arr
        targets.append((s, bstar))
    return img, 4, 8, targets


def test_profile_families_whole_plane(wva, oracle, ob, ctx):
    """every family's whole plane; each of the three ways of deciding p_block runs somewhere"""
    total = dict(zero=0, closed_form=0, exact=0)
    cases = [(name,) + family(wva, name) for name in FAMILIES]
    img, R, B, targets = _near_max(wva)
    cases.append(("near_max", img, R, B))
    for name, img, R, B in cases:
        ctx.upload(img)
        ctx.analyze_grid(R, B, want_cube=False)
        p = ctx.grid_blocking()
        counts = ctx.grid_blocking_counts()
        _, _, want = ob.grid_plane_blocking(img, R, B, threads=_threads(oracle))
        bad = _mismatch(p, want)
        assert bad is None, (name, bad, float(p[bad]), float(want[bad]))
        for k in total:
            total[k] += counts[k]
        print("%s blocking counts: %s" % (name, counts))
        if name == "near_max":
            exact, _ = ctx.grid_blocking_exact()
            idx = np.array([((s * img.A) * R) * B + bstar - 1 for s, bstar in targets])
            idx = idx[~np.isnan(p[idx])]                    # analysed (a pair may lack its perf row)
            assert len(idx) >= 4 and (p[idx] > 1e-3).all(), p[idx]
            closed = np.setdiff1d(idx, exact)
            assert len(closed) > 0                          # the closed form decided some of these
    assert total["zero"] > 0 and total["closed_form"] > 0 and total["exact"] > 0, total


def test_blocking_calls_do_not_disturb_analyze_and_optimize(wva, ctx):
    """cube, status bytes, winners, pair records, decisions and totals are byte-identical with and without the new calls
    in between; a call with no sweep behind it returns WVA_ESTATE"""
    from inferno_autoscaler_b200 import binding, distributed as D
    import torch
    img = wva.synth.make_system(40, 4, seed=41, n_types=2)
    R, B = 16, 160

    def run(with_blocking):
        ctx.upload(img)
        ctx.analyze(R, B, want_cube=True)
        if with_blocking:
            ctx.grid_blocking()
            ctx.grid_best_blocking()
            ctx.grid_blocking(download=False)
        cp, sp, n = ctx.grid_cube_device()
        torch.cuda.synchronize()
        dev = torch.device("cuda", ctx.device)
        cube = D.device_tensor(cp, n * 8, np.float32, dev).cpu().numpy().tobytes()
        status = D.device_tensor(sp, n, np.uint8, dev).cpu().numpy().tobytes()
        best = ctx.grid_fetch().tobytes()
        pairs, feas = ctx.pairs_fetch()
        if with_blocking:
            ctx.grid_best_blocking()
        acc, chosen = ctx.solve(unlimited=True)
        count, cost = ctx.allocate_by_type()
        return cube, status, best, pairs, feas.tobytes(), acc.tobytes(), chosen, count.tobytes(), cost.tobytes()

    a, b = run(False), run(True)
    for i in (0, 1, 2, 4, 5, 7, 8):
        assert a[i] == b[i], i
    assert a[3].equal_bits(b[3])[0] and a[6].equal_bits(b[6])[0]

    ctx.upload(img)
    for call in (ctx.grid_best_blocking, ctx.grid_blocking_counts, ctx.grid_blocking_device, ctx.grid_blocking):
        with pytest.raises(binding.WvaError) as e:
            call()
        assert e.value.code == wva.abi.ESTATE
    ctx.analyze_grid(R, B)
    ctx.grid_blocking()
    assert ctx.grid_blocking_device()[1] == img.S * img.A * R * B
    ctx.update_servers(3, img.take([3]))
    for call in (ctx.grid_best_blocking, ctx.grid_blocking_counts, ctx.grid_blocking_device, ctx.grid_blocking):
        with pytest.raises(binding.WvaError) as e:
            call()
        assert e.value.code == wva.abi.ESTATE


def test_plane_follows_the_last_successful_sweep(wva, oracle, ob, ctx):
    """a sweep call that fails leaves the previous sweep in place: the plane and its host array have that sweep's extent,
    whatever extents the failed call asked for"""
    from inferno_autoscaler_b200 import binding
    img = wva.synth.make_system(10, 3, seed=53, n_types=2)
    R, B = 8, 64
    ctx.upload(img)
    ctx.analyze_grid(R, B)
    before = ctx.grid_blocking()
    assert len(before) == img.S * img.A * R * B
    for r_max, b_max in ((2000, 1), (1, 9000), (2000, 9000)):
        with pytest.raises(binding.WvaError) as e:
            ctx.analyze_grid(r_max, b_max)
        assert e.value.code == wva.abi.EINVAL
        after = ctx.grid_blocking()
        assert len(after) == len(before) and after.tobytes() == before.tobytes()
    _, _, want = ob.grid_plane_blocking(img, R, B, threads=_threads(oracle))
    assert _mismatch(before, want) is None


def test_shard_slice(wva, oracle, ob, ctx):
    img = wva.synth.make_system(30, 3, seed=43, n_types=2)
    R, B = 8, 96
    ctx.upload(img)
    ctx.set_shard(11, 7)
    best, _, _ = ctx.analyze_grid(R, B)
    p = ctx.grid_blocking()
    assert len(p) == 7 * img.A * R * B
    _, _, want = ob.grid_plane_blocking(img, R, B, s0=11, s1=18, threads=_threads(oracle))
    assert _mismatch(p, want) is None
    wb = ctx.grid_best_blocking()
    has = best["acc"] >= 0
    widx = ((np.flatnonzero(has) * img.A + best["acc"][has]) * R + best["replicas"][has] - 1) * B + best["batch"][has] - 1
    assert _mismatch(wb[has], p[widx]) is None and np.isnan(wb[~has]).all()
    ctx.upload(img)


def _group_winners(wva, oracle, ob, n_dev):
    from inferno_autoscaler_b200 import binding
    img = wva.synth.make_system(24, 3, seed=47, n_types=2)
    R, B = 8, 64
    g = binding.Group(list(range(n_dev)))
    try:
        g.upload(img)
        g.analyze(R, B)
        best = g.grid_fetch()
        wb = g.grid_best_blocking()
    finally:
        g.close()
    has = best["acc"] >= 0
    assert has.any() and np.isnan(wb[~has]).all()
    _, st, want = ob.grid_candidates_blocking(img, np.flatnonzero(has), best["acc"][has], best["replicas"][has],
                                              best["batch"][has], threads=_threads(oracle))
    assert (st & 1).all() and _mismatch(wb[has], want) is None


def test_group_one_device(wva, oracle, ob):
    _group_winners(wva, oracle, ob, 1)


def test_group_two_devices(wva, oracle, ob):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _group_winners(wva, oracle, ob, 2)
