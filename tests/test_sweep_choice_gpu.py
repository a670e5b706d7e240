"""GPU: the sweep's per-server choice above 64 replicas and on the candidate values of sweep_choice_cases, against the
oracle bit for bit (a NaN on both sides counting as equal), in every set_certified_tails mode; the images' branches
are shown to be reached in test_sweep_choice_cpu.

  * every image in modes 1, 33, 0, 3, 5, 9 and 17: the whole cube, the status plane and the winners; the literal and
    deferred lists where the image is built to fill them; the scan's row plan at this device's SM count
  * Analyze (pair sizing beside the sweep) on R1 at r_max = 1024
  * a second, fused sweep of R2 (more than 4 096 deferred chains) byte-equal to the first
  * p_block of the winners of R1 and V, and the whole blocking plane of R1
  * on V: pair records, the unlimited solve and the per-type totals, which hold NaN, -Inf and negative costs
"""
import numpy as np
import pytest

from sweep_choice_cases import H100_SMS, IMAGES, MODES, image, oracle_sweep, row_plan
from test_profile_edges_gpu import cube_mismatch, literal_from_tables
from test_sweep_choice_cpu import SCAN_PLAN

pytestmark = pytest.mark.gpu


def _threads(oracle):
    return max(1, oracle.hardware_threads())


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _same_f32(got, want):
    return bool(((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all())


def _same_best(got, want):
    """winner records equal, a NaN float on both sides counting as equal (the device's NaN cost of a NaN-cost
    accelerator is the canonical 0x7fffffff, the host's keeps the input's payload)"""
    return (all(np.array_equal(got[f], want[f]) for f in ("acc", "replicas", "batch")) and
            all(_same_f32(got[f], want[f]) for f in ("cost", "value", "itl", "ttft", "rho")))


@pytest.mark.parametrize("mode", MODES)
def test_sweep_matches_oracle(wva, oracle, ctx, mode):
    """cube, status and winners of every image against the oracle; the lists the images fill"""
    sms = _num_sms()
    ctx.set_certified_tails(mode)
    try:
        for name in IMAGES:
            img, R, B = image(wva, name)
            w_best, w_cube, w_status = oracle_sweep(oracle, wva, name)
            ctx.upload(img)
            best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
            lists = ctx.grid_list_sizes()
            assert np.array_equal(status, w_status), (name, mode, int(np.flatnonzero(status != w_status)[0]))
            bad = cube_mismatch(cube, w_cube)
            assert bad is None, (name, mode, bad)
            assert _same_best(best, w_best), (name, mode)
            kernel, shape = row_plan(mode, img.S * img.A, R, B, sms)
            if kernel == "scan" and name in SCAN_PLAN:
                assert len(shape) > 1, (name, sms)
                if sms == H100_SMS:
                    assert shape == SCAN_PLAN[name], (name, shape)
            if name == "R2":                                   # the zero profile's candidates, all of them literal
                pred = literal_from_tables(img, R, B)
                assert pred == R * B and lists["literal"] >= pred, (mode, lists)
                if kernel == "scan":
                    assert lists["literal"] == pred and lists["deferred"] > 4096, (mode, lists)
            if name == "R1" and kernel == "scan":              # rows with lambda below 2^-100 or 0: exact chains
                assert lists["deferred"] > 0, (mode, lists)
            print("mode %d %s: %s %d blocks per pair, lists %s, %d winners (%d above 64)" %
                  (mode, name, kernel, len(shape), lists, int((best["acc"] >= 0).sum()),
                   int((best["replicas"] > 64).sum())))
    finally:
        ctx.set_certified_tails(1)


def test_analyze_r1(wva, oracle, ctx):
    """Analyze at r_max = 1024: the sweep's winners equal analyze_grid's and the oracle's, pair records the oracle's"""
    img, R, B = image(wva, "R1")
    ctx.upload(img)
    grid_best, _, _ = ctx.analyze_grid(R, B)
    ctx.analyze(R, B, want_cube=False)
    best = ctx.grid_fetch()
    assert best.tobytes() == grid_best.tobytes() == oracle_sweep(oracle, wva, "R1")[0].tobytes()
    got, gfe = ctx.pairs_fetch()
    want, wfe, _ = oracle.analyze_pairs(img, threads=_threads(oracle))
    assert np.array_equal(gfe, wfe)
    ok, field = got.equal_bits(want)
    assert ok, field


def test_fused_second_sweep_r2(wva, oracle, ctx):
    """R2 defers more than 4 096 chains: the next sweep on the context is fused, and byte-equal to the first"""
    img, R, B = image(wva, "R2")
    ctx.upload(img)
    ctx.grid_set_fused(False)
    try:
        first = ctx.analyze_grid(R, B, want_cube=True)
        assert ctx.grid_last_fused() == 0
        lists = ctx.grid_list_sizes()
        assert lists["deferred"] > 4096, lists
        ctx.grid_set_fused(True)
        second = ctx.analyze_grid(R, B, want_cube=True)
        assert ctx.grid_last_fused() == 1
        assert ctx.grid_list_sizes() == lists
    finally:
        ctx.grid_set_fused(True)
    for a, b in zip(first, second):
        assert a.tobytes() == b.tobytes()
    assert second[0].tobytes() == oracle_sweep(oracle, wva, "R2")[0].tobytes()


@pytest.mark.parametrize("name", ["R1", "V"])
def test_best_blocking(wva, oracle, ob, ctx, name):
    """p_block of each winner (NaN where there is none); on R1 the whole plane"""
    img, R, B = image(wva, name)
    ctx.upload(img)
    best, _, _ = ctx.analyze_grid(R, B)
    wb = ctx.grid_best_blocking()
    has = best["acc"] >= 0
    assert has.any() and (~has).any() and np.isnan(wb[~has]).all()
    srv = np.flatnonzero(has).astype(np.int32)
    _, st, want = ob.grid_candidates_blocking(img, srv, best["acc"][has], best["replicas"][has], best["batch"][has],
                                              threads=_threads(oracle))
    assert (st & 1).all() and _same_f32(wb[has], want)
    if name == "R1":
        p = ctx.grid_blocking()
        _, w_st, w_p = ob.grid_plane_blocking(img, R, B, threads=_threads(oracle))
        assert _same_f32(p, w_p)


def test_value_image_pairs_solve_totals(wva, oracle, ctx):
    """V: pair records, the unlimited solve's decisions and the per-type totals against the oracle"""
    img, _, _ = image(wva, "V")
    ctx.upload(img)
    got, gfe = ctx.analyze_pairs()
    want, wfe, _ = oracle.analyze_pairs(img, threads=_threads(oracle))
    assert np.array_equal(gfe, wfe)
    ok, field = got.equal_bits(want)
    assert ok, field
    acc, chosen = ctx.solve(unlimited=True)
    w_acc, w_chosen = oracle.solve(img, want, wfe, unlimited=True)
    assert np.array_equal(acc, w_acc)
    ok, field = chosen.equal_bits(w_chosen)
    assert ok, field
    cnt, cst = ctx.allocate_by_type()
    w_cnt, w_cst = oracle.allocate_by_type(img, w_acc, w_chosen)
    assert np.array_equal(cnt, w_cnt) and _same_f32(cst, w_cst)
    assert np.isnan(w_cst).any() and np.isneginf(w_cst).any() and (w_chosen.cost < 0).any()
    print("V totals: count %s, cost %s" % (w_cnt, w_cst))
