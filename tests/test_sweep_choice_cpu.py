"""CPU: the images of sweep_choice_cases reach the branches of the sweep's per-server choice that the GPU tests compare
with the oracle: winners above 64 replicas, at block starts and at r_max; -0, -Inf, NaN, +Inf, negative and subnormal
candidate values; ties between accelerators.  Also the host's row plans, restated, and the key order, restated over
the oracle's whole cube."""
import numpy as np
import pytest

from sweep_choice_cases import (FIXTURE, H100_SMS, IMAGES, MODES, R1_MIN_REP, VALUE_FIXTURES, F, chunk_starts, image,
                                lambda_row, oracle_sweep, rate_row, restated_best, row_plan)
from test_parity_full_gpu import prove_winners

# the scan kernels' blocks at 132 SMs (rows per block of a pair)
SCAN_PLAN = {"R1": [64] * 16, "R2": [56, 44], "R3": [8] * 128, "R4a": [8] * 8 + [1], "R4b": [40, 25]}


def _pairs(img):
    return img.S * img.A


def test_row_plans_at_h100(wva):
    """the scan plan of every R image at 132 SMs is the one the images are built for; k_grid, k_grid_wrow and
    k_grid_rows plans of the same shards"""
    for name, shape in SCAN_PLAN.items():
        img, R, B = image(wva, name)
        for mode in (1, 33):
            assert row_plan(mode, _pairs(img), R, B, H100_SMS) == ("scan", shape), (name, mode)
    img, R, B = image(wva, "R1")
    assert row_plan(0, 36, R, B, H100_SMS) == ("grid", [18] * 56 + [16])        # 2112 blocks wanted: 57 per pair
    assert row_plan(3, 36, R, B, H100_SMS) == ("grid", [18] * 56 + [16])
    assert row_plan(9, 36, R, B, H100_SMS) == ("wrow", [8] * 128)
    assert row_plan(5, 36, R, B, H100_SMS) == ("rows", [1024])
    assert row_plan(17, 36, R, B, H100_SMS) == ("rows", [1024])                 # 36 864 rows >= 32 768
    assert row_plan(17, 1, 1024, 512, H100_SMS) == ("grid", [1] * 1024)         # R3: one row per block
    assert row_plan(9, 1, 65, 64, H100_SMS) == ("wrow", [8] * 8 + [1])          # R4a
    assert row_plan(0, 600, 100, 48, H100_SMS) == ("grid", [25] * 4)            # R2
    assert row_plan(0, 600, 65, 64, H100_SMS) == ("grid", [17] * 3 + [14])      # R4b
    # fewer SMs: fewer blocks per pair, never fewer than r_max / 64 in the scan
    assert row_plan(1, 36, 1024, 64, 8) == ("scan", [64] * 16)
    assert row_plan(1, 1, 1024, 512, 8) == ("scan", [32] * 32)
    assert chunk_starts([40, 25]) == [1, 41]


def _winners(oracle, wva, name):
    return oracle_sweep(oracle, wva, name)[0]


def test_r_images_reach_their_rows(wva, oracle):
    """winners above 64, at block starts on both sides of block boundaries, at r_max, and none where
    min_replicas > r_max; the rows whose lambda is below 2^-100 and whose rate rounds to 0"""
    best = _winners(oracle, wva, "R1")
    img, R, B = image(wva, "R1")
    r1 = [int(x) if a >= 0 else None for a, x in zip(best["acc"], best["replicas"])]
    assert r1[:8] == [1, 1, 1, 64, 65, 129, R, None]                  # min_replicas -1, 0, 1, 64, 65, 129, r_max, +1
    assert list(img.srv_min_replicas[:8]) == R1_MIN_REP
    starts = chunk_starts(SCAN_PLAN["R1"])
    assert {65, 129} <= set(starts) and 64 + 1 in starts
    assert r1[8] == R and img.acc_cost[best["acc"][8]] < 0           # negative cost: the largest feasible r
    tiny = img.srv_arrival_rpm[9]
    assert float(lambda_row(tiny, 100)) >= 2.0 ** -100 > float(lambda_row(tiny, 101))
    assert r1[9] == 129                                              # decided on a row whose lambda is below 2^-100
    zero = img.srv_arrival_rpm[10]
    assert rate_row(zero, 199) > 0 and all(rate_row(zero, r) == 0 for r in range(200, R + 1))
    assert 64 < r1[11] < R and r1[11] not in starts                  # loaded: inside a middle block
    assert best["batch"][11] > 1
    # R2, R4b: both sides of their one boundary, r_max, none above it
    for name, edge in (("R2", 56), ("R4b", 40)):
        img, R, B = image(wva, name)
        best = _winners(oracle, wva, name)
        got = set(best["replicas"][best["acc"] >= 0].tolist())
        assert {edge, edge + 1, R} <= got, (name, sorted(got))
        assert edge + 1 in chunk_starts(SCAN_PLAN[name])
        assert (best["acc"][img.srv_min_replicas > R] < 0).all()
    img, R, B = image(wva, "R2")
    lam = np.array([lambda_row(img.srv_arrival_rpm[s], 1) for s in range(img.S)])
    assert (lam < F(2.0 ** -100)).sum() == 3
    # R3: the last block's first row; R4a: the one-row block
    assert int(_winners(oracle, wva, "R3")["replicas"][0]) == 1017 == chunk_starts(SCAN_PLAN["R3"])[-1]
    assert int(_winners(oracle, wva, "R4a")["replicas"][0]) == 65 == chunk_starts(SCAN_PLAN["R4a"])[-1]


def _row_values(oracle, wva):
    img, R, _ = image(wva, "V")
    return oracle.grid_row_values(img, R)


def _bits(x):
    return np.asarray(x, dtype=F).view(np.uint32)


def test_value_fixtures_reach_their_branches(wva, oracle):
    """each V server's winner is the one its fixture is built for, and the row values show why"""
    img, R, B = image(wva, "V")
    best = _winners(oracle, wva, "V")
    vals = _row_values(oracle, wva)
    for s, (name, accs, cur, rep, cost, mn, keep, want) in enumerate(VALUE_FIXTURES):
        got = None if best["acc"][s] < 0 else (int(best["acc"][s]), int(best["replicas"][s]))
        assert got == want, (name, got)
    v = lambda name: vals[FIXTURE[name]]
    r = np.arange(1, R + 1)
    # -0: the raw penalty of the current (-0) accelerator is -0 off the current row; the sweep's value is +0, which
    # ties with +0 on accelerator 0: the lower index wins
    raw = (F(-0.0) * r.astype(F)) - F(0.0)
    assert np.signbit(raw).all()
    for name in ("negzero_tie", "negzero_tie_hi", "negzero_cur", "negzero_cur_lo", "negzero_tie_min65"):
        assert (_bits(v(name)[1]) == 0).all(), name
    assert (_bits(v("negzero_tie")[0]) == 0).all()
    # -Inf off the current row, NaN elsewhere; the NaN fixtures: NaN everywhere but the current row
    x = v("neginf")
    assert np.isneginf(np.delete(x[2], 119)).all() and x[2][119] == 0 and np.isnan(x[3]).all()
    for name in ("nan_cur", "nan_cur_blocked", "nan_cur_above", "nan_cur_lo", "negnan_cur", "nan_cur_zero_rep"):
        s = FIXTURE[name]
        cur, rep = int(img.srv_cur_acc[s]), int(img.srv_cur_replicas[s])
        finite = np.argwhere(~np.isnan(vals[s]))
        assert [tuple(t) for t in finite] == ([(cur, rep - 1)] if 1 <= rep <= R else []), name
        assert best["acc"][s] < 0 or (best["acc"][s], best["replicas"][s]) == (cur, rep), name
    assert np.isnan(v("nan_acc")[9]).all() and np.isnan(np.delete(v("inf_minus_inf")[8], 139)).all()
    # +Inf and overflow: 3e38 at r = 1 is finite, the largest float32's penalty overflows, every r >= 2 overflows
    assert np.isposinf(v("inf_acc")[8]).all()
    x = v("huge")
    assert np.isfinite(x[6][0]) and np.isposinf(x[7][0]) and np.isposinf(x[6:8, 1:]).all()
    # negative: decreasing in r; subnormal: increasing, above +0
    assert (np.diff(v("neg")[4]) < 0).all()
    sub = v("subnormal")[5]
    assert (sub > 0).all() and (sub < F(1e-38)).all() and (np.diff(sub) > 0).all()
    assert np.isneginf(v("neginf_acc")[10]).all()
    # identical accelerators and perf_acc_count <= 0: equal rows, the lower index wins
    for name in ("identical", "acc_count_le0"):
        assert np.array_equal(_bits(v(name)[2]), _bits(v(name)[3])), name
    # keepAccelerator with an unknown current accelerator: no candidate at all
    assert np.isnan(v("keep_unknown")).all()
    assert (best["replicas"][best["acc"] >= 0] > 64).sum() >= 8


@pytest.mark.parametrize("name", IMAGES)
def test_key_order_restated(wva, oracle, name):
    """(canonical value, a, r, b), NaN never chosen, over the oracle's whole cube gives the oracle's winners"""
    img, R, B = image(wva, name)
    best, cube, status = oracle_sweep(oracle, wva, name)
    want = restated_best(img, R, B, oracle.grid_row_values(img, R), cube, status)
    assert want.tobytes() == best.tobytes(), name


def test_prove_winners_on_value_image(wva, oracle):
    """prove_winners accepts the oracle's own winners of V and refuses a tied winner moved to the higher index"""
    img, R, B = image(wva, "V")
    best = _winners(oracle, wva, "V")
    srv = np.arange(img.S)
    prove_winners(wva, oracle, img, srv, best, R, B)
    for name in ("identical", "acc_count_le0", "identical_min129"):
        moved = best.copy()
        s = FIXTURE[name]
        assert moved["acc"][s] == 2
        moved["acc"][s] = 3
        with pytest.raises(AssertionError):
            prove_winners(wva, oracle, img, srv, moved, R, B)


def test_modes_cover_every_kernel(wva):
    """the seven modes the GPU tests run reach the scan kernels, k_grid, k_grid_rows and k_grid_wrow on these images"""
    kinds = {row_plan(m, _pairs(image(wva, n)[0]), image(wva, n)[1], image(wva, n)[2], H100_SMS)[0]
             for m in MODES for n in IMAGES}
    assert kinds == {"scan", "grid", "rows", "wrow"}
