"""CPU: the fixtures of test_sweep_slices_gpu reach the sweep's size-driven branches, and the oracle's results they are
checked against.

grid_run (csrc/wva_b200.cu) chooses three branches by size alone, each of which re-plans or re-launches the sweep:

  slices      the sweep runs over slices of floor(2^30 / (A * b_max * 16)) servers, so that the published service-rate
              tables (16 B per pair and batch size) stay within 1 GB; every slice relaunches the sweep kernels with
              pair_base = first server of the slice * A and reuses the row, table, slot and list buffers
  fused hint  a slice launches all its kernels without a host round trip when the last slice swept on the context
              deferred more than 4096 chains; its list then has 2 * that count + 65536 slots, and a list that outgrows
              them redoes the slice stop and go
  literal     the materialised-p[] list starts at 65536 entries per call; more redo the slice with a larger list (and the
              blocking plane rescans with a larger literal list when it needs more than 65536 entries)

The fixtures, shared with the GPU tests:

  F1  servers [0, 17000) of config 5's image (100 000 servers x 16 accelerators), r = 64, b = 512: three slices
  F2  an image at A = 256 (the C-ABI's limit), b = 512, 1100 servers, r = 2: three slices, the last one partial, with the
      cube kept (9.2 GB on the device)
  F3  the zero profile family tiled 20 times: more than 2 x 65536 literal candidates.  A server's results do not depend
      on the other servers, so the expected cube, status bytes, winners and blocking plane are the family's tiled.
"""
import numpy as np
import pytest

from test_profile_edges_gpu import family, literal_from_tables

F = np.float32
TABLE_BYTES = 1 << 30                # the published rate tables of one slice (double2 per pair and batch size)
LIST_START = 1 << 16                 # first capacity of the sweep's literal list and of the plane's literal list

F1_COUNT, F1_R, F1_B = 17_000, 64, 512
F2_S, F2_A, F2_R, F2_B = 1100, 256, 2, 512
F3_TILES = 20


def slice_plan(ns, A, b_max):
    """[(first server, servers)] of the slices grid_run sweeps a shard of ns servers in"""
    per = max(1, min(ns, TABLE_BYTES // (A * b_max * 16)))
    return [(s, min(per, ns - s)) for s in range(0, ns, per)]


_IMAGES = {}


def config5_image(wva):
    """config 5's image, generated as bench.py --config 5 generates it"""
    if "c5" not in _IMAGES:
        c = wva.synth.CONFIGS[5]
        _IMAGES["c5"] = wva.synth.make_system(c["S"], c["A"], seed=5, n_types=c["T"])
    return _IMAGES["c5"]


def f2_image(wva):
    """F2: 1100 servers x 256 accelerators (8 types) from the synthetic generator"""
    if "f2" not in _IMAGES:
        _IMAGES["f2"] = wva.synth.make_system(F2_S, F2_A, seed=256, n_types=8)
    return _IMAGES["f2"]


def f3_image(wva, tiles=F3_TILES):
    """F3: the zero profile family, its servers repeated `tiles` times -> (image, r_max, b_max)"""
    img, R, B = family(wva, "zero")
    return img.take(np.tile(np.arange(img.S), tiles)), R, B


def tile_results(best, cube, status, tiles):
    return np.tile(best, tiles), np.tile(cube, tiles), np.tile(status, tiles)


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


def test_slice_rule_f1_f2(wva):
    """F1 and F2 are swept in at least three slices, the last one partial; config 5 on one GPU takes 13"""
    c5 = wva.synth.CONFIGS[5]
    assert slice_plan(c5["S"], c5["A"], c5["b_max"])[0] == (0, 8192) and len(slice_plan(c5["S"], c5["A"], c5["b_max"])) == 13
    f1 = slice_plan(F1_COUNT, c5["A"], F1_B)
    assert f1 == [(0, 8192), (8192, 8192), (16384, 616)]
    f2 = slice_plan(F2_S, F2_A, F2_B)
    assert f2 == [(0, 512), (512, 512), (1024, 76)]
    for plan in (f1, f2):
        assert len(plan) >= 3 and plan[-1][1] < plan[0][1]
    # one slice: the shards the GPU tests compare against, and F3
    assert len(slice_plan(616, c5["A"], F1_B)) == 1
    img, R, B = f3_image(wva)
    assert len(slice_plan(img.S, img.A, B)) == 1
    assert F2_A == 256 and f2_image(wva).A == F2_A              # the C-ABI's largest A (WVA_GRID_MAX_A)


def test_f3_literal_prediction(wva):
    """every F3 candidate behind a bad table entry goes to the literal list: 20 x the zero family's count, more than
    twice the list's first capacity"""
    img, R, B = family(wva, "zero")
    one = literal_from_tables(img, R, B)
    tiled, _, _ = f3_image(wva)
    pred = literal_from_tables(tiled, R, B)
    assert pred == F3_TILES * one
    assert pred > 2 * LIST_START, pred


def test_tiled_oracle_equals_tiled_results(wva, oracle, ob):
    """on 3 tiles the oracle's sweep and blocking plane of the tiled image are the family's results tiled"""
    th = oracle.hardware_threads()
    img, R, B = family(wva, "zero")
    tiled, _, _ = f3_image(wva, tiles=3)
    want = tile_results(*oracle.analyze_grid(img, R, B, want_cube=True, threads=th)[:3], 3)
    got = oracle.analyze_grid(tiled, R, B, want_cube=True, threads=th)[:3]
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    _, st1, p1 = ob.grid_plane_blocking(img, R, B, threads=th)
    _, st3, p3 = ob.grid_plane_blocking(tiled, R, B, threads=th)
    assert np.array_equal(st3, np.tile(st1, 3))
    assert np.tile(p1, 3).tobytes() == p3.tobytes()


def test_oracle_terminates_on_f3(wva, oracle, ob):
    """the oracle sweeps all of F3 and its blocking plane (the GPU tests use the tiled family results)"""
    th = oracle.hardware_threads()
    tiled, R, B = f3_image(wva)
    best, cube, status, _ = oracle.analyze_grid(tiled, R, B, want_cube=True, threads=th)
    assert len(status) == tiled.S * tiled.A * R * B
    ok = int(((status & 0xfe) == 0).sum())
    assert ok > 0 and (best["acc"] >= 0).any()
    _, st, p = ob.grid_plane_blocking(tiled, R, B, threads=th)
    assert np.array_equal(st, status)
    assert int((~np.isnan(p)).sum()) == ok
