"""GPU: sweeps that span several server slices, the fused flow's list hint, and the list retries, against the oracle.

The fixtures F1, F2, F3 and the slice rule are in test_sweep_slices_cpu, which checks that they reach their branches.
Every test here creates its own contexts, so that each one starts with a known hint (the deferred-list length of the
last slice swept on a context), and asserts that its branch was taken: the number of slices, wva_grid_last_fused, the
literal count, and plane lists that grew.

  H   hint primer: config 3 servers [250, 750), swept stop and go, defers ~6 600 chains: the next sweep on that context
      is fused
"""
import numpy as np
import pytest

from test_parity_full_gpu import _decode, prove_winners
from test_profile_edges_gpu import cube_mismatch, family, literal_from_tables
from test_sweep_slices_cpu import (F1_B, F1_COUNT, F1_R, F2_B, F2_R, LIST_START, F3_TILES, config5_image, f2_image,
                                   f3_image, slice_plan)

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


@pytest.fixture
def fresh(wva):
    """factory of new contexts (no hint, lists at their first capacities), all closed when the test ends"""
    from inferno_autoscaler_b200 import binding
    made = []

    def make():
        made.append(binding.Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


def _threads(oracle):
    return max(1, oracle.hardware_threads())


def _sweep(c, R, B):
    """winners-only sweep of c's shard -> (winners, list sizes, counters)"""
    c.analyze_grid_device(R, B, want_cube=False)
    return c.grid_fetch(), c.grid_list_sizes(), c.grid_counters()


def prime_hint(wva, c):
    """H on context c: returns the hint it leaves"""
    img, cfg = wva.synth.baseline_config(3)
    c.grid_set_fused(False)
    c.upload(img)
    c.set_shard(250, 500)
    _sweep(c, cfg["r_max"], cfg["b_max"])
    assert c.grid_last_fused() == 0
    hint = c.grid_list_sizes()["deferred"]
    assert hint > 4096, hint
    return hint


def _device_cube_at(c, ids):
    """metrics and status bytes of the cube left on c's device, at shard-relative candidate ids"""
    import torch
    from inferno_autoscaler_b200 import distributed as D
    cp, sp, n = c.grid_cube_device()
    torch.cuda.synchronize()
    dev = torch.device("cuda", c.device)
    ix = torch.as_tensor(np.asarray(ids, dtype=np.int64), device=dev)
    cube = D.device_tensor(cp, n * 8, np.float32, dev).view(n, 8)
    status = D.device_tensor(sp, n, np.uint8, dev)
    m = cube.index_select(0, ix).cpu().numpy().copy().view(np.dtype(cube_dtype())).reshape(-1)
    return m, status.index_select(0, ix).cpu().numpy(), n


def _device_status(c):
    import torch
    from inferno_autoscaler_b200 import distributed as D
    _, sp, n = c.grid_cube_device()
    torch.cuda.synchronize()
    return D.device_tensor(sp, n, np.uint8, torch.device("cuda", c.device)).cpu().numpy()


def cube_dtype():
    from inferno_autoscaler_b200 import abi
    return abi.METRICS_DTYPE


def _check_ids(oracle, img, first, ids, m, st, R, B):
    """cube entries at shard-relative ids (shard starting at server `first`) against the oracle, bit for bit"""
    s, a, r, b = _decode(np.asarray(ids, dtype=np.int64), img.A, R, B)
    o_m, o_st = oracle.grid_candidates(img, s + first, a, r, b, threads=_threads(oracle))
    assert np.array_equal(o_st, st)
    bad = cube_mismatch(m, o_m)
    assert bad is None, (int(ids[bad // 8]), bad % 8)


def _boundary_servers(plan, count, width=4):
    """servers within `width` of each slice boundary (and of the shard's ends)"""
    edges = [s for s, _ in plan] + [count]
    out = set()
    for e in edges:
        out.update(range(max(0, e - width), min(count, e + width + 1)))
    return np.array(sorted(out), dtype=np.int64)


def _pairs_match_oracle(wva, oracle, img, got, gfe, servers):
    """pair records of `servers` (runs of consecutive indices) against the oracle's Server.Calculate"""
    A = img.A
    for run in np.split(servers, np.flatnonzero(np.diff(servers) != 1) + 1):
        s0, n = int(run[0]), len(run)
        want, wfe, _ = oracle.analyze_pairs(img.shard(s0, n), threads=_threads(oracle))
        part = wva.abi.AllocArrays(n * A)
        for name, _ in wva.abi.ALLOC_FIELDS:
            getattr(part, name)[:] = getattr(got, name)[s0 * A:(s0 + n) * A]
        assert np.array_equal(gfe[s0 * A:(s0 + n) * A], wfe), s0
        ok, field = part.equal_bits(want)
        assert ok, (s0, field)


# ---- 1. multi-slice winners (F1) -------------------------------------------------------------------------------------

def test_multi_slice_winners(wva, oracle, ob, fresh):
    img = config5_image(wva)
    A, R, B = img.A, F1_R, F1_B
    plan = slice_plan(F1_COUNT, A, B)
    assert len(plan) == 3
    c = fresh()
    c.upload(img)
    c.set_shard(0, F1_COUNT)
    best, lists, counters = _sweep(c, R, B)
    assert c.grid_last_fused() == 1                # slices 2 and 3 inherit slice 1's hint
    deferred, n_def = c.grid_deferred(cap=1 << 24)
    # the same slices as shards of their own, stop and go, on a second context
    ref = fresh()
    ref.grid_set_fused(False)
    ref.upload(img)
    parts = []
    for s0, n in plan:
        ref.set_shard(s0, n)
        parts.append(_sweep(ref, R, B))
    last_ids, n_last = ref.grid_deferred(cap=1 << 24)
    # several slices ran: the deferred list fetched is the last slice's alone
    assert n_def == len(deferred) < lists["deferred"]
    assert n_def == n_last == parts[-1][1]["deferred"] > 0
    assert np.array_equal(np.sort(deferred), np.sort(last_ids) + np.uint64(plan[-1][0] * A * R * B))
    assert sum(p[1]["deferred"] for p in parts) == lists["deferred"]
    assert sum(p[1]["literal"] for p in parts) == lists["literal"]
    want = np.concatenate([p[0] for p in parts])
    assert best.tobytes() == want.tobytes()
    ok = sum(p[2]["candidates_ok"] for p in parts)
    alg = sum(p[2]["steps_algorithmic"] for p in parts)
    assert counters["candidates_ok"] == ok and counters["steps_algorithmic"] == alg

    # a repeated reconcile: slice 1 starts from slice 3's hint, its list outgrows 2 * hint + 65536 slots and it is redone
    assert parts[0][1]["deferred"] > 2 * parts[-1][1]["deferred"] + LIST_START
    best2, lists2, counters2 = _sweep(c, R, B)
    assert c.grid_last_fused() == 1
    assert best2.tobytes() == best.tobytes() and lists2 == lists
    assert counters2["candidates_ok"] == ok and counters2["steps_algorithmic"] == alg
    assert counters2["steps_executed"] > counters["steps_executed"]          # slice 1 ran twice

    # the oracle: winners at the slice boundaries and at random, their blocking probability, the last slice's list
    rng = np.random.default_rng(17)
    srv = np.union1d(_boundary_servers(plan, F1_COUNT), rng.choice(F1_COUNT, 250, replace=False))
    prove_winners(wva, oracle, img, srv, best[srv], R, B)
    wb = c.grid_best_blocking()
    has = srv[best["acc"][srv] >= 0]
    assert len(has) > 100 and np.isnan(wb[srv[best["acc"][srv] < 0]]).all()
    _, st, p = ob.grid_candidates_blocking(img, has, best["acc"][has], best["replicas"][has], best["batch"][has],
                                           threads=_threads(oracle))
    assert (st & 1).all() and wb[has].view(np.uint32).tobytes() == p.view(np.uint32).tobytes()
    s0, n = plan[-1]
    ref.set_shard(s0, n)
    ref.analyze_grid_device(R, B, want_cube=True)
    assert ref.grid_list_sizes()["deferred"] == n_last
    m, st, _ = _device_cube_at(ref, np.sort(last_ids).astype(np.int64))
    _check_ids(oracle, img, s0, np.sort(last_ids), m, st, R, B)

    # Analyze (pair sizing beside the sweep): the same winners; the boundary servers' pair records
    c.analyze(R, B, want_cube=False)
    assert c.grid_fetch().tobytes() == best.tobytes()
    got, gfe = c.pairs_fetch()
    _pairs_match_oracle(wva, oracle, img, got, gfe, _boundary_servers(plan, F1_COUNT))
    print("F1: %d slices, deferred %d (last slice %d), literal %d, candidates_ok %d; %d winners proven" %
          (len(plan), lists["deferred"], n_def, lists["literal"], ok, len(has)))


# ---- 2. multi-slice cube (F2) ----------------------------------------------------------------------------------------

def test_multi_slice_cube(wva, oracle, fresh):
    img = f2_image(wva)
    A, R, B = img.A, F2_R, F2_B
    plan = slice_plan(img.S, A, B)
    assert len(plan) >= 3 and plan[-1][1] < plan[0][1]
    c = fresh()
    c.upload(img)
    c.analyze_grid_device(R, B, want_cube=True)
    best = c.grid_fetch()
    lists, counters = c.grid_list_sizes(), c.grid_counters()
    deferred, n_def = c.grid_deferred(cap=1 << 24)
    assert n_def == len(deferred) < lists["deferred"]
    status = _device_status(c)
    # 10^6 cube entries, half of them on the servers at the slice boundaries; every id of the last slice's list
    ncand = img.S * A * R * B
    per_srv = A * R * B
    rng = np.random.default_rng(256)
    near = _boundary_servers(plan, img.S)
    ids = np.concatenate([rng.choice(near, 500_000) * per_srv + rng.integers(0, per_srv, 500_000),
                          rng.integers(0, ncand, 500_000), deferred.astype(np.int64)])
    ids = np.unique(ids)
    assert len(ids) > 900_000
    m, st, n = _device_cube_at(c, ids)
    assert n == ncand and np.array_equal(st, status[ids])
    _check_ids(oracle, img, 0, ids, m, st, R, B)
    # winners: the boundary servers', and those at accelerators >= 128 (the key's upper accelerator bits)
    hi = np.flatnonzero(best["acc"] >= 128)
    assert len(hi) > 0
    srv = np.union1d(near, hi[:20])
    prove_winners(wva, oracle, img, srv, best[srv], R, B)
    # the same slices as shards of their own: status bytes, winners, lists, counters
    parts, ok, alg = [], 0, 0
    for s0, k in plan:
        c.set_shard(s0, k)
        c.analyze_grid_device(R, B, want_cube=True)
        parts.append((c.grid_fetch(), _device_status(c), c.grid_list_sizes()["deferred"]))
        ok += c.grid_counters()["candidates_ok"]
        alg += c.grid_counters()["steps_algorithmic"]
    assert np.concatenate([p[1] for p in parts]).tobytes() == status.tobytes()
    assert np.concatenate([p[0] for p in parts]).tobytes() == best.tobytes()
    assert sum(p[2] for p in parts) == lists["deferred"] and parts[-1][2] == n_def
    assert counters["candidates_ok"] == ok and counters["steps_algorithmic"] == alg
    print("F2: %d slices, %d candidates, deferred %d (last slice %d); %d cube entries and %d winners (%d at acc >= 128) "
          "checked" % (len(plan), ncand, lists["deferred"], n_def, len(ids), int((best["acc"][srv] >= 0).sum()), len(hi)))


# ---- 3. the fused flow's list outgrows its slots ---------------------------------------------------------------------

OUTGROWN_FIRST, OUTGROWN_COUNT = 40_000, 4_000


def test_fused_list_outgrown(wva, oracle, fresh):
    img = config5_image(wva)
    A, R, B = img.A, F1_R, F1_B
    assert len(slice_plan(OUTGROWN_COUNT, A, B)) == 1
    c = fresh()
    hint = prime_hint(wva, c)
    c.grid_set_fused(True)
    c.upload(img)
    c.set_shard(OUTGROWN_FIRST, OUTGROWN_COUNT)
    best, lists, counters = _sweep(c, R, B)
    assert lists["deferred"] > 2 * hint + LIST_START, (lists, hint)
    assert c.grid_last_fused() == 0                                       # the fused attempt was thrown away
    deferred, _ = c.grid_deferred(cap=1 << 24)
    ref = fresh()
    ref.grid_set_fused(False)
    ref.upload(img)
    ref.set_shard(OUTGROWN_FIRST, OUTGROWN_COUNT)
    r_best, r_lists, r_counters = _sweep(ref, R, B)
    r_deferred, _ = ref.grid_deferred(cap=1 << 24)
    assert best.tobytes() == r_best.tobytes() and lists == r_lists
    assert np.array_equal(np.sort(deferred), np.sort(r_deferred))
    assert counters["candidates_ok"] == r_counters["candidates_ok"]
    assert counters["steps_algorithmic"] == r_counters["steps_algorithmic"]
    # the oracle: 200 winners, and deferred candidates of the shard's first 256 servers (swept with the cube kept)
    rng = np.random.default_rng(40)
    srv = np.sort(rng.choice(OUTGROWN_COUNT, 200, replace=False))
    prove_winners(wva, oracle, img, OUTGROWN_FIRST + srv, best[srv], R, B)
    per_srv = A * R * B
    head = np.sort(deferred[deferred < 256 * per_srv]).astype(np.int64)
    head = head[rng.choice(len(head), min(len(head), 3000), replace=False)]
    assert len(head) > 1000
    ref.set_shard(OUTGROWN_FIRST, 256)
    ref.analyze_grid_device(R, B, want_cube=True)
    m, st, _ = _device_cube_at(ref, head)
    _check_ids(oracle, img, OUTGROWN_FIRST, head, m, st, R, B)
    print("outgrown list: hint %d, deferred %d, candidates_ok %d" % (hint, lists["deferred"], counters["candidates_ok"]))


# ---- 4. a large hint, then a short or empty list ---------------------------------------------------------------------

def _large_hint(wva, c):
    """the hint a stop-and-go sweep of test 3's shard leaves (~100 000)"""
    img = config5_image(wva)
    c.grid_set_fused(False)
    c.upload(img)
    c.set_shard(OUTGROWN_FIRST, OUTGROWN_COUNT)
    _sweep(c, F1_R, F1_B)
    hint = c.grid_list_sizes()["deferred"]
    assert hint > 2 * 4096
    c.grid_set_fused(True)
    return hint


def _whole_sweep_vs_oracle(oracle, c, img, R, B):
    best, cube, status = c.analyze_grid(R, B, want_cube=True)
    assert c.grid_last_fused() == 1
    o_best, o_cube, o_status, _ = oracle.analyze_grid(img, R, B, want_cube=True, threads=_threads(oracle))
    assert np.array_equal(status, o_status)
    assert cube.tobytes() == o_cube.tobytes()
    assert best.tobytes() == o_best.tobytes()
    assert c.grid_counters()["candidates_ok"] == int(((o_status & 0xfe) == 0).sum())
    return c.grid_list_sizes()


def test_large_hint_short_list(wva, oracle, fresh):
    c = fresh()
    img2, cfg = wva.synth.baseline_config(2)
    R, B = cfg["r_max"], cfg["b_max"]
    # every server without load: an empty deferred list
    idle = img2.shard(0, img2.S)
    idle.srv_arrival_rpm[:] = 0.0
    hint = _large_hint(wva, c)
    c.upload(idle)
    lists = _whole_sweep_vs_oracle(oracle, c, idle, R, B)
    assert lists["deferred"] == 0
    # config 2: a few deferred chains
    hint = _large_hint(wva, c)
    c.upload(img2)
    lists = _whole_sweep_vs_oracle(oracle, c, img2, R, B)
    assert lists["deferred"] < hint
    print("large hint %d: config 2 deferred %d, literal %d" % (hint, lists["deferred"], lists["literal"]))


# ---- 5. the literal list outgrows its first capacity (F3) ------------------------------------------------------------

_F3 = {}


def _f3_expected(wva, oracle, ob):
    """the zero family's oracle sweep and blocking plane, tiled like F3"""
    if not _F3:
        th = _threads(oracle)
        img, R, B = family(wva, "zero")
        o_best, o_cube, o_status, _ = oracle.analyze_grid(img, R, B, want_cube=True, threads=th)
        _, _, p = ob.grid_plane_blocking(img, R, B, threads=th)
        _F3.update(best=np.tile(o_best, F3_TILES), cube=np.tile(o_cube, F3_TILES), status=np.tile(o_status, F3_TILES),
                   plane=np.tile(p, F3_TILES), ok=F3_TILES * int(((o_status & 0xfe) == 0).sum()))
        # p_block of each server's winner
        has = o_best["acc"] >= 0
        wb = np.full(img.S, np.nan, dtype=F)
        srv = np.flatnonzero(has)
        wb[has] = p[((srv * img.A + o_best["acc"][has]) * R + o_best["replicas"][has] - 1) * B + o_best["batch"][has] - 1]
        _F3["best_blocking"] = np.tile(wb, F3_TILES)
    return _F3


def _same_f32(got, want):
    return bool(((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all())


@pytest.mark.parametrize("flow", ["stop_and_go", "fused", "fused_off"])
def test_literal_redo(wva, oracle, ob, fresh, flow):
    img, R, B = f3_image(wva)
    pred = literal_from_tables(img, R, B)
    assert pred > 2 * LIST_START
    want = _f3_expected(wva, oracle, ob)
    c = fresh()
    if flow != "stop_and_go":
        prime_hint(wva, c)
        c.grid_set_fused(flow == "fused")
    c.upload(img)
    best, cube, status = c.analyze_grid(R, B, want_cube=True)
    assert c.grid_last_fused() == (1 if flow == "fused" else 0)
    lists = c.grid_list_sizes()
    assert lists["literal"] == pred
    assert np.array_equal(status, want["status"])
    assert cube_mismatch(cube, want["cube"]) is None
    assert best.tobytes() == want["best"].tobytes()
    assert c.grid_counters()["candidates_ok"] == want["ok"]
    # the blocking plane, whose literal list grows past its first 65536 entries on this context
    p = c.grid_blocking()
    listed, n_listed = c.grid_blocking_exact(cap=1 << 22)
    assert n_listed >= pred > LIST_START
    assert _same_f32(p, want["plane"])
    assert _same_f32(c.grid_best_blocking(), want["best_blocking"])
    print("F3 %s: literal %d, plane listed %d, candidates_ok %d" % (flow, lists["literal"], n_listed, want["ok"]))
