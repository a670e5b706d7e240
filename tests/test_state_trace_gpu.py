"""GPU: call-to-call state of a context -- incremental updates of the resident image, shards and tuning switches
between calls -- against fresh uploads and the oracle.

Every result of the traces of test_state_trace_cpu (trace A: 300 servers x 6 accelerators, trace B: 8190 servers x 16
across sweep slices) is compared with two references after each operation:
  - the witness: another context that uploads the expected image (kept in numpy by the test, not by the binding) with
    the same switches and shard, and makes the same calls; bit for bit;
  - the oracle, on the servers the operation touched plus a few random ones (servers are independent in the pair
    records, the sweep and its blocking plane), and on the whole image for the decisions.
The binding's host mirror of the image (Context.image) is checked against the expected image at every step, and the
validity matrix checks which results each mutation keeps and which it invalidates (WVA_ESTATE).
"""
import ctypes as C

import numpy as np
import pytest

from test_pairs_plane_cpu import choose, oracle_plane, rec_bytes, to_recs
from test_parity_full_gpu import prove_winners
from test_state_trace_cpu import (A_BATCHES, B_B, B_R, apply, copy_image, expected_bytes, touched, trace_a, trace_a_base,
                                  trace_b)

pytestmark = pytest.mark.gpu
A_R, A_B = 4, 64
B_BATCHES = [1, 64, 512]
RANKED = (2, 1, 0)


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


@pytest.fixture
def fresh(wva):
    """factory of new contexts (default switches, no hint), all closed when the test ends"""
    from inferno_autoscaler_b200 import binding
    made = []

    def make():
        made.append(binding.Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


def _th(oracle):
    return max(1, oracle.hardware_threads())


def _policies(wva):
    return (wva.abi.POLICY_PRIORITY_EXHAUSTIVE, wva.abi.POLICY_ROUND_ROBIN)


def shard_info(c):
    from inferno_autoscaler_b200 import binding
    f, n = C.c_int32(-1), C.c_int32(-1)
    assert binding.lib().wva_shard_info(c._h, C.byref(f), C.byref(n)) == 0
    return f.value, n.value


def f32_bytes(x):
    """float32 array as bytes, NaN payloads folded"""
    x = np.array(x, dtype=np.float32, copy=True)
    x[np.isnan(x)] = np.nan
    return x.tobytes()


def _device_bytes(ptr, n):
    import torch
    from inferno_autoscaler_b200 import distributed as D
    if n == 0:
        return b""
    torch.cuda.synchronize()
    return D.device_tensor(ptr, n, np.uint8, torch.device("cuda", 0)).cpu().numpy().tobytes()


def _alloc_bytes(wva, acc, chosen):
    return acc.tobytes() + rec_bytes(to_recs(wva, chosen, np.zeros(len(acc), np.uint8)))


def _try(fn):
    from inferno_autoscaler_b200 import binding
    try:
        return fn()
    except binding.WvaError as e:
        return ("error", e.code)


def _failed(r):
    return isinstance(r, tuple) and len(r) == 2 and isinstance(r[0], str)


def reads(wva, c):
    """every result the read calls return (or their error code); the order keeps each read from changing a later one"""
    def cube():
        cp, sp, n = c.grid_cube_device()
        return _device_bytes(cp, n * 32) + _device_bytes(sp, n)

    def blk_device():
        p, n = c.grid_blocking_device()
        return _device_bytes(p, n * 4)

    def size():
        n = C.c_size_t()
        from inferno_autoscaler_b200 import binding
        c._ck(binding.lib().wva_grid_blocking_size(c._h, C.byref(n)))
        return n.value

    out = {}
    out["solution_fetch"] = _try(lambda: _alloc_bytes(wva, *c.solution_fetch()))
    out["allocate_by_type"] = _try(lambda: b"".join(x.tobytes() for x in c.allocate_by_type()))
    out["grid_fetch"] = _try(lambda: c.grid_fetch().tobytes())
    out["grid_cube_device"] = _try(cube)
    out["grid_deferred"] = _try(lambda: c.grid_deferred(cap=1 << 20)[0].tobytes())
    out["grid_blocking_device"] = _try(blk_device)
    out["grid_blocking_counts"] = _try(c.grid_blocking_counts)
    out["grid_blocking_exact"] = _try(lambda: c.grid_blocking_exact(cap=1 << 20)[0].tobytes())
    out["grid_blocking_size"] = _try(size)
    out["grid_blocking"] = _try(lambda: f32_bytes(c.grid_blocking()))
    out["grid_best_blocking"] = _try(lambda: f32_bytes(c.grid_best_blocking()))
    out["pairs_fetch"] = _try(lambda: rec_bytes(to_recs(wva, *c.pairs_fetch())))
    out["shard"] = shard_info(c)
    return out


def run_calls(wva, c, R, B, batches, small):
    """every compute call on c's image and shard -> (bytes per result, raw results for the oracle).  Leaves pair records,
    unlimited decisions, the sweep and its blocking plane valid."""
    from inferno_autoscaler_b200 import binding
    out, raw = {}, {}
    p, fe = c.analyze_pairs()
    raw["pairs"] = (p, fe)
    out["pairs"] = rec_bytes(to_recs(wva, p, fe))
    c.analyze(R, B, want_cube=small)
    assert rec_bytes(to_recs(wva, *c.pairs_fetch())) == out["pairs"]
    raw["best"] = c.grid_fetch()
    out["best"] = raw["best"].tobytes()
    if small:
        cp, sp, n = c.grid_cube_device()
        out["cube"], out["status"] = _device_bytes(cp, n * 32), _device_bytes(sp, n)
        raw["plane"] = c.grid_blocking()
        out["plane"] = f32_bytes(raw["plane"])
    raw["best_blocking"] = c.grid_best_blocking()
    out["best_blocking"] = f32_bytes(raw["best_blocking"])
    plane, pbest = c.analyze_pairs_batches(batches, plane=small)
    raw["batches"] = (plane, pbest)
    out["batches"] = (rec_bytes(plane) if small else b"") + rec_bytes(pbest)
    first, count = shard_info(c)
    whole = (first, count) == (0, c.image.S)
    for ranked in RANKED if whole else ():
        for pol in _policies(wva) if ranked == 2 else _policies(wva)[:1] if small else ():
            c.solve_set_ranked(ranked)
            c.analyze_pairs(download=False)
            acc, ch = c.solve(unlimited=False, policy=pol)
            cnt, cost = c.allocate_by_type()
            raw[("limited", pol)] = (acc, ch, cnt, cost)
            out[("limited", ranked, pol)] = (_alloc_bytes(wva, acc, ch), cnt.tobytes() + cost.tobytes(), c.solve_greedy_path())
    c.solve_set_ranked(2)
    c.analyze_pairs(download=False)
    if not whole:
        with pytest.raises(binding.WvaError) as e:
            c.solve(unlimited=False)
        assert e.value.code == wva.abi.ESTATE
        c.analyze_pairs(download=False)
    acc, ch = c.solve(unlimited=True)
    raw["unlimited"] = (acc, ch)
    out["unlimited"] = _alloc_bytes(wva, acc, ch) + b"".join(x.tobytes() for x in c.allocate_by_type())
    return out, raw


def assert_mirror(wva, c, img, shard):
    """the binding's host image, the library's dimensions and shard equal the expected ones"""
    got = c.image
    assert (got.S, got.A, got.M, got.T) == (img.S, img.A, img.M, img.T)
    for name, _ in img.ALL_FIELDS:
        assert getattr(got, name).tobytes() == getattr(img, name).tobytes(), name
    assert c.dims() == (img.S, img.A, img.M, img.T)
    assert shard_info(c) == shard


def do_op(c, op):
    """op on the context under test; the error code it returned"""
    from inferno_autoscaler_b200 import binding
    try:
        if op.kind == "servers":
            c.update_servers(op.first, op.rows)
        elif op.kind == "models":
            c.update_models(op.first, op.rows)
        elif op.kind in ("remove", "removes"):
            for i in np.atleast_1d(op.index):
                c.remove_server(int(i))
        elif op.kind == "capacity":
            c.set_capacity(np.floor(c.image.type_capacity * op.scale).astype(np.int64))
        elif op.kind == "shard":
            c.set_shard(op.first, op.index)
    except binding.WvaError as e:
        return e.code
    return 0


def witness_calls(wva, w, img, shard, R, B, batches, small):
    w.upload(copy_image(img))
    if shard != (0, img.S):
        w.set_shard(*shard)
    return run_calls(wva, w, R, B, batches, small)[0]


def _same(got, want, what):
    bad = [k for k in want if got.get(k) != want[k]]
    assert not bad, "%s: %s differ" % (what, bad)


def _plane_rows(rel, A, R, B):
    """cube indices of every candidate of shard-relative servers rel"""
    per = A * R * B
    return (np.asarray(rel, dtype=np.int64)[:, None] * per + np.arange(per)).reshape(-1)


def oracle_checks(wva, oracle, ob, img, shard, rows, raw, R, B, batches, small):
    """the context's results on `rows` (absolute server indices inside the shard) and its decisions against the oracle"""
    th = _th(oracle)
    A = img.A
    first, count = shard
    rows = np.array(sorted(r for r in set(rows) if first <= r < first + count), dtype=np.int64)
    if len(rows):
        sub = img.take(rows)
        p, fe = raw["pairs"]
        want, wfe, _ = oracle.analyze_pairs(sub, threads=th)
        ix = (rows[:, None] * A + np.arange(A)).reshape(-1)
        assert rec_bytes(to_recs(wva, want, wfe)) == rec_bytes(to_recs(wva, p, fe)[ix])
        rel = rows - first
        best = raw["best"][rel]
        if small:
            o_best, _, _, _ = oracle.analyze_grid(sub, R, B, want_cube=False, threads=th)
            assert o_best.tobytes() == best.tobytes()
            _, _, o_p = ob.grid_plane_blocking(sub, R, B, threads=th)
            assert f32_bytes(o_p) == f32_bytes(raw["plane"][_plane_rows(rel, A, R, B)])
        else:
            prove_winners(wva, oracle, img, rows, best, R, B)
        has = best["acc"] >= 0
        wb = raw["best_blocking"][rel]
        assert np.isnan(wb[~has]).all()
        if has.any():
            _, st, o_wb = ob.grid_candidates_blocking(img, rows[has], best["acc"][has], best["replicas"][has],
                                                      best["batch"][has], threads=th)
            assert (st & 1).all() and f32_bytes(o_wb) == f32_bytes(wb[has])
        plane, pbest = raw["batches"]
        o_plane = oracle_plane(wva, oracle, sub, batches, threads=th)
        if small:
            pix = (rel[:, None] * A + np.arange(A)).reshape(-1)
            assert rec_bytes(o_plane) == rec_bytes(plane[pix])
        assert rec_bytes(choose(o_plane, A)) == rec_bytes(pbest[rel])
    if (first, count) != (0, img.S):
        return
    p, fe = raw["pairs"]
    acc, ch = raw["unlimited"]
    o_acc, o_ch = oracle.solve(img, p, fe, unlimited=True)
    assert acc.tobytes() == o_acc.tobytes() and ch.equal_bits(o_ch)[0]
    for pol in _policies(wva):
        if ("limited", pol) not in raw:
            continue
        acc, ch, cnt, cost = raw[("limited", pol)]
        o_acc, o_ch = oracle.solve(img, p, fe, unlimited=False, policy=pol)
        assert acc.tobytes() == o_acc.tobytes() and ch.equal_bits(o_ch)[0], pol
        o_cnt, o_cost = oracle.allocate_by_type(img, o_acc, o_ch)
        assert cnt.tobytes() == o_cnt.tobytes() and cost.tobytes() == o_cost.tobytes()


def replay(wva, oracle, ob, fresh, base, ops, R, B, batches, small, n_random=4, new_witness=(), on_checkpoint=None):
    import time
    c, w = fresh(), fresh()
    img, shard = copy_image(base), (0, base.S)
    c.upload(copy_image(base))
    prev = c.upload_bytes()
    run_calls(wva, c, R, B, batches, small)
    if on_checkpoint:
        on_checkpoint(-1, None, c)
    rng = np.random.default_rng(99)
    for k, op in enumerate(ops):
        unchanged = op.code != 0 or (op.kind in ("servers", "models") and op.count() == 0)
        before = reads(wva, c) if unchanged else None
        code = do_op(c, op)
        assert code == op.code, (op, code)
        new_img, new_shard = apply(wva, op, img, shard, None)
        assert c.upload_bytes() == expected_bytes(op, prev, img.A, img.T), op
        prev = c.upload_bytes()
        rows = touched(op, img, new_img)[:12]
        t0 = time.time()
        img, shard = new_img, new_shard
        assert_mirror(wva, c, img, shard)
        if unchanged:
            assert reads(wva, c) == before, op                      # nothing changed, nothing was invalidated
        got, raw = run_calls(wva, c, R, B, batches, small)
        wit = fresh() if k in new_witness else w
        _same(got, witness_calls(wva, wit, img, shard, R, B, batches, small), op)
        if img.S:
            rows = list(rows) + list(rng.choice(img.S, min(n_random, img.S), replace=False))
        t1 = time.time()
        oracle_checks(wva, oracle, ob, img, shard, rows, raw, R, B, batches, small)
        print("%-28s S=%-5d calls %.2f s, oracle %.2f s" % (op.tag, img.S, t1 - t0, time.time() - t1), flush=True)
        if on_checkpoint:
            on_checkpoint(k, op, c)
    return c


def test_trace_a(wva, oracle, ob, fresh):
    base, ops, _ = trace_a(wva)
    empty_at = [k for k, op in enumerate(ops) if op.tag == "remove_to_empty"][0]
    sizes = []

    def note(k, op, c):
        sizes.append(c.image.S)
        if op is not None and op.tag == "remove_to_empty":
            assert c.image.S == 0 and c.grid_fetch().size == 0
    replay(wva, oracle, ob, fresh, base, ops, A_R, A_B, A_BATCHES, small=True, new_witness=(0, empty_at + 1),
           on_checkpoint=note)
    assert 0 in sizes and max(sizes) == max(op.first + op.rows.S for op in ops if op.kind == "servers" and op.code == 0)
    print("trace A: %d operations, S went %s" % (len(ops), sizes))


def test_trace_b(wva, oracle, ob, fresh):
    base, ops, _ = trace_b(wva)
    seen = []

    def note(k, op, c):
        seen.append((c.image.S, c.grid_last_fused(), c.grid_list_sizes()["deferred"]))
    replay(wva, oracle, ob, fresh, base, ops, B_R, B_B, B_BATCHES, small=False, on_checkpoint=note)
    print("trace B: (S, last slice fused, deferred chains) of the first sweep and after each operation: %s" % seen)
    # the first sweep after the extension starts from the hint the 8190-server sweep left, and runs fused
    assert seen[0][0] == 8190 and seen[0][2] > 4096
    assert seen[1][:2] == (8200, 1)


# ---- which results a mutation keeps ------------------------------------------------------------------------------------

KEEP_ALL, INVALIDATE_ALL, CAPACITY, SHARD = "keep", "invalidate", "capacity", "shard"
MUTATIONS = {
    "servers_same_S": INVALIDATE_ALL, "servers_extend": INVALIDATE_ALL, "models": INVALIDATE_ALL,
    "models_extend": INVALIDATE_ALL, "remove": INVALIDATE_ALL, "set_capacity": CAPACITY, "set_shard": SHARD,
    "fail_priority": KEEP_ALL, "fail_ecapacity": KEEP_ALL, "fail_remove": KEEP_ALL, "zero_rows_servers": KEEP_ALL,
    "zero_rows_models": KEEP_ALL, "pstore_2": KEEP_ALL, "pstore_1": KEEP_ALL, "warp_max_0": KEEP_ALL,
    "certified_0": KEEP_ALL, "certified_33": KEEP_ALL, "tail_cap_64": KEEP_ALL, "fused_0": KEEP_ALL, "ranked_0": KEEP_ALL,
}
DECISIONS = ("solution_fetch", "allocate_by_type")
SWEEP = ("grid_fetch", "grid_cube_device", "grid_deferred", "grid_blocking_device", "grid_blocking_counts",
         "grid_blocking_exact", "grid_blocking_size", "grid_blocking", "grid_best_blocking")


def _mutate(wva, c, img, name):
    big = wva.synth.make_system(100, img.A, seed=102, n_types=img.T)
    big.srv_model[:] = 0
    if name == "servers_same_S":
        r = img.take([7]); r.srv_arrival_rpm[0] *= np.float32(2.0); c.update_servers(7, r)
    elif name == "servers_extend":
        c.update_servers(img.S, img.take([3, 4]))
    elif name in ("models", "models_extend"):
        c.update_models(1 if name == "models" else img.M, _one_model(wva, img, 2))
    elif name == "remove":
        c.remove_server(5)
    elif name == "set_capacity":
        c.set_capacity(img.type_capacity // 2)
    elif name == "set_shard":
        c.set_shard(1, img.S - 3)
    elif name.startswith("fail") or name.startswith("zero"):
        from inferno_autoscaler_b200 import binding
        bad = img.take([6]); bad.srv_priority[0] = 0
        if name == "zero_rows_servers":
            c.update_servers(4, img.take([]))
        elif name == "zero_rows_models":
            from test_state_trace_cpu import empty_rows
            c.update_models(2, empty_rows(wva, img))
        else:
            with pytest.raises(binding.WvaError) as e:
                if name == "fail_priority":
                    c.update_servers(6, bad)
                elif name == "fail_ecapacity":
                    c.update_servers(img.S, big)
                else:
                    c.remove_server(img.S)
            assert e.value.code == {"fail_ecapacity": wva.abi.ECAPACITY}.get(name, wva.abi.EINVAL)
    else:
        setter, value = name.rsplit("_", 1)
        {"pstore": c.pairs_set_pstore, "warp_max": c.pairs_set_warp_max, "certified": c.set_certified_tails,
         "tail_cap": c.grid_set_tail_cap, "fused": c.grid_set_fused, "ranked": c.solve_set_ranked}[setter](int(value))


def _one_model(wva, img, m):
    from test_state_trace_cpu import models_of
    return models_of(wva, img, [m])


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_validity_matrix(wva, fresh, name):
    img = wva.synth.make_system(40, 4, seed=101, n_types=2)
    img.srv_max_batch[9] = 3300                           # one pair table in HBM
    img.type_capacity[:] = [30, 30]
    c = fresh()
    c.upload(copy_image(img))
    c.set_shard(2, 34)
    c.analyze(A_R, A_B, want_cube=True)
    c.grid_blocking()
    c.grid_best_blocking()
    c.solve(unlimited=True)
    c.allocate_by_type()
    before = reads(wva, c)
    assert all(not (isinstance(v, tuple) and v and v[0] == "error") for v in before.values()), before
    decisions = c.solution_fetch()
    _mutate(wva, c, img, name)
    after = reads(wva, c)
    kind = MUTATIONS[name]
    estate = ("error", wva.abi.ESTATE)
    for key, v in after.items():
        if key == "shard":
            want = {INVALIDATE_ALL: (0, c.image.S), SHARD: (1, img.S - 3)}.get(kind, before["shard"])
        elif kind == KEEP_ALL or (kind == CAPACITY and key not in DECISIONS):
            want = before[key]
        else:
            want = estate
        assert v == want, (key, v if isinstance(v, tuple) else "bytes", want if isinstance(want, tuple) else "bytes")
    # the unlimited solve reads the pair records: the same decisions while they are kept
    got = _try(lambda: c.solve(unlimited=True))
    if kind in (KEEP_ALL, CAPACITY):
        assert _alloc_bytes(wva, *got) == _alloc_bytes(wva, *decisions)
    else:
        assert got == estate


def test_blocking_plane_and_records_follow_their_calls(wva, fresh):
    """the plane's device views need a wva_grid_blocking after every sweep; a limited solve consumes the pair records"""
    img = wva.synth.make_system(30, 3, seed=103, n_types=2)
    img.type_capacity[:] = [20, 20]
    c = fresh()
    c.upload(img)
    estate = ("error", wva.abi.ESTATE)
    for _ in range(2):
        c.analyze_grid_device(A_R, A_B, want_cube=False)
        assert _try(c.grid_blocking_device) == estate and _try(c.grid_blocking_counts) == estate
        assert _try(c.grid_blocking_exact) == estate
        c.grid_blocking()
        assert c.grid_blocking_device()[1] == 30 * 3 * A_R * A_B and not _failed(_try(c.grid_blocking_counts))
    c.analyze_pairs(download=False)
    c.solve(unlimited=False, policy=wva.abi.POLICY_PRIORITY_EXHAUSTIVE)
    assert _try(c.pairs_fetch) == estate and _try(lambda: c.solve(unlimited=True)) == estate
    assert not _failed(_try(c.solution_fetch))


# ---- switches between calls on one image ------------------------------------------------------------------------------

SWITCHES = [("pstore", 2, "pairs"), ("pstore", 0, "pairs"), ("pstore", 1, "pairs"), ("pstore", 3, "pairs"),
            ("pstore", 0, "pairs"), ("warp_max", 0, "pairs"), ("warp_max", 1 << 22, "pairs"),
            ("certified", 0, "sweep"), ("certified", 33, "sweep"), ("certified", 1, "sweep"),
            ("tail_cap", 64, "sweep"), ("tail_cap", -1, "sweep"), ("fused", 0, "sweep"), ("fused", 1, "sweep"),
            ("ranked", 1, "limited"), ("ranked", 0, "limited"), ("ranked", 2, "limited")]
DEFAULTS = {"pstore": 0, "warp_max": 1 << 22, "certified": 1, "tail_cap": -1, "fused": 1, "ranked": 2}


def _set(c, name, value):
    {"pstore": c.pairs_set_pstore, "warp_max": c.pairs_set_warp_max, "certified": c.set_certified_tails,
     "tail_cap": c.grid_set_tail_cap, "fused": c.grid_set_fused, "ranked": c.solve_set_ranked}[name](value)


def _call(wva, c, what):
    if what == "pairs":
        return rec_bytes(to_recs(wva, *c.analyze_pairs()))
    if what == "sweep":
        c.analyze(A_R, A_B, want_cube=True)
        cp, sp, n = c.grid_cube_device()
        return (c.grid_fetch().tobytes(), _device_bytes(cp, n * 32), _device_bytes(sp, n), f32_bytes(c.grid_blocking()),
                f32_bytes(c.grid_best_blocking()), rec_bytes(to_recs(wva, *c.pairs_fetch())))
    c.analyze_pairs(download=False)
    out = []
    for pol in _policies(wva):
        acc, ch = c.solve(unlimited=False, policy=pol)
        out.append((_alloc_bytes(wva, acc, ch), b"".join(x.tobytes() for x in c.allocate_by_type())))
        c.analyze_pairs(download=False)
    return out, c.solve_greedy_path()


def test_switches_between_calls(wva, fresh):
    """each switch changed on a context between two calls on the same image: the next call equals a witness that had the
    switch set before its upload (pstore 2 after a call made with the tables in shared memory re-plans the HBM tables)"""
    img = trace_a_base(wva)
    c, w = fresh(), fresh()
    c.upload(copy_image(img))
    first = _call(wva, c, "pairs")
    state = dict(DEFAULTS)
    for name, value, what in SWITCHES:
        _set(c, name, value)
        state[name] = value
        got = _call(wva, c, what)
        for k, v in state.items():
            _set(w, k, v)
        w.upload(copy_image(img))
        assert got == _call(wva, w, what), (name, value)
        if what == "pairs":
            assert got == first, (name, value)
