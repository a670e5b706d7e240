"""GPU: the library's own NCCL paths -- wva_comm_* (a communicator per context) and wva_group_* with several members --
on ONE device, through the loopback NCCL stand-in (nccl_loopback/).

  * the stand-in itself, loaded privately in this process: rank-order all-gathers of 0 .. 2^20 bytes on 1 - 8 ranks,
    stream order on both sides of the call, a count mismatch refused on every rank, a rendezvous timeout;
  * a communicator per context (tests/nccl_loopback_driver.py, one host thread per rank): shards, pair rows, sweep
    winners, unlimited and limited decisions and the global totals against the oracle on the images and plans of
    tests/rank_emulation.py, the all-gathers each call issues, shards that leave a gap or overlap (refused on every
    rank), and the shard that uploads and row-changing updates leave behind;
  * groups of 2 - 5 members on device 0: every assembled host output against the oracle or one plain context, the
    errors of the assembled scenario call, and a tuning switch on one member.

The multi-rank runs happen in a subprocess that never imports torch: torch brings its own libnccl.so.2, which the
library would otherwise bind.
"""
import ctypes as C
import functools
import json
import os
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rank_emulation as re_  # noqa: E402
from test_pairs_plane_cpu import rec_bytes, to_recs  # noqa: E402

pytestmark = pytest.mark.gpu

abi = re_.abi
HERE = os.path.dirname(os.path.abspath(__file__))
DRIVER = os.path.join(HERE, "nccl_loopback_driver.py")
NONE, PEXH, PRR, RR = abi.POLICY_NONE, abi.POLICY_PRIORITY_EXHAUSTIVE, abi.POLICY_PRIORITY_ROUND_ROBIN, abi.POLICY_ROUND_ROBIN
PATH = {2: 3, 1: 2, 0: 1}                       # wva_solve_set_ranked setting -> path at A <= 32: scan, ranked queue, heap
SUCCESS, SYSTEM_ERROR, INVALID_ARGUMENT, INVALID_USAGE = 0, 2, 4, 5
RUN_TIMEOUT = 900

_FULL = [(p, d, 2) for p in (NONE, PEXH, PRR, RR) for d in (False, True)] + [(PEXH, False, 1), (RR, True, 0)]
COMM_CASES = {
    ("P1", 2): [(PEXH, False, 2)],
    ("P1", 3): _FULL,
    ("P1", 5): [(RR, True, 2)],
    ("P2", 2): [(NONE, False, 2), (PRR, True, 1)],
    ("P2", 5): [(RR, True, 2), (PEXH, False, 0)],
    ("P3", 8): [(NONE, False, 2), (PEXH, True, 0)],
}
GROUP_LIMITED = [(p, d, 2) for p in (NONE, PEXH, PRR, RR) for d in (False, True)]
GROUP_CASES = [("P2", 2), ("P2", 5), ("P1", 3), ("W", 3)]
BATCHES = [1, 64, 3000, 3100]                   # crosses the 3 072-entry shared-memory slice of the batch list


def chunk_bytes(S, A, G):
    """the packed pair-row chunk one rank contributes to the limited solve's all-gather"""
    return (16 + -(-S // G) * A * 45 + 15) // 16 * 16


# ---- the driver --------------------------------------------------------------------------------------------------
def image_arrays(prefix, img):
    out = {prefix + ".dims": np.array([img.S, img.A, img.M, img.T], dtype=np.int64)}
    for name, _ in img.ALL_FIELDS:
        out[prefix + "." + name] = getattr(img, name)
    return out


def drive(case, cfg, img=None, **arrays):
    """run one case of the driver in a torch-free subprocess; its outputs as a dict"""
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.npz"), os.path.join(d, "out.npz")
        z = dict(arrays, cfg=np.array(json.dumps(cfg)))
        if img is not None:
            z.update(image_arrays("img", img))
        np.savez(src, **z)
        p = subprocess.Popen([sys.executable, DRIVER, case, src, dst], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        try:
            log, _ = p.communicate(timeout=RUN_TIMEOUT)
        except subprocess.TimeoutExpired:
            p.kill()
            p.communicate()
            raise
        assert p.returncode == 0, log.decode(errors="replace")[-4000:]
        with np.load(dst, allow_pickle=False) as f:
            return dict(f)


def allocs(out, key, n):
    a = abi.AllocArrays(n)
    for name, _ in abi.ALLOC_FIELDS:
        getattr(a, name)[:] = out[key + "." + name]
    return a


def totals_bytes(count, cost):
    return np.asarray(count, dtype=np.int64).tobytes() + np.asarray(cost, dtype=np.float32).tobytes()


def same_floats(got, want):
    got, want = np.asarray(got, dtype=np.float32), np.asarray(want, dtype=np.float32)
    return bool(((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all())


# ---- a. the stand-in itself --------------------------------------------------------------------------------------
class UniqueId(C.Structure):
    _fields_ = [("internal", C.c_char * 128)]


@pytest.fixture(scope="module")
def loopback():
    """the stand-in loaded privately (RTLD_LOCAL, by path), so that torch's libnccl.so.2 in this process is not touched"""
    import nccl_loopback
    L = C.CDLL(nccl_loopback.build(), mode=os.RTLD_LOCAL)
    vp = C.c_void_p
    L.ncclGetUniqueId.argtypes = [C.POINTER(UniqueId)]
    L.ncclCommInitRank.argtypes = [C.POINTER(vp), C.c_int, UniqueId, C.c_int]
    L.ncclCommDestroy.argtypes = [vp]
    L.ncclAllGather.argtypes = [vp, vp, C.c_size_t, C.c_int, vp, vp]
    L.loopback_counters.argtypes = [vp, C.c_int, C.POINTER(C.c_uint64)]
    return L


def lb_counters(L, comm):
    v = (C.c_uint64 * 7)()
    assert L.loopback_counters(comm, 0, v) == SUCCESS
    return list(v)


def on_threads(n, fn):
    res, err = [None] * n, [None] * n

    def body(r):
        try:
            res[r] = fn(r)
        except BaseException as e:      # noqa: B902 - re-raised below
            err[r] = e
    th = [threading.Thread(target=body, args=(r,)) for r in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in err:
        if e is not None:
            raise e
    return res


def init_comms(L, G, ranks=None):
    uid = UniqueId()
    assert L.ncclGetUniqueId(C.byref(uid)) == SUCCESS

    def init(r):
        c = C.c_void_p()
        return L.ncclCommInitRank(C.byref(c), G, uid, r), c
    return on_threads(len(ranks) if ranks is not None else G, lambda i: init(ranks[i] if ranks is not None else i))


@pytest.mark.parametrize("G", [1, 2, 3, 8])
def test_loopback_allgather(loopback, G):
    import torch
    L = loopback
    res = init_comms(L, G)
    assert [rc for rc, _ in res] == [SUCCESS] * G
    comms = [c for _, c in res]
    groups0 = lb_counters(L, comms[0])[5:]
    streams = [torch.cuda.Stream(device=0) for _ in range(G)]
    gen = torch.Generator(device="cpu").manual_seed(G)
    try:
        for count in (0, 1, 13, 1 << 20):
            want = [torch.randint(0, 256, (count,), dtype=torch.uint8, generator=gen) for _ in range(G)]
            send = [torch.zeros(max(count, 1), dtype=torch.uint8, device="cuda:0") for _ in range(G)]
            recv = [torch.full((max(G * count, 1),), 0x5A, dtype=torch.uint8, device="cuda:0") for _ in range(G)]
            src = [w.to("cuda:0") for w in want]
            torch.cuda.synchronize()

            def rank(r):
                with torch.cuda.stream(streams[r]):
                    torch.cuda._sleep(2_000_000)                     # the fill lands late: the gather must wait for it
                    send[r][:count].copy_(src[r])
                    rc = L.ncclAllGather(send[r].data_ptr(), recv[r].data_ptr(), count, 0, comms[r], streams[r].cuda_stream)
                    send[r].fill_(0xEE)                              # after the call: must not reach any peer
                return rc
            assert on_threads(G, rank) == [SUCCESS] * G
            torch.cuda.synchronize()
            whole = torch.cat(want).numpy().tobytes()
            for r in range(G):
                assert recv[r][:G * count].cpu().numpy().tobytes() == whole, (count, r)
                k = lb_counters(L, comms[r])
                assert k[1] == count
            # a datatype other than ncclInt8 is refused before anything is enqueued
            assert L.ncclAllGather(send[0].data_ptr(), recv[0].data_ptr(), count, 7, comms[0], streams[0].cuda_stream) == INVALID_ARGUMENT
        assert [lb_counters(L, c)[0] for c in comms] == [4] * G
        assert lb_counters(L, comms[0])[5:] == groups0 == [0, 0]
    finally:
        for c in comms:
            assert L.ncclCommDestroy(c) == SUCCESS


def test_loopback_count_mismatch(loopback):
    import torch
    L, G = loopback, 3
    comms = [c for rc, c in init_comms(L, G) if rc == SUCCESS]
    assert len(comms) == G
    send = [torch.arange(8, dtype=torch.uint8, device="cuda:0") + 16 * r for r in range(G)]
    recv = [torch.zeros(8 * G, dtype=torch.uint8, device="cuda:0") for _ in range(G)]
    s = torch.cuda.current_stream(0).cuda_stream
    try:
        counts = [4, 4, 5]
        rcs = on_threads(G, lambda r: L.ncclAllGather(send[r].data_ptr(), recv[r].data_ptr(), counts[r], 0, comms[r], s))
        assert rcs == [INVALID_USAGE] * G
        torch.cuda.synchronize()
        assert all(int(x.abs().sum()) == 0 for x in recv)                      # nothing moved
        # the communicator goes on working
        assert on_threads(G, lambda r: L.ncclAllGather(send[r].data_ptr(), recv[r].data_ptr(), 8, 0, comms[r], s)) == [SUCCESS] * G
        torch.cuda.synchronize()
        whole = torch.cat(send).cpu().numpy().tobytes()
        assert all(x.cpu().numpy().tobytes() == whole for x in recv)
    finally:
        for c in comms:
            L.ncclCommDestroy(c)


def test_loopback_rendezvous_timeout(loopback):
    """two of three ranks arrive: both get ncclSystemError after the timeout, no device work involved"""
    import time
    old = os.environ.get("NCCL_LOOPBACK_TIMEOUT_S")
    os.environ["NCCL_LOOPBACK_TIMEOUT_S"] = "1"
    try:
        t0 = time.monotonic()
        res = init_comms(loopback, 3, ranks=[0, 2])
        dt = time.monotonic() - t0
    finally:
        if old is None:
            del os.environ["NCCL_LOOPBACK_TIMEOUT_S"]
        else:
            os.environ["NCCL_LOOPBACK_TIMEOUT_S"] = old
    assert [rc for rc, _ in res] == [SYSTEM_ERROR] * 2
    assert all(not c.value for _, c in res)
    assert 0.9 < dt < 30


# ---- b. a communicator per context -------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _winners(name):
    import oracle
    ref = re_.reference(name)
    r_max, b_max = re_.SWEEP[name]
    return oracle.analyze_grid(ref.img, r_max, b_max, want_cube=False, threads=oracle.hardware_threads())[0]


def check_limited(oracle, out, key, img, pairs, feasible, G, policy, delayed, ranked, gathers=1):
    """every rank: the oracle's decisions, the global totals, one pair all-gather (`gathers`) and one totals all-gather"""
    what = (key, policy, delayed, ranked)
    w_acc, w_chosen = oracle.solve(img, pairs, feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
    w_count, w_cost = re_.expected_totals(oracle, img, w_acc, w_chosen, G)
    for r in range(G):
        p = "%s.r%d" % (key, r)
        assert int(out[p + ".path"]) == PATH[ranked], what + (r,)
        assert np.array_equal(out[p + ".acc"], w_acc), what + (r, np.nonzero(out[p + ".acc"] != w_acc)[0][:8])
        ok, field = allocs(out, p + ".chosen", img.S).equal_bits(w_chosen)
        assert ok, what + (r, field)
        assert totals_bytes(out[p + ".count"], out[p + ".cost"]) == totals_bytes(w_count, w_cost), what + (r,)
        k = out[p + ".counters"]                  # before, after the solve, after the refused solve, after the totals
        assert k[1][0] - k[0][0] == gathers and k[1][1] == chunk_bytes(img.S, img.A, G), what + (r, k)
        assert int(out[p + ".again"]) == abi.ESTATE and (k[2] == k[1]).all(), what + (r, k)
        assert k[3][0] - k[2][0] == 1 and k[3][1] == 12 * img.T, what + (r, k)


@pytest.mark.parametrize("name,G", list(COMM_CASES), ids=["%s-G%d" % c for c in COMM_CASES])
def test_comm_ranks(oracle, name, G):
    ref = re_.reference(name)
    img, A = ref.img, ref.img.A
    r_max, b_max = re_.SWEEP[name]
    limited = COMM_CASES[(name, G)]
    out = drive("comm", dict(G=G, sweep=[r_max, b_max], limited=limited), img)
    plan = re_.plan(img.S, G)
    o_best = _winners(name)
    w_count, w_cost = re_.expected_totals(oracle, img, ref.acc, ref.chosen, G)
    for r, (f, n) in enumerate(plan):
        assert tuple(out["r%d.info" % r]) == (r, G)
        assert tuple(out["r%d.shard" % r]) == (f, n)
        p = "unl.r%d" % r
        m = slice(f * A, (f + n) * A)
        assert np.array_equal(out[p + ".feasible"][m], ref.feasible[m]), (r, f, n)
        ok, field = allocs(out, p + ".pairs", img.S * A).equal_bits(ref.pairs, mask=m)
        assert ok, (r, f, n, field)
        assert out[p + ".best"].tobytes() == o_best[f:f + n].tobytes(), (r, f, n)
        assert np.array_equal(out[p + ".acc"][f:f + n], ref.acc[f:f + n]), (r, f, n)
        ok, field = allocs(out, p + ".chosen", img.S).equal_bits(ref.chosen, mask=slice(f, f + n))
        assert ok, (r, f, n, field)
        assert totals_bytes(out[p + ".count"], out[p + ".cost"]) == totals_bytes(w_count, w_cost), (r, out[p + ".count"], w_count)
        k = out[p + ".counters"]   # before the analysis; after analyze, fetches, unlimited solve, batches, loads; after totals
        assert (k[1] == k[0]).all(), (r, k)
        assert k[2][0] - k[1][0] == 1 and k[2][1] == 12 * img.T, (r, k)
    for i, (policy, delayed, ranked) in enumerate(limited):
        check_limited(oracle, out, "lim%d" % i, img, ref.pairs, ref.feasible, G, policy, delayed, ranked)
    for r in range(G):
        assert out["r%d.destroyed" % r][2] == 1, r            # one ncclCommDestroy per rank, on either way out
    created, destroyed, g_start, g_end = out["final"][3:]
    assert (created, destroyed, g_start, g_end) == (G, G, 0, 0)


def bad_plans(S, G):
    """shards that leave one server out and shards that overlap by one, each no larger than ceil(S / G)"""
    plan = [list(x) for x in re_.plan(S, G)]
    cap = -(-S // G)
    gap = [list(x) for x in plan]
    r = next(r for r, (f, n) in enumerate(gap) if n > 0)
    gap[r][1] -= 1
    over = [list(x) for x in plan]
    r = next(r for r, (f, n) in enumerate(over) if n < cap and 0 < f + n < S)
    over[r][1] += 1
    for p in (gap, over):
        assert all(n <= cap for _, n in p)
    return [gap, over]


@pytest.mark.parametrize("name,G", [("P2", 2), ("P2", 5), ("P3", 8)], ids=["P2-G2", "P2-G5", "P3-G8"])
def test_shards_that_do_not_tile(oracle, name, G):
    """a gap or an overlap between the ranks' shards fails the limited solve on every rank (after its one all-gather);
    wva_comm_shard, wva_analyze_pairs and the next limited solve then match the oracle"""
    ref = re_.reference(name)
    img = ref.img
    plans = bad_plans(img.S, G)
    out = drive("comm", dict(G=G, sweep=list(re_.SWEEP[name]), bad_shards=plans), img)
    for i in range(len(plans)):
        for r in range(G):
            k = out["bad%d.r%d.counters" % (i, r)]
            assert int(out["bad%d.r%d.rc" % (i, r)]) == abi.EINVAL, (plans[i], r)
            assert k[1][0] - k[0][0] == 1, (plans[i], r, k)
        check_limited(oracle, out, "bad%d.repair" % i, img, ref.pairs, ref.feasible, G, PEXH, False, 2)


def updated(img, update, rows=None, first=None, index=None):
    """the image after the update (what the library's rows and the binding's image become)"""
    out = img.shard(0, img.S)
    if update == "update_servers":
        for name, _ in abi.SRV_FIELDS:
            a = getattr(out, name)
            newS = max(img.S, first + rows.S)
            if newS > img.S:
                a = np.concatenate([a, np.zeros(newS - img.S, dtype=a.dtype)])
            a[first:first + rows.S] = getattr(rows, name)
            setattr(out, name, a)
        out.S = max(img.S, first + rows.S)
    elif update == "update_models":
        for name, _ in abi.PERF_FIELDS:
            getattr(out, name)[first * img.A:(first + rows.M) * img.A] = getattr(rows, name)
    elif update == "remove_server":
        for name, _ in abi.SRV_FIELDS:
            a = getattr(out, name)
            a[index] = a[img.S - 1]
            setattr(out, name, a[:img.S - 1].copy())
        out.S -= 1
    return out


def _model_rows(img, m):
    """new perf rows for model m: its profile with alpha and gamma scaled (the pair records change)"""
    rows = type(img)(0, img.A, 1, img.T)
    for name, _ in abi.PERF_FIELDS:
        setattr(rows, name, getattr(img, name)[m * img.A:(m + 1) * img.A].copy())
    rows.perf_alpha = (rows.perf_alpha * np.float32(1.25)).astype(np.float32)
    rows.perf_gamma = (rows.perf_gamma * np.float32(0.75)).astype(np.float32)
    return rows


UPDATES = ["upload", "update_servers", "update_models", "remove_server"]


@pytest.mark.parametrize("update", UPDATES)
def test_shard_after_upload_and_updates(oracle, update):
    """with a communicator attached, an upload (no wva_comm_shard after it) and every row-changing update leave the
    rank's communicator range of the new S: pair rows are sized there only and the totals are the global ones"""
    name, G = "P2", 5
    ref = re_.reference(name)
    img = ref.img
    cfg = dict(G=G, sweep=list(re_.SWEEP[name]), no_comm_shard=True)
    arrays = {}
    new = img
    if update == "update_servers":
        rows = img.take([3, 17])
        cfg.update(update=update, first=img.S)
        arrays = image_arrays("rows", rows)
        new = updated(img, update, rows=rows, first=img.S)
    elif update == "update_models":
        m = int(img.srv_model[0])
        rows = _model_rows(img, m)
        cfg.update(update=update, first=m)
        arrays = image_arrays("rows", rows)
        new = updated(img, update, rows=rows, first=m)
    elif update == "remove_server":
        cfg.update(update=update, index=7)
        new = updated(img, update, index=7)
    out = drive("comm", cfg, img, **arrays)
    plan = re_.plan(img.S, G)
    for r in range(G):
        assert tuple(out["r%d.upload_shard" % r]) == plan[r], r
    if update != "upload":
        for r, sh in enumerate(re_.plan(new.S, G)):
            assert tuple(out["r%d.update_shard" % r]) == sh, r
            assert tuple(out["r%d.update_dims" % r])[:2] == (new.S, new.A)
    pairs, feas, _ = oracle.analyze_pairs(new)
    acc, chosen = oracle.solve(new, pairs, feas, unlimited=True)
    w_count, w_cost = re_.expected_totals(oracle, new, acc, chosen, G)
    A = new.A
    for r, (f, n) in enumerate(re_.plan(new.S, G)):
        p = "unl.r%d" % r
        m = slice(f * A, (f + n) * A)
        got = allocs(out, p + ".pairs", new.S * A)
        ok, field = got.equal_bits(pairs, mask=m)
        assert ok and np.array_equal(out[p + ".feasible"][m], feas[m]), (r, field)
        outside = np.ones(new.S * A, dtype=bool)
        outside[m] = False
        assert not out[p + ".feasible"][outside].any() and not got.num_replicas[outside].any(), r   # sized there only
        assert np.array_equal(out[p + ".acc"][f:f + n], acc[f:f + n]), r
        assert totals_bytes(out[p + ".count"], out[p + ".cost"]) == totals_bytes(w_count, w_cost), \
            (r, out[p + ".count"], w_count)


# ---- c. groups on one device -------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def group_reference(name):
    if name != "W":
        return re_.reference(name), re_.SWEEP[name]
    import oracle
    synth = re_._wva.synth
    img = synth.make_system(24, 4, seed=81, n_types=2, max_pair_batch=512, tps_fraction=0.2, keep_fraction=0.2)
    assert 0 < (img.srv_max_batch > 0).sum() < img.S                 # servers with a batch-size override
    pairs, feasible, _ = oracle.analyze_pairs(img)
    acc, chosen = oracle.solve(img, pairs, feasible, unlimited=True)
    synth.set_capacity_from_demand(img, acc, chosen.num_replicas, fraction=re_.CAPACITY_FRACTION)
    return re_.Reference(img, pairs, feasible, acc, chosen), (4, 32)


def loads_columns(img):
    """five scenarios (n_l differs from A on every group image, so a row offset in units of A shows)"""
    base = img.srv_arrival_rpm.astype(np.float32)
    cols = [np.float32(f) * base for f in (0.0, 1.0, 3.0, 0.25)] + [np.full(img.S, -1.0, dtype=np.float32)]
    return np.stack(cols, axis=1).astype(np.float32)


@pytest.mark.parametrize("name,G", GROUP_CASES, ids=["%s-G%d" % c for c in GROUP_CASES])
def test_group_members_on_one_device(wva, oracle, name, G):
    import oracle_blocking
    oracle_blocking.build()
    ref, (r_max, b_max) = group_reference(name)
    img, A, S = ref.img, ref.img.A, ref.img.S
    rpm = loads_columns(img)
    out = drive("group", dict(G=G, sweep=[r_max, b_max], batches=BATCHES, limited=GROUP_LIMITED), img, rpm=rpm)
    assert [tuple(x) for x in out["shards"]] == re_.plan(S, G)
    assert list(out["shards.create"][5:]) == [0, 0]
    w_recs = to_recs(wva, ref.pairs, ref.feasible)

    ok, field = allocs(out, "p0.pairs", S * A).equal_bits(ref.pairs)
    assert ok and np.array_equal(out["p0.feasible"], ref.feasible), field
    o_best = oracle.analyze_grid(img, r_max, b_max, want_cube=False, threads=oracle.hardware_threads())[0]
    has = o_best["acc"] >= 0
    assert has.any()
    _, st, w_pb = oracle_blocking.grid_candidates_blocking(img, np.flatnonzero(has), o_best["acc"][has],
                                                           o_best["replicas"][has], o_best["batch"][has],
                                                           threads=oracle.hardware_threads())
    assert (st & 1).all()
    w_block = np.full(S, np.nan, dtype=np.float32)
    w_block[has] = w_pb
    w_acc_u, w_chosen_u = ref.acc, ref.chosen
    w_tot_u = re_.expected_totals(oracle, img, w_acc_u, w_chosen_u, G)
    w_lim = []
    for policy, delayed, _ in GROUP_LIMITED:
        acc, chosen = oracle.solve(img, ref.pairs, ref.feasible, unlimited=False, delayed_best_effort=delayed, policy=policy)
        w_lim.append((acc, chosen, re_.expected_totals(oracle, img, acc, chosen, G)))

    for key in ("base", "tails"):
        for cube in (0, 1):
            k = "%s.cube%d" % (key, cube)
            ok, field = allocs(out, k + ".pairs", S * A).equal_bits(ref.pairs)
            assert ok and np.array_equal(out[k + ".feasible"], ref.feasible), (k, field)
            assert out[k + ".best"].tobytes() == o_best.tobytes(), k
            assert same_floats(out[k + ".p_block"], w_block), k
        # the assembled planes equal one context over the whole image; the scenario at the uploaded rates equals the
        # oracle's pair records
        for what in ("batches", "batches_best", "loads", "loads_best"):
            assert rec_bytes(out["%s.%s" % (key, what)]) == rec_bytes(out["single." + what]), (key, what)
        assert rec_bytes(out[key + ".loads"][:, 1, :].reshape(-1)) == rec_bytes(w_recs), key
        assert np.array_equal(out[key + ".unl.acc"], w_acc_u), key
        assert allocs(out, key + ".unl.chosen", S).equal_bits(w_chosen_u)[0], key
        assert totals_bytes(out[key + ".unl.count"], out[key + ".unl.cost"]) == totals_bytes(*w_tot_u), key
        for i, ((policy, delayed, _), (acc, chosen, tot)) in enumerate(zip(GROUP_LIMITED, w_lim)):
            k = "%s.lim%d" % (key, i)
            assert np.array_equal(out[k + ".acc"], acc), (k, policy, delayed)
            ok, field = allocs(out, k + ".chosen", S).equal_bits(chosen)
            assert ok, (k, policy, delayed, field)
            assert totals_bytes(out[k + ".count"], out[k + ".cost"]) == totals_bytes(*tot), (k, policy, delayed)
    # errors of the assembled scenario call
    assert list(out["err.rc"]) == [abi.EINVAL, abi.EINVAL]
    assert list(out["err.untouched"]) == [0xA5] * 4                  # neither plane nor best written
    msg_nan, msg_zero = (str(x) for x in out["err.msg"])
    assert "NaN" in msg_nan and "device 0" in msg_zero, (msg_nan, msg_zero)
    assert rec_bytes(out["after.loads"]) == rec_bytes(out["base.loads"])
    assert rec_bytes(out["after.loads_best"]) == rec_bytes(out["base.loads_best"])
    assert list(out["final"][5:]) == [0, 0]                          # the library never groups its collectives
    assert out["closed"][4] - out["shards.create"][4] == G           # every member's communicator destroyed
