"""Torch-free subprocess that runs the library's own multi-rank paths on ONE GPU through the loopback NCCL stand-in.

    python nccl_loopback_driver.py CASE IN.npz OUT.npz

The stand-in (nccl_loopback/libnccl_loopback.so, SONAME libnccl.so.2) is loaded with RTLD_GLOBAL before anything else,
so the library's dlopen("libnccl.so.2") binds to it.  The process must never map another libnccl: importing torch would
bring its own, and the library would then use whichever it found first.  The driver checks /proc/self/maps before and
after the case and exits with status 3 and a message when anything but the stand-in is mapped.

IN.npz holds the image's arrays ("img.<field>", "img.dims"), any further images ("<name>.<field>"), other arrays the case
needs, and "cfg", a JSON string.  OUT.npz receives every output and counter; the oracle side stays with the caller
(tests/test_nccl_loopback_gpu.py).  Cases:
  unique_id  wva_comm_unique_id only (needs no device);
  comm       G contexts on device 0, one host thread each, attached by wva_comm_init;
  group      one wva_group over [0] * G, plus one plain context over the whole image.
"""
import ctypes as C
import json
import os
import sys
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
STAND_IN = os.path.realpath(os.path.join(ROOT, "nccl_loopback", "libnccl_loopback.so"))
WRONG_NCCL = 3

_stand_in = C.CDLL(STAND_IN, mode=C.RTLD_GLOBAL)


def check_maps():
    """exit unless the stand-in is the only libnccl in this process"""
    with open("/proc/self/maps") as f:
        paths = {ln.split(None, 5)[5].strip() for ln in f if len(ln.split(None, 5)) == 6}
    nccl = {os.path.realpath(p) for p in paths if os.path.basename(p).startswith("libnccl")}
    if nccl != {STAND_IN}:
        sys.stderr.write("nccl_loopback_driver: libnccl mapped besides the stand-in (%s): another copy of NCCL (torch, "
                         "a sitecustomize) would take the library's collectives\n" % sorted(nccl - {STAND_IN}))
        sys.exit(WRONG_NCCL)


check_maps()

if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import wva_import  # noqa: E402

wva = wva_import.load()
abi = wva.abi
from inferno_autoscaler_b200 import binding  # noqa: E402

_stand_in.loopback_counters.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]


def counters(rank):
    """the stand-in's counters of rank `rank` of the newest communicator: gathers, bytes of the last one, destroyed,
    then process-wide: communicators created, destroyed, ncclGroupStart and ncclGroupEnd calls"""
    v = (C.c_uint64 * 7)()
    rc = _stand_in.loopback_counters(None, int(rank), v)
    assert rc == 0, rc
    return np.array(list(v), dtype=np.int64)


def image(z, name):
    S, A, M, T = (int(x) for x in z[name + ".dims"])
    img = wva.image.SystemImage(S, A, M, T)
    for f, dt in img.ALL_FIELDS:
        setattr(img, f, np.ascontiguousarray(z[name + "." + f], dtype=dt))
    return img


def run_all(G, fn):
    """fn(rank) on G host threads at once (ctypes releases the GIL inside the library); re-raises the first failure"""
    res, err = [None] * G, [None] * G

    def body(r):
        try:
            res[r] = fn(r)
        except BaseException as e:          # noqa: B902 - re-raised below
            err[r] = e

    th = [threading.Thread(target=body, args=(r,)) for r in range(G)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in err:
        if e is not None:
            raise e
    return res


def code_of(call, *args):
    """WVA_OK, or the code of the WvaError the call raised"""
    try:
        call(*args)
        return abi.OK
    except binding.WvaError as e:
        return e.code


def put_allocs(out, key, allocs):
    for name, _ in abi.ALLOC_FIELDS:
        out[key + "." + name] = getattr(allocs, name)


def shard_of(ctx):
    f, n = C.c_int32(0), C.c_int32(0)
    rc = binding.lib().wva_shard_info(ctx._h, C.byref(f), C.byref(n))
    assert rc == abi.OK
    return f.value, n.value


def limited(out, key, ctxs, G, policy, delayed, ranked):
    """re-size the pairs, one limited solve on every rank, a refused second solve on the scaled rows, the totals"""
    def body(r):
        c = ctxs[r]
        c.analyze_pairs(download=False)
        k0 = counters(r)
        c.solve_set_ranked(ranked)
        try:
            acc, chosen = c.solve(unlimited=False, delayed_best_effort=delayed, policy=policy)
            path = c.solve_greedy_path()
        finally:
            c.solve_set_ranked(2)
        k1 = counters(r)
        again = code_of(c.solve, False, delayed, policy)        # the records are scaled: wva_analyze_pairs first
        k2 = counters(r)
        count, cost = c.allocate_by_type()
        k3 = counters(r)
        return acc, chosen, path, again, np.stack([k0, k1, k2, k3]), count, cost
    for r, (acc, chosen, path, again, ks, count, cost) in enumerate(run_all(G, body)):
        p = "%s.r%d" % (key, r)
        out[p + ".acc"] = acc
        put_allocs(out, p + ".chosen", chosen)
        out[p + ".path"] = np.int64(path)
        out[p + ".again"] = np.int64(again)
        out[p + ".counters"] = ks
        out[p + ".count"], out[p + ".cost"] = count, cost


def case_unique_id(z, cfg, out):
    out["id"] = np.frombuffer(binding.comm_unique_id(), dtype=np.uint8)


def case_comm(z, cfg, out):
    G = int(cfg["G"])
    r_max, b_max = cfg["sweep"]
    uid = binding.comm_unique_id()
    imgs = [image(z, "img") for _ in range(G)]          # one copy per rank: the binding's updates edit ctx.image
    ctxs = [binding.Context(0) for _ in range(G)]
    try:
        def attach(r):
            c = ctxs[r]
            c.comm_init(uid, r, G)
            c.upload(imgs[r])
            up = shard_of(c)
            if not cfg.get("no_comm_shard"):
                c.comm_shard()
            return c.comm_info(), up, shard_of(c)
        for r, (info, up, sh) in enumerate(run_all(G, attach)):
            out["r%d.info" % r], out["r%d.upload_shard" % r], out["r%d.shard" % r] = np.array(info), np.array(up), np.array(sh)

        update = cfg.get("update")
        if update:                                      # a row-changing update, no wva_comm_shard after it
            def upd(r):
                c = ctxs[r]
                if update == "update_servers":
                    c.update_servers(int(cfg["first"]), image(z, "rows"))
                elif update == "update_models":
                    c.update_models(int(cfg["first"]), image(z, "rows"))
                elif update == "remove_server":
                    c.remove_server(int(cfg["index"]))
                else:
                    raise KeyError(update)
                return shard_of(c), c.dims()
            for r, (sh, dims) in enumerate(run_all(G, upd)):
                out["r%d.update_shard" % r], out["r%d.update_dims" % r] = np.array(sh), np.array(dims)

        for plan in cfg.get("bad_shards", []):          # shards that do not tile the image, then the repair
            key = "bad%d" % cfg["bad_shards"].index(plan)

            def bad(r):
                c = ctxs[r]
                c.set_shard(*plan[r])
                c.analyze_pairs(download=False)
                k0 = counters(r)
                rc = code_of(c.solve, False, False, abi.POLICY_PRIORITY_EXHAUSTIVE)
                k1 = counters(r)
                c.comm_shard()
                return rc, np.stack([k0, k1])
            for r, (rc, ks) in enumerate(run_all(G, bad)):
                out["%s.r%d.rc" % (key, r)], out["%s.r%d.counters" % (key, r)] = np.int64(rc), ks
            limited(out, key + ".repair", ctxs, G, abi.POLICY_PRIORITY_EXHAUSTIVE, False, 2)

        def unlimited(r):
            c = ctxs[r]
            k0 = counters(r)
            c.analyze(r_max, b_max)
            pairs, feas = c.pairs_fetch()
            best = c.grid_fetch()
            acc, chosen = c.solve(unlimited=True)
            f, n = c.first, c.count
            c.analyze_pairs_batches([1, 64])
            c.analyze_pairs_loads(np.stack([c.image.srv_arrival_rpm[f:f + n]] * 2, axis=1))
            k1 = counters(r)
            count, cost = c.allocate_by_type()
            k2 = counters(r)
            return pairs, feas, best, acc, chosen, np.stack([k0, k1, k2]), count, cost
        for r, (pairs, feas, best, acc, chosen, ks, count, cost) in enumerate(run_all(G, unlimited)):
            p = "unl.r%d" % r
            put_allocs(out, p + ".pairs", pairs)
            out[p + ".feasible"], out[p + ".best"], out[p + ".acc"] = feas, best, acc
            put_allocs(out, p + ".chosen", chosen)
            out[p + ".counters"], out[p + ".count"], out[p + ".cost"] = ks, count, cost

        for i, (policy, delayed, ranked) in enumerate(cfg.get("limited", [])):
            limited(out, "lim%d" % i, ctxs, G, policy, bool(delayed), ranked)

        def destroy(r):
            ctxs[r].comm_destroy() if r % 2 == 0 else ctxs[r].close()     # both ways a rank lets go of its communicator
            return counters(r)
        for r, k in enumerate(run_all(G, destroy)):
            out["r%d.destroyed" % r] = k
    finally:
        for c in ctxs:
            c.close()
    out["final"] = counters(0)


def case_group(z, cfg, out):
    G = int(cfg["G"])
    r_max, b_max = cfg["sweep"]
    img = image(z, "img")
    batches = np.asarray(cfg["batches"], dtype=np.int32)
    rpm = np.ascontiguousarray(z["rpm"], dtype=np.float32)
    g = binding.Group([0] * G)
    try:
        out["shards.create"] = counters(0)
        g.upload(img)
        out["shards"] = np.array([shard_of(c) for c in g.ctxs])
        g.analyze(0, 0)
        put_allocs(out, "p0.pairs", g.pairs_fetch()[0])
        out["p0.feasible"] = g.pairs_fetch()[1]

        def sweep(key):
            for cube in (False, True):
                k = "%s.cube%d" % (key, cube)
                g.analyze(r_max, b_max, want_cube=cube)
                pairs, feas = g.pairs_fetch()
                put_allocs(out, k + ".pairs", pairs)
                out[k + ".feasible"], out[k + ".best"], out[k + ".p_block"] = feas, g.grid_fetch(), g.grid_best_blocking()
            out[key + ".batches"], out[key + ".batches_best"] = g.analyze_pairs_batches(batches)
            pl, best = g.analyze_pairs_loads(rpm)
            out[key + ".loads"], out[key + ".loads_best"] = pl, best
            acc, chosen = g.solve(unlimited=True)
            out[key + ".unl.acc"] = acc
            put_allocs(out, key + ".unl.chosen", chosen)
            out[key + ".unl.count"], out[key + ".unl.cost"] = g.allocate_by_type()
            for i, (policy, delayed, ranked) in enumerate(cfg["limited"]):
                k = "%s.lim%d" % (key, i)
                g.analyze(0, 0)
                for c in g.ctxs:
                    c.solve_set_ranked(ranked)
                try:
                    acc, chosen = g.solve(unlimited=False, delayed_best_effort=bool(delayed), policy=policy)
                finally:
                    for c in g.ctxs:
                        c.solve_set_ranked(2)
                out[k + ".acc"] = acc
                put_allocs(out, k + ".chosen", chosen)
                out[k + ".count"], out[k + ".cost"] = g.allocate_by_type()
                out[k + ".gathers"] = np.array([counters(r)[0] for r in range(G)])

        sweep("base")

        # errors: a NaN rate and n_l = 0 leave the caller's plane and best untouched and name a device or the rate
        L = binding.lib()
        n_l = rpm.shape[1]
        plane = np.frombuffer(np.full(img.S * n_l * img.A * abi.PAIR_REC_DTYPE.itemsize, 0xA5, dtype=np.uint8).tobytes(),
                              dtype=abi.PAIR_REC_DTYPE).copy()
        best = np.frombuffer(np.full(img.S * n_l * abi.PAIR_REC_DTYPE.itemsize, 0xA5, dtype=np.uint8).tobytes(),
                             dtype=abi.PAIR_REC_DTYPE).copy()
        bad = rpm.copy()
        bad[img.S - 1, n_l - 1] = np.nan                 # the last device's last row
        rc_nan = L.wva_group_analyze_pairs_loads(g._h, n_l, abi.ptr(bad, C.c_float), plane.ctypes.data, best.ctypes.data)
        msg_nan = L.wva_group_last_error(g._h).decode()
        rc_zero = L.wva_group_analyze_pairs_loads(g._h, 0, abi.ptr(rpm, C.c_float), plane.ctypes.data, best.ctypes.data)
        msg_zero = L.wva_group_last_error(g._h).decode()
        out["err.rc"] = np.array([rc_nan, rc_zero])
        out["err.untouched"] = np.array([plane.view(np.uint8).min(), plane.view(np.uint8).max(),
                                         best.view(np.uint8).min(), best.view(np.uint8).max()])
        out["err.msg"] = np.array([msg_nan, msg_zero])
        pl, bs = g.analyze_pairs_loads(rpm)
        out["after.loads"], out["after.loads_best"] = pl, bs

        # a tuning switch on one member: certified tails off on ctx 1
        g.ctxs[1].set_certified_tails(0)
        sweep("tails")
        out["final"] = counters(0)
    finally:
        g.close()
    out["closed"] = counters(0)

    # one plain context over the whole image: what the assembled plane must equal
    ctx = binding.Context(0)
    try:
        ctx.upload(img)
        pl, best = ctx.analyze_pairs_batches(batches)
        out["single.batches"], out["single.batches_best"] = pl, best
        pl, best = ctx.analyze_pairs_loads(rpm)
        out["single.loads"], out["single.loads_best"] = pl, best
    finally:
        ctx.close()


CASES = {"unique_id": case_unique_id, "comm": case_comm, "group": case_group}


def main(argv):
    case, src, dst = argv[1:4]
    z = dict(np.load(src, allow_pickle=False)) if os.path.exists(src) else {}
    cfg = json.loads(str(z["cfg"])) if "cfg" in z else {}
    out = {}
    CASES[case](z, cfg, out)
    check_maps()
    np.savez(dst, **out)


if __name__ == "__main__":
    main(sys.argv)
