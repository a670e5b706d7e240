"""Torch-free subprocess that runs wva_solve_capacities through the library's own multi-rank paths on ONE GPU, with the
loopback NCCL stand-in (loaded by tests/nccl_loopback_driver.py, whose helpers this reuses).

    python solve_capacities_loopback_driver.py CASE IN.npz OUT.npz

IN.npz holds the image ("img.<field>", "img.dims"), the capacity list "caps" and "cfg" (JSON: G, policy, delayed).
Cases:
  comm   G contexts on device 0 attached by wva_comm_init, each sizing only its wva_comm_shard rows; every rank calls
         wva_solve_capacities twice (the first call gathers the rows, the second finds them complete), the stand-in's
         all-gather counters are read around each call;
  group  one wva_group over [0] * G: wva_group_solve_capacities after wva_group_analyze, its all-gather counters, a
         refused call (one member without valid records) that must leave every member's counters alone, and one plain
         context over the whole image for comparison.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import nccl_loopback_driver as nd  # noqa: E402  (loads the stand-in before the library)

import numpy as np  # noqa: E402

abi, binding = nd.abi, nd.binding


def put(out, key, res):
    acc, recs, count, cost = res
    out[key + ".acc"], out[key + ".recs"], out[key + ".count"], out[key + ".cost"] = acc, recs, count, cost


def case_comm(z, cfg, out):
    G, policy, delayed = int(cfg["G"]), int(cfg["policy"]), bool(cfg["delayed"])
    caps = np.ascontiguousarray(z["caps"], dtype=np.int64)
    uid = binding.comm_unique_id()
    imgs = [nd.image(z, "img") for _ in range(G)]
    ctxs = [binding.Context(0) for _ in range(G)]
    try:
        def body(r):
            c = ctxs[r]
            c.comm_init(uid, r, G)
            c.upload(imgs[r])
            c.comm_shard()
            c.analyze_pairs(download=False)
            k0 = nd.counters(r)[0]
            first = c.solve_capacities(caps, delayed_best_effort=delayed, policy=policy)
            k1 = nd.counters(r)[0]
            second = c.solve_capacities(caps, delayed_best_effort=delayed, policy=policy)
            k2 = nd.counters(r)[0]
            return nd.shard_of(c), first, second, np.array([k1 - k0, k2 - k1]), c.solve_capacities_counters()["path"]
        for r, (shard, first, second, gathers, path) in enumerate(nd.run_all(G, body)):
            p = "r%d" % r
            out[p + ".shard"] = np.array(shard)
            put(out, p + ".first", first)
            put(out, p + ".second", second)
            out[p + ".gathers"] = gathers
            out[p + ".path"] = np.int64(path)
    finally:
        for c in ctxs:
            c.close()


def case_group(z, cfg, out):
    G, policy, delayed = int(cfg["G"]), int(cfg["policy"]), bool(cfg["delayed"])
    caps = np.ascontiguousarray(z["caps"], dtype=np.int64)
    img = nd.image(z, "img")
    g = binding.Group([0] * G)
    try:
        g.upload(img)
        out["shards"] = np.array([nd.shard_of(c) for c in g.ctxs])
        g.analyze(0, 0)
        k0 = np.array([nd.counters(r)[0] for r in range(G)])
        put(out, "group", g.solve_capacities(caps, delayed_best_effort=delayed, policy=policy))
        k1 = np.array([nd.counters(r)[0] for r in range(G)])
        put(out, "again", g.solve_capacities(caps, delayed_best_effort=delayed, policy=policy))
        k2 = np.array([nd.counters(r)[0] for r in range(G)])
        out["gathers"] = np.stack([k1 - k0, k2 - k1])
        # the last member loses its records (a shard change drops them): the call is refused before any member gathers
        last = g.ctxs[G - 1]
        last.set_shard(last.first, last.count)
        out["refused"] = np.int64(nd.code_of(g.solve_capacities, caps))
        out["refused.msg"] = np.array(binding.lib().wva_group_last_error(g._h).decode())
        out["refused.gathers"] = np.array([nd.counters(r)[0] for r in range(G)]) - k2
    finally:
        g.close()
    ctx = binding.Context(0)
    try:
        ctx.upload(img)
        ctx.analyze_pairs(download=False)
        put(out, "single", ctx.solve_capacities(caps, delayed_best_effort=delayed, policy=policy))
    finally:
        ctx.close()


CASES = {"comm": case_comm, "group": case_group}


def main(argv):
    case, src, dst = argv[1:4]
    z = dict(np.load(src, allow_pickle=False))
    cfg = json.loads(str(z["cfg"]))
    out = {}
    CASES[case](z, cfg, out)
    nd.check_maps()
    np.savez(dst, **out)


if __name__ == "__main__":
    main(sys.argv)
