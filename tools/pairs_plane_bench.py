"""Time pair sizing over a batch-size list against the loop a caller writes without it, on one GPU.

    python tools/pairs_plane_bench.py [--rounds 10] [--warmup 2]

Config 3 (1 000 servers x 8 accelerators), two lists: L10 = {1, 2, 4, ..., 512} and L512 = {1, ..., 512}.
  plane   one wva_analyze_pairs_batches call, plane and per-server choice copied to the host
  loop    per batch size b: wva_system_update_servers with srv_max_batch = b on every server, wva_analyze_pairs,
          wva_pairs_fetch (what a caller has to do without the list call)
The two alternate round by round.  Both end in a device synchronisation inside the library; the host clock around them
is also bracketed by torch.cuda.synchronize.  Before timing, the plane is checked byte for byte against the loop's
records.  Prints one JSON line per list (median and min-max over the rounds) and the card's name, power limit and max
SM clock, queried in the same run.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FIELDS = ["acc", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate_per_replica"]


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True).strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:      # the query is informative only
        return dict(error=str(e))


def stats(ts):
    ts = sorted(ts)
    return dict(median_ms=round(1e3 * ts[len(ts) // 2], 3), min_ms=round(1e3 * ts[0], 3), max_ms=round(1e3 * ts[-1], 3))


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser(description="pair sizing over a batch-size list vs the per-b loop")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    import wva_import
    wva = wva_import.load()
    from inferno_autoscaler_b200 import binding
    img, _ = wva.synth.baseline_config(3)
    ctx = binding.Context(0)
    ctx.upload(img)
    rows = img.shard(0, img.S)

    def plane_call(batch):
        return ctx.analyze_pairs_batches(batch)[0]

    def loop(batch):
        cols = []
        for b in batch:
            rows.srv_max_batch[:] = b
            ctx.update_servers(0, rows)
            ctx.analyze_pairs(download=False)
            allocs, fe = ctx.pairs_fetch()
            cols.append((allocs, fe))
        return cols

    print(json.dumps(dict(card=card())), flush=True)
    for name, batch in (("L10", [1 << k for k in range(10)]), ("L512", list(range(1, 513)))):
        plane = plane_call(batch)
        for j, (allocs, fe) in enumerate(loop(batch)):
            col = plane[:, j]
            assert np.array_equal(col["feasible"], fe), (name, j)
            for f in FIELDS:
                assert col[f].tobytes() == getattr(allocs, f).tobytes(), (name, j, f)
        for _ in range(args.warmup):
            plane_call(batch); loop(batch)
        tp, tl = [], []
        for _ in range(args.rounds):
            tp.append(timed(lambda: plane_call(batch))[0])
            tl.append(timed(lambda: loop(batch))[0])
        print(json.dumps(dict(workload="config3", list=name, n_b=len(batch), plane=stats(tp), loop=stats(tl),
                              same_bytes=True, counters=ctx.pairs_batches_counters())), flush=True)
    print(json.dumps(dict(card=card())), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
