"""Time the blocking-probability calls beside the candidate sweep on one GPU.

    python tools/block_bench.py [--steps 10] [--warmup 2] [--no-config4]

Config 3 (bench.py's default workload: 1 000 servers x 8 accelerators x replicas 1-64 x batch 1-512, metric cube kept),
in one process, alternating step by step:
  sweep            wva_analyze_grid_device (the sweep alone)
  sweep+plane      the same sweep followed by wva_grid_blocking (plane left in HBM)
  winners          wva_grid_best_blocking on its own (after a sweep)
Then config 4 on a single GPU (10 000 servers, winners only: the cube does not fit): the sweep, wva_grid_best_blocking
and wva_grid_blocking.  Every time is a host clock around calls that end in a device synchronisation; the median and
the spread (min, max) over the timed steps are printed, with the three counts of each plane and the card's name and
power limit.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description="blocking-probability calls beside the sweep")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-config4", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    import __graft_entry__ as g
    wva = g.build()
    from inferno_autoscaler_b200 import binding
    result = dict(card=card())
    ctx = binding.Context(0)
    try:
        img, c = wva.synth.baseline_config(3)
        R, B = c["r_max"], c["b_max"]
        ctx.upload(img)
        sweep = lambda: ctx.analyze_grid_device(R, B, want_cube=True)               # noqa: E731
        plane = lambda: (ctx.analyze_grid_device(R, B, want_cube=True), ctx.grid_blocking(download=False))   # noqa: E731
        for _ in range(args.warmup):
            sweep(); plane(); ctx.grid_best_blocking()
        t = dict(sweep=[], sweep_plane=[], winners=[])
        for _ in range(args.steps):
            t["sweep"].append(timed(sweep))
            t["sweep_plane"].append(timed(plane))
            t["winners"].append(timed(ctx.grid_best_blocking))
        result["config3"] = dict(candidates=img.S * img.A * R * B, counts=ctx.grid_blocking_counts(),
                                 **{k: stats(v) for k, v in t.items()})
        if not args.no_config4:
            img4, c4 = wva.synth.baseline_config(4)
            R4, B4 = c4["r_max"], c4["b_max"]
            ctx.upload(img4)
            sweep4 = lambda: ctx.analyze_grid_device(R4, B4, want_cube=False)         # noqa: E731
            sweep4(); ctx.grid_best_blocking(); ctx.grid_blocking(download=False)
            t4 = dict(sweep=[], winners=[], plane=[])
            for _ in range(max(1, args.steps // 2)):
                t4["sweep"].append(timed(sweep4))
                t4["winners"].append(timed(ctx.grid_best_blocking))
                t4["plane"].append(timed(lambda: ctx.grid_blocking(download=False)))
            result["config4_single_gpu"] = dict(candidates=img4.S * img4.A * R4 * B4, counts=ctx.grid_blocking_counts(),
                                                **{k: stats(v) for k, v in t4.items()})
    finally:
        ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
