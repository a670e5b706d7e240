"""Time the limited solve over a list of capacity vectors against the loop a caller writes without it, on one GPU.

    python tools/solve_capacities_bench.py [--rounds 5] [--warmup 1]

Config 3 (1 000 servers x 8 accelerators, 3 types), n_c = 32, 128 and 1 024 capacity vectors.  Vector j sets each type
to a fraction of the unlimited demand (synth.set_capacity_from_demand), the fractions drawn from [0.05, 1.2] per type.
  call    one wva_solve_capacities call (PriorityExhaustive best effort), decisions, records and totals copied to the host
  device  the same call with every output pointer NULL: the solves, collect and totals kernels run, nothing is copied out
  loop    per vector: wva_system_set_capacity, wva_analyze_pairs, wva_solve (limited), wva_solution_fetch,
          wva_allocate_by_type -- what a caller has to do without the call.  A limited wva_solve scales the records it
          consumed, and wva_pairs_device / wva_pairs_commit refuse them afterwards, so re-analysis is the only way back to
          valid records through the public interface; a loop that restores saved records instead has no public door.
The three alternate round by round.  All end in a device synchronisation inside the library; the host clock around them
is also bracketed by torch.cuda.synchronize.  Before timing, the call's outputs are checked byte for byte against the
loop's.  Prints one JSON line per n_c (median and min-max over the rounds, the call's counters) and the card's name,
power limit and max SM clock, queried in the same run.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pairs_plane_bench import card, stats, timed  # noqa: E402

POLICY = 1      # PriorityExhaustive


def capacities(wva, img, acc, chosen, n_c, seed):
    rng = np.random.default_rng(seed)
    out = np.zeros((n_c, img.T), dtype=np.int64)
    saved = img.type_capacity.copy()
    demand = wva.synth.set_capacity_from_demand(img, acc, chosen.num_replicas, 1.0)
    img.type_capacity[:] = saved
    for j in range(n_c):
        out[j] = np.ceil(rng.uniform(0.05, 1.2, img.T) * demand).astype(np.int64)
    return out


def main():
    ap = argparse.ArgumentParser(description="limited solve over capacity vectors vs the per-vector loop")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
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
    ctx.analyze_pairs(download=False)
    acc, chosen = ctx.solve(unlimited=True)
    saved = img.type_capacity.copy()

    def call(caps):
        return ctx.solve_capacities(caps, policy=POLICY)

    def loop(caps):
        out = []
        for cap in caps:
            ctx.set_capacity(cap)
            ctx.analyze_pairs(download=False)
            ctx.solve(unlimited=False, policy=POLICY, download=False)
            a, ch = ctx.solution_fetch()
            out.append((a, ch, ctx.allocate_by_type()))
        ctx.set_capacity(saved)
        ctx.analyze_pairs(download=False)
        return out

    print(json.dumps(dict(card=card())), flush=True)
    for n_c, seed in ((32, 201), (128, 202), (1024, 203)):
        caps = capacities(wva, img, acc, chosen, n_c, seed)
        c_acc, c_recs, c_count, c_cost = call(caps)
        for j, (a, ch, (count, cost)) in enumerate(loop(caps)):
            assert c_acc[j].tobytes() == a.tobytes(), (n_c, j)
            has = a >= 0
            assert (c_recs[j]["feasible"] == has).all(), (n_c, j)
            for f in ("acc", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate_per_replica"):
                assert c_recs[j][f].tobytes() == getattr(ch, f).tobytes(), (n_c, j, f)
            assert c_count[j].tobytes() == count.tobytes() and c_cost[j].tobytes() == cost.tobytes(), (n_c, j)
        for _ in range(args.warmup):
            call(caps); loop(caps)
        tc, td, tl = [], [], []
        for _ in range(args.rounds):
            tc.append(timed(lambda: call(caps))[0])
            td.append(timed(lambda: ctx.solve_capacities(caps, policy=POLICY, download=False))[0])
            tl.append(timed(lambda: loop(caps))[0])
        print(json.dumps(dict(workload="config3", n_c=n_c, call=stats(tc), device=stats(td), loop=stats(tl), same_bytes=True,
                              counters=ctx.solve_capacities_counters())), flush=True)
    print(json.dumps(dict(card=card())), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
