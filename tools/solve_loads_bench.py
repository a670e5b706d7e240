"""Time the limited solve over a matrix of arrival-rate scenarios against the loop a caller writes without it, on one GPU.

    python tools/solve_loads_bench.py [--rounds 5] [--warmup 1]

Config 3 (1 000 servers x 8 accelerators, 3 types) with capacities at 60 % of the unlimited demand at the uploaded load
(synth.set_capacity_from_demand), so that they bind in most scenarios; n_l = 24 and 96 scenarios, scenario j at
0.2 + 1.8 j / (n_l - 1) times the uploaded rates.  PriorityExhaustive best effort.
  call    one wva_solve_loads call, decisions, records and totals copied to the host
  device  the same call with every output pointer NULL: sizing, orders, scans, collect and totals run, nothing is copied out
  loop    per scenario: wva_system_update_servers with the scenario's rates, wva_analyze_pairs, wva_solve (limited),
          wva_solution_fetch, wva_allocate_by_type -- what a caller has to do without the call
The three alternate round by round.  All end in a device synchronisation inside the library; the host clock around them
is also bracketed by torch.cuda.synchronize.  Before timing, the call's outputs are checked byte for byte against the
loop's.  Prints one JSON line per n_l (median and min-max over the rounds, the call's counters) and the card's name,
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


def main():
    ap = argparse.ArgumentParser(description="limited solve over arrival-rate scenarios vs the per-scenario loop")
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
    wva.synth.set_capacity_from_demand(img, acc, chosen.num_replicas, 0.6)
    ctx.upload(img)
    base = img.shard(0, img.S)

    def call(rpm):
        return ctx.solve_loads(rpm, policy=POLICY)

    def loop(rpm):
        out = []
        for j in range(rpm.shape[1]):
            rows = base.shard(0, base.S)
            rows.srv_arrival_rpm[:] = rpm[:, j]
            ctx.update_servers(0, rows)
            ctx.analyze_pairs(download=False)
            ctx.solve(unlimited=False, policy=POLICY, download=False)
            a, ch = ctx.solution_fetch()
            out.append((a, ch, ctx.allocate_by_type()))
        ctx.update_servers(0, base)
        return out

    print(json.dumps(dict(card=card())), flush=True)
    for n_l in (24, 96):
        fac = np.linspace(0.2, 2.0, n_l).astype(np.float32)
        rpm = (img.srv_arrival_rpm.astype(np.float32)[:, None] * fac[None, :]).astype(np.float32)
        c_acc, c_recs, c_count, c_cost = call(rpm)
        for j, (a, ch, (count, cost)) in enumerate(loop(rpm)):
            assert c_acc[j].tobytes() == a.tobytes(), (n_l, j)
            assert (c_recs[j]["feasible"] == (a >= 0)).all(), (n_l, j)
            for f in ("acc", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate_per_replica"):
                assert c_recs[j][f].tobytes() == getattr(ch, f).tobytes(), (n_l, j, f)
            assert c_count[j].tobytes() == count.tobytes() and c_cost[j].tobytes() == cost.tobytes(), (n_l, j)
        placed = (c_acc >= 0).sum(axis=1)
        for _ in range(args.warmup):
            call(rpm); loop(rpm)  # noqa: E702
        tc, td, tl = [], [], []
        for _ in range(args.rounds):
            tc.append(timed(lambda: call(rpm))[0])
            td.append(timed(lambda: ctx.solve_loads(rpm, policy=POLICY, download=False))[0])
            tl.append(timed(lambda: loop(rpm))[0])
        print(json.dumps(dict(workload="config3", n_l=n_l, call=stats(tc), device=stats(td), loop=stats(tl), same_bytes=True,
                              placed_min=int(placed.min()), placed_max=int(placed.max()), servers=img.S,
                              counters=ctx.solve_loads_counters())), flush=True)
    print(json.dumps(dict(card=card())), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
