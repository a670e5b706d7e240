"""Time pair sizing over arrival-rate scenarios against the loop a caller writes without it, on one GPU.

    python tools/pairs_loads_bench.py [--rounds 10] [--warmup 2]

Config 3 (1 000 servers x 8 accelerators), n_l = 24 and n_l = 96 seeded scenario columns.  Each column scales the
uploaded rates by a factor drawn from [0, 4]; a few columns hold zeros (every server idle).
  call    one wva_analyze_pairs_loads call, plane and per-(server, scenario) choice copied to the host
  loop    per scenario j: wva_system_update_servers with srv_arrival_rpm = column j, wva_analyze_pairs, wva_pairs_fetch,
          wva_solve(unlimited), wva_solution_fetch (what a caller has to do without the call)
The two alternate round by round.  Both end in a device synchronisation inside the library; the host clock around them
is also bracketed by torch.cuda.synchronize.  Before timing, the plane and the choices are checked byte for byte against
the loop's records.  Prints one JSON line per n_l (median and min-max over the rounds, the call's counters) and the
card's name, power limit and max SM clock, queried in the same run.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from pairs_plane_bench import FIELDS, card, stats, timed  # noqa: E402


def scenarios(base, n_l, seed):
    rng = np.random.default_rng(seed)
    fac = rng.uniform(0.0, 4.0, n_l).astype(np.float32)
    fac[rng.choice(n_l, max(1, n_l // 12), replace=False)] = 0.0
    return (base.astype(np.float32)[:, None] * fac[None, :]).astype(np.float32)


def main():
    ap = argparse.ArgumentParser(description="pair sizing over arrival-rate scenarios vs the per-scenario loop")
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

    def call(rpm):
        return ctx.analyze_pairs_loads(rpm)

    def loop(rpm):
        out = []
        for j in range(rpm.shape[1]):
            rows.srv_arrival_rpm[:] = rpm[:, j]
            ctx.update_servers(0, rows)
            ctx.analyze_pairs(download=False)
            allocs, fe = ctx.pairs_fetch()
            ctx.solve(unlimited=True, download=False)
            acc, chosen = ctx.solution_fetch()
            out.append((allocs, fe, acc, chosen))
        return out

    print(json.dumps(dict(card=card())), flush=True)
    for n_l, seed in ((24, 101), (96, 102)):
        rpm = scenarios(img.srv_arrival_rpm, n_l, seed)
        plane, best = call(rpm)
        for j, (allocs, fe, acc, chosen) in enumerate(loop(rpm)):
            col = plane[:, j].reshape(-1)
            assert np.array_equal(col["feasible"], fe), (n_l, j)
            for f in FIELDS:
                assert col[f].tobytes() == getattr(allocs, f).tobytes(), (n_l, j, f)
            b = best[:, j]
            has = acc >= 0
            assert (b["acc"][~has] == -1).all(), (n_l, j)
            assert (b["feasible"] == has).all(), (n_l, j)
            for f in FIELDS:
                assert b[f][has].tobytes() == getattr(chosen, f)[has].tobytes(), (n_l, j, f)
        for _ in range(args.warmup):
            call(rpm); loop(rpm)
        tc, tl = [], []
        for _ in range(args.rounds):
            tc.append(timed(lambda: call(rpm))[0])
            tl.append(timed(lambda: loop(rpm))[0])
        print(json.dumps(dict(workload="config3", n_l=n_l, call=stats(tc), loop=stats(tl), same_bytes=True,
                              counters=ctx.pairs_loads_counters())), flush=True)
    print(json.dumps(dict(card=card())), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
