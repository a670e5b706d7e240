"""Images, shard plans and expected totals for the sharded Analyze -> Optimize exchange, emulated on one device.

Several contexts on one GPU, each sharded like one rank of `distributed.shard_range`, stand in for a multi-rank run: the
candidate rows move between them by device-to-device copies and the totals blocks are concatenated in rank order by
hand, so the only part of the multi-GPU flow left out is the collective itself.  Shared by
tests/test_rank_emulation_cpu.py (the plans have the shapes claimed below, and a bit-exact check of the cost totals can
tell summation orders apart on these images) and tests/test_rank_emulation_gpu.py (every rank's results against the
oracle).

  * P1: 5 000 servers x 6 accelerators, 3 types, with accelerator costs spread over six magnitudes and none of them an
    integer, so float32 cost sums round and their order shows in the bits.  G = 2, 3, 5: shards of 1 000 - 2 500 servers
    starting at servers that are not multiples of 1 024 and spanning one to three of k_totals' 1 024-server staging
    blocks.
  * P2: 61 x 4, 2 types; G = 2 and 5 give shards whose sizes differ by one server.
  * P3: 5 x 3; G = 8 leaves several shards empty.
  * P4: P2 as one rank (G = 1).

Every image gets capacities of 0.55 of its unlimited demand, so that limited solves bind.  Expected totals of a plan:
each shard's partial is oracle.allocate_by_type over [first, first + count) (ascending server order), the global cost is
the float32 left fold of the partials over the ranks in rank order starting from +0 (what k_totals_merge computes), and
the global count is the int64 sum of the partials, which wraps like the device's.
"""
import functools

import numpy as np

import wva_import

_wva = wva_import.load()
abi = _wva.abi
from inferno_autoscaler_b200 import distributed  # noqa: E402

P1_COSTS = np.array([0.37, 3.1, 41.3, 977.7, 1.3e4, 2.9e5], dtype=np.float32)
CAPACITY_FRACTION = 0.55
STAGE = 1024                                    # servers k_totals stages per round of its in-order sum

PLANS = {"P1": (2, 3, 5), "P2": (2, 5), "P3": (8,), "P4": (1,)}
# (r_max, b_max) of the sweep wva_analyze runs beside pair sizing
SWEEP = {"P1": (2, 16), "P2": (4, 32), "P3": (4, 32), "P4": (4, 32)}


def plan(S, G):
    """[(first, count)] of ranks 0 .. G-1"""
    return [distributed.shard_range(S, r, G) for r in range(G)]


def cases():
    """every (image, G) pair the tests run"""
    return [(name, G) for name, gs in PLANS.items() for G in gs]


class Reference:
    """an image with its capacities, and the oracle's pair rows, feasibility and unlimited decisions over all of it"""

    def __init__(self, img, pairs, feasible, acc, chosen):
        self.img, self.pairs, self.feasible, self.acc, self.chosen = img, pairs, feasible, acc, chosen


def _image(name):
    synth = _wva.synth
    if name == "P1":
        img = synth.make_system(5000, 6, seed=1701, n_types=3, max_pair_batch=256)
        img.acc_cost[:] = P1_COSTS
    elif name in ("P2", "P4"):
        img = synth.make_system(61, 4, seed=1702, n_types=2)
    elif name == "P3":
        img = synth.make_system(5, 3, seed=1703)
    else:
        raise KeyError(name)
    return img


@functools.lru_cache(maxsize=None)
def reference(name):
    """the image `name` with capacities set from its unlimited demand, and the oracle's results over the whole image"""
    import oracle
    img = _image(name)
    pairs, feasible, _ = oracle.analyze_pairs(img, threads=oracle.hardware_threads())
    acc, chosen = oracle.solve(img, pairs, feasible, unlimited=True)
    _wva.synth.set_capacity_from_demand(img, acc, chosen.num_replicas, fraction=CAPACITY_FRACTION)
    return Reference(img, pairs, feasible, acc, chosen)


def partials(oracle, img, acc, chosen, G):
    """[(count[T], cost[T])] of every rank of the plan: the oracle's AllocateByType over the rank's servers"""
    return [oracle.allocate_by_type(img, acc, chosen, f, f + c) for f, c in plan(img.S, G)]


def fold_cost(parts, order=None):
    """float32 left fold of the partial costs over the ranks in `order` (rank order by default), starting from +0"""
    order = range(len(parts)) if order is None else order
    k = np.zeros(len(parts[0][1]), dtype=np.float32)
    for r in order:
        k = (k + parts[r][1]).astype(np.float32)
    return k


def sum_count(parts):
    """int64 sum of the partial counts (wraps as the device's does)"""
    out = np.zeros(len(parts[0][0]), dtype=np.int64)
    with np.errstate(over="ignore"):
        for c, _ in parts:
            out = out + c
    return out


def expected_totals(oracle, img, acc, chosen, G):
    """(count, cost) a G-rank run must hold on every rank after the exchange"""
    parts = partials(oracle, img, acc, chosen, G)
    return sum_count(parts), fold_cost(parts)


def contributions(img, acc, chosen, t):
    """float32 cost each server adds to type t's total (+0 for a server of another type or without an allocation)"""
    ok = (np.asarray(acc) >= 0) & (chosen.acc >= 0) & (img.srv_model >= 0)
    ty = np.where(ok, img.acc_type[np.where(ok, chosen.acc, 0)], -1)
    return np.where(ty == t, chosen.cost, np.float32(0.0)).astype(np.float32)


def ascending_sum(v):
    k = np.float32(0.0)
    for x in v:
        k = np.float32(k + x)
    return k


def pairwise_sum(v):
    """float32 tree sum: halves summed recursively, then added"""
    if len(v) == 0:
        return np.float32(0.0)
    if len(v) == 1:
        return np.float32(v[0])
    h = len(v) // 2
    return np.float32(pairwise_sum(v[:h]) + pairwise_sum(v[h:]))
