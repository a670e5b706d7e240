"""CPU: the pieces of pair sizing over a batch-size list (wva_analyze_pairs_batches) that need no GPU -- the record
layout of wva_pair_rec, the per-server choice restated in numpy against the oracle's SolveUnlimited, and the oracle's
zero-load records under a batch-size override.  The helpers here are shared with test_pairs_plane_gpu.py."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
MAX_F32 = np.finfo(np.float32).max
FIELDS = ["acc", "num_replicas", "batch_size", "cost", "value", "itl", "ttft", "rho", "max_arrv_rate_per_replica"]


def override(img, b):
    """the image with ServerSpec.MaxBatchSize = b on every server"""
    out = img.shard(0, img.S)
    out.srv_max_batch[:] = b
    return out


def to_recs(wva, allocs, feasible):
    """AllocArrays + feasible flags -> wva_pair_rec records (pad bytes 0)"""
    r = np.zeros(len(feasible), dtype=wva.abi.PAIR_REC_DTYPE)
    for name in FIELDS:
        r[name] = getattr(allocs, name)
    r["feasible"] = feasible
    return r


def oracle_plane(wva, oracle, img, batch, threads=None):
    """the reference's records of every pair under every override of `batch`: [S * A, n_b]"""
    threads = threads or oracle.hardware_threads()
    cols = []
    for b in batch:
        allocs, fe, _ = oracle.analyze_pairs(override(img, int(b)), threads=threads)
        cols.append(to_recs(wva, allocs, fe))
    return np.stack(cols, axis=1)


def choose(plane, A, positions=False):
    """SolveUnlimited (solver.go:63-79) over each server's records, scanned a then j: the first feasible record whose
    value is strictly below MaxFloat32 and every earlier choice.  plane [ns * A, n_b] -> best [ns] (and the scan
    position a * n_b + j of each choice, -1 for none)"""
    ns = plane.shape[0] // A
    rows = plane.reshape(ns, -1)
    v = rows["value"]
    with np.errstate(invalid="ignore"):
        ok = (rows["feasible"] != 0) & (v < MAX_F32)
    masked = np.where(ok, v, np.inf).astype(np.float64)
    lo = masked.min(axis=1)
    best = np.zeros(ns, dtype=plane.dtype)
    best["acc"] = -1
    has = lo < np.inf                                      # -Inf is a value like any other
    pos = np.where(has, np.argmax(masked == lo[:, None], axis=1), -1)     # -0 == +0: the earlier one
    best[has] = rows[np.nonzero(has)[0], pos[has]]
    return (best, pos) if positions else best


def rec_bytes(r, names=None):
    """the records' fields as bytes, field by field, NaN payloads folded (they are not part of the contract, see
    AllocArrays.equal_bits)"""
    out = []
    for name in names or r.dtype.names:
        x = np.array(r[name], copy=True)
        if x.dtype == np.float32:
            x[np.isnan(x)] = np.nan
        out.append(x.tobytes())
    return b"".join(out)


def test_pair_rec_layout_matches_c(wva):
    abi = wva.abi
    src = r"""
#include <stddef.h>
#include <stdio.h>
#include "wva_b200.h"
#define P(f) printf("%s %zu\n", #f, offsetof(wva_pair_rec, f));
int main(void) {
    printf("size %zu\n", sizeof(wva_pair_rec));
    P(acc) P(feasible) P(pad) P(num_replicas) P(batch_size) P(cost) P(value) P(itl) P(ttft) P(rho)
    P(max_arrv_rate_per_replica)
    return 0;
}
"""
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, "layout.c"), os.path.join(tmp, "layout")
        open(c, "w").write(src)
        subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", exe, c])
        out = subprocess.check_output([exe], text=True)
    got = dict((k, int(v)) for k, v in (line.split() for line in out.splitlines()))
    dt = abi.PAIR_REC_DTYPE
    assert got.pop("size") == dt.itemsize == 48
    assert got == {name: dt.fields[name][1] for name in dt.names}


def _choice_image(wva):
    img = wva.synth.make_system(60, 5, seed=41, n_types=3, max_pair_batch=512)
    img.srv_arrival_rpm[:10] = 0.0
    img.srv_min_replicas[:10] = np.arange(10) % 2
    # current allocations whose cost makes the transition penalty +Inf, NaN (Inf - Inf) or huge
    img.srv_cur_acc[10:30] = np.arange(20) % 5
    img.srv_cur_replicas[10:30] = 3
    img.srv_cur_cost[10:15] = np.inf
    img.srv_cur_cost[15:20] = -np.inf
    img.srv_cur_cost[20:25] = F(3e38)
    return img


@pytest.mark.parametrize("b", [1, 16, 512])
def test_choice_restatement_equals_oracle_solve(wva, oracle, b):
    img = override(_choice_image(wva), b)
    allocs, fe, _ = oracle.analyze_pairs(img, threads=oracle.hardware_threads())
    A = img.A
    # values the choice must never take or must tie on, written into feasible records
    v = allocs.value.reshape(img.S, A)
    f = fe.reshape(img.S, A)
    f[30:45] = 1
    v[30:33] = [np.nan, 5.0, 5.0, 7.0, 6.0]                    # NaN skipped; the first 5.0 of two is kept
    v[33:36] = [MAX_F32, np.inf, MAX_F32, np.inf, np.nan]      # nothing below MaxFloat32: no choice
    v[36:39] = [0.0, -0.0, 0.0, 1.0, 2.0]                      # +0 first: -0 does not replace it
    v[39:42] = [-0.0, 0.0, 3.0, np.nan, -0.0]                  # -0 first
    v[42:45] = [np.nextafter(MAX_F32, F(0)), MAX_F32, np.inf, np.nan, MAX_F32]
    with np.errstate(invalid="ignore"):
        natural = v[10:25][f[10:25] == 1]
    assert np.isnan(natural).any() and np.isinf(natural).any()        # from the current allocations alone
    chosen_acc, chosen = oracle.solve(img, allocs, fe, unlimited=True)
    best, pos = choose(to_recs(wva, allocs, fe)[:, None], A, positions=True)
    # n_b = 1: the scan position is the accelerator, the oracle's key of the chosen record
    assert np.array_equal(pos, chosen_acc)
    has = chosen_acc >= 0
    rec = to_recs(wva, chosen, np.ones(img.S, np.uint8))
    assert rec_bytes(rec[has], FIELDS) == rec_bytes(best[has], FIELDS)
    assert np.all(best["feasible"][~has] == 0) and np.all(best["acc"][~has] == -1)
    assert (pos[33:36] == -1).all() and (pos[42:45] == 0).all()
    assert (pos[36:39] == 0).all() and (pos[39:42] == 0).all() and (pos[30:33] == 1).all()
    assert np.signbit(best["value"][39]) and not np.signbit(best["value"][36])


def test_oracle_zero_load_records_follow_the_override(wva, oracle):
    img = wva.synth.make_system(12, 3, seed=43, n_types=2)
    img.srv_arrival_rpm[:] = 0.0
    img.srv_min_replicas[:] = np.arange(12) % 2
    img.srv_keep_acc[:] = 0
    img.srv_max_batch[:] = 77                 # the server's own override is replaced
    img.perf_valid[:] = 1; img.srv_target_valid[:] = 1
    for b in (1, 3, 900, 8192):
        allocs, fe, _ = oracle.analyze_pairs(override(img, b))
        rep = np.repeat(img.srv_min_replicas, img.A)
        assert fe.all()
        assert (allocs.batch_size[rep == 1] == b).all() and (allocs.num_replicas[rep == 1] == 1).all()
        # minNumReplicas 0: the zero-replica record, whose batch is 0 whatever the override (allocation.go:262-267)
        assert (allocs.batch_size[rep == 0] == 0).all() and (allocs.acc[rep == 0] == -1).all()
