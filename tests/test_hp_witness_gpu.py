"""GPU: the device's outputs inside the high-precision witness's intervals (hp_witness.py), which stand apart from the
oracle every other GPU test compares with.

  * sweep cube, status bytes and winners in every set_certified_tails mode: a small image swept whole (in = 0 / out = 1
    and TPS-target servers, b = 1 .. 160 across the scan kernels' chunk edges), 500 random rows of config 3 at all 512
    batch sizes, every candidate grid_deferred lists and every server's winner;
  * the blocking plane (grid_blocking) and the winners' p_block (grid_best_blocking) on the same candidates;
  * wva_queue_analyze on random configurations (b log-uniform in 1 .. 8192, q in {0, 1, 10 b, random}, every in / out
    special case) and on the entries of tests/golden/hard_rounding.json;
  * wva_queue_size and the pair records: properties only (Size's bisection path turns on float32 comparisons an
    interval cannot settle).
The witness runs on host processes before and after the device calls; each test prints both times.
"""
import math
import time

import numpy as np
import pytest

import hp_witness as W
from test_hard_rounding_cpu import hex_f32, load_fixture
from test_hp_witness_cpu import (ERR_PAIR, cands, grid_ids, image_cands, image_feasible, queue_cfgs, rate_max,
                                 sweep_image, oracle_analyze)

pytestmark = pytest.mark.gpu
F = np.float32
MODES = (1, 33, 0, 3, 5, 9, 17)


def _pick(res, ids):
    return {k: v[ids] for k, v in res.items()}


def _check_candidates(what, res, c, img, s, r, metrics, status):
    """statuses where determined, metrics inside, feasible bits where the witness decides them -> counters"""
    usable = (status & 0xFE) != ERR_PAIR
    st = status & 0xFE
    bad = np.flatnonzero(usable & (st != res["status"]))
    assert len(bad) == 0, (what, "status", bad[:5], st[bad[:5]], res["status"][bad[:5]])
    w = res["witnessed"] & usable
    ins = W.inside(res, metrics.view(F).reshape(-1, 8))
    bad = np.flatnonzero(w & ~ins.all(axis=1))
    assert len(bad) == 0, (what, "metrics", bad[:5], [W.FIELDS[j] for j in np.flatnonzero(~ins[bad[0]])])
    fe = image_feasible(img, res, c, s, r)
    det = usable & (fe >= 0)
    bad = np.flatnonzero(det & (fe != (status & 1)))
    assert len(bad) == 0, (what, "feasible", bad[:5])
    single = W.singleton(res)[w].all(axis=1).sum()
    return dict(candidates=int(usable.sum()), witnessed=int(w.sum()),
                not_witnessed=int((usable & (res["status"] == W.OK) & ~res["witnessed"]).sum()),
                bit_determined=int(single), feasible_undetermined=int((usable & (fe < 0)).sum()))


def _check_winners(what, img, best, res_of, R, B, first=0):
    """each server's winner is feasible by the witness or undetermined"""
    n = 0
    for j, x in enumerate(best):
        if x["acc"] < 0:
            continue
        s = first + j
        cid = ((j * img.A + int(x["acc"])) * R + int(x["replicas"]) - 1) * B + int(x["batch"]) - 1
        res, c = res_of(cid)
        fe = image_feasible(img, res, c, np.array([s]), np.array([int(x["replicas"])]))
        assert fe[0] != 0, (what, s, x)
        n += 1
    return n


def _p_block_inside(what, res, p, ok):
    w = res["witnessed"] & ok
    assert np.isnan(p[~ok]).all(), what
    inside = (p[w] >= res["pb_lo"][w]) & (p[w] <= res["pb_hi"][w])
    assert inside.all(), (what, np.flatnonzero(w)[~inside][:5])
    return int(w.sum())


# ---- 1. a small image swept whole --------------------------------------------------------------------------------------

def test_sweep_small_image(wva, ctx):
    """16 x 3 x 16 x 160 whole, every mode: statuses, metrics, feasible bits, winners; the plane and the winners'
    p_block"""
    img = sweep_image(wva, S=16, A=3, seed=21)
    R, B = 16, 160
    s, a, r, b = grid_ids(img, R, B)
    c = image_cands(img, s, a, r, b)
    t0 = time.time()
    res = W.analyze(c)
    t_w = time.time() - t0
    t_dev = 0.0
    ctx.upload(img)
    try:
        for mode in MODES:
            ctx.set_certified_tails(mode)
            t0 = time.time()
            best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
            t_dev += time.time() - t0
            cnt = _check_candidates("small mode %d" % mode, res, c, img, s, r, cube, status)
            nw = _check_winners("small mode %d" % mode, img, best, lambda i: (_pick(res, [i]), c[[i]]), R, B)
            if mode == 1:
                t0 = time.time()
                p = ctx.grid_blocking()
                pb = ctx.grid_best_blocking()
                t_dev += time.time() - t0
                npb = _p_block_inside("small plane", res, p, status & 0xFE == W.OK)
                for j, x in enumerate(best):
                    if x["acc"] >= 0:
                        cid = ((j * img.A + int(x["acc"])) * R + int(x["replicas"]) - 1) * B + int(x["batch"]) - 1
                        if res["witnessed"][cid]:
                            assert res["pb_lo"][cid] <= pb[j] <= res["pb_hi"][cid], (j, x)
                print("small: %s, %d winners, %d p_block witnessed" % (cnt, nw, npb))
            assert nw > 0 and cnt["witnessed"] > 0.5 * cnt["candidates"]
    finally:
        ctx.set_certified_tails(1)
    print("small image: witness %.1f s, device %.1f s" % (t_w, t_dev))


# ---- 2. config 3: random rows, deferred candidates, winners ------------------------------------------------------------

def test_sweep_config3_rows(wva, ctx):
    """500 random rows (s, a, r) of a 40-server slice of config 3 at all 512 batch sizes, every candidate grid_deferred
    lists and every winner, in every mode; the plane and the winners' p_block"""
    img, cfg = wva.synth.baseline_config(3)
    R, B = cfg["r_max"], cfg["b_max"]
    first, count = 300, 40
    rng = np.random.default_rng(3)
    rows = rng.choice(count * img.A * R, 500, replace=False)
    row_ids = (rows[:, None] * B + np.arange(B)[None, :]).reshape(-1)
    per_mode, t_dev = {}, 0.0
    ctx.upload(img)
    try:
        ctx.set_shard(first, count)
        for mode in MODES:
            ctx.set_certified_tails(mode)
            t0 = time.time()
            best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
            deferred, n_def = ctx.grid_deferred()
            assert n_def == len(deferred)
            ids = np.unique(np.concatenate([row_ids, deferred.astype(np.int64)]))
            keep = dict(ids=ids, cube=cube[ids].copy(), status=status[ids].copy(), best=best.copy(), n_def=n_def)
            if mode == 1:
                keep["plane"] = ctx.grid_blocking()[ids].copy()
                keep["best_pb"] = ctx.grid_best_blocking()
            t_dev += time.time() - t0
            per_mode[mode] = keep
            del cube, status
    finally:
        ctx.set_certified_tails(1)
        ctx.set_shard(0, img.S)
    win_ids = []
    for k in per_mode.values():
        for j, x in enumerate(k["best"]):
            if x["acc"] >= 0:
                win_ids.append(((j * img.A + int(x["acc"])) * R + int(x["replicas"]) - 1) * B + int(x["batch"]) - 1)
    all_ids = np.unique(np.concatenate([k["ids"] for k in per_mode.values()] + [np.array(win_ids, np.int64)]))
    s, a, r, b = grid_ids(img, R, B, first, first + count)
    s, a, r, b = s[all_ids], a[all_ids], r[all_ids], b[all_ids]
    c = image_cands(img, s, a, r, b)
    t0 = time.time()
    res = W.analyze(c)
    t_w = time.time() - t0
    pos = {int(i): j for j, i in enumerate(all_ids)}
    for mode, k in per_mode.items():
        sel = np.array([pos[int(i)] for i in k["ids"]])
        cnt = _check_candidates("config 3 mode %d" % mode, _pick(res, sel), c[sel], img, s[sel], r[sel], k["cube"],
                                k["status"])
        nw = _check_winners("config 3 mode %d" % mode, img, k["best"],
                            lambda i: (_pick(res, [pos[i]]), c[[pos[i]]]), R, B, first)
        print("config 3 mode %d: %s, %d deferred, %d winners" % (mode, cnt, k["n_def"], nw))
        if mode == 1:
            st = k["status"] & 0xFE
            npb = _p_block_inside("config 3 plane", _pick(res, sel), k["plane"], st == W.OK)
            nbw = 0
            for j, x in enumerate(k["best"]):
                if x["acc"] >= 0:
                    cid = pos[((j * img.A + int(x["acc"])) * R + int(x["replicas"]) - 1) * B + int(x["batch"]) - 1]
                    if res["witnessed"][cid]:
                        assert res["pb_lo"][cid] <= k["best_pb"][j] <= res["pb_hi"][cid], (j, x)
                        nbw += 1
            print("config 3 plane: %d p_block witnessed, %d winners' p_block" % (npb, nbw))
            assert k["n_def"] > 0 and nw > 0
    print("config 3: %d candidates, witness %.1f s, device %.1f s" % (len(all_ids), t_w, t_dev))


# ---- 3. wva_queue_analyze ----------------------------------------------------------------------------------------------

def random_analyze_items(n, seed):
    rng = np.random.default_rng(seed)
    rows = []
    toks = [(0, 1), (0, 64), (512, 1), (128, 128), (2000, 200)]
    for _ in range(n):
        b = int(np.exp(rng.uniform(0, np.log(8192))))
        q = int(rng.choice([0, 1, 10 * b, int(rng.integers(0, 4 * b + 1))]))
        p = (F(rng.uniform(1, 30)), F(rng.uniform(0.001, 1)), F(rng.uniform(0, 250)), F(rng.uniform(0, 0.1)))
        tok = toks[int(rng.integers(0, len(toks)))] if rng.random() < 0.5 else \
            (int(rng.integers(0, 4000)), int(rng.integers(1, 1000)))
        rmax = rate_max(b, q, *p, *tok)
        x = rng.random()
        rate = rmax if x < 0.05 else F(float(rmax) * float(np.exp(rng.uniform(np.log(1e-5), 0))))
        rows.append((b, q) + p + tok + (rate,))
    return cands(rows)


def test_queue_analyze_random(wva, oracle, ctx):
    """2 000 random configurations through wva_queue_analyze: statuses and metrics inside the witness"""
    c = random_analyze_items(2000, 7)
    t0 = time.time()
    res = W.analyze(c)
    t_w = time.time() - t0
    t0 = time.time()
    m, st = ctx.queue_analyze(queue_cfgs(wva, c), c["rate"])
    t_dev = time.time() - t0
    assert (st == res["status"]).all(), np.flatnonzero(st != res["status"])[:5]
    w = res["witnessed"]
    ins = W.inside(res, m.view(F).reshape(-1, 8))
    assert ins[w].all(), np.flatnonzero(w & ~ins.all(axis=1))[:5]
    print("queue_analyze: %d items, %d witnessed, %d not witnessed, %d bit-determined; witness %.1f s, device %.2f s"
          % (len(c), w.sum(), ((st == W.OK) & ~w).sum(), W.singleton(res)[w].all(axis=1).sum(), t_w, t_dev))
    assert w.sum() > 0.8 * (st == W.OK).sum()


def test_queue_analyze_hard_rounding(wva, oracle, ctx):
    """the 340 entries of tests/golden/hard_rounding.json through wva_queue_analyze: inside the witness, and bit for bit
    equal to the oracle"""
    E = load_fixture()["entries"]
    rows = []
    for e in E:
        rate = F(F(F(hex_f32(e["arrival"])) / F(60)) / F(e["r"]))
        rows.append((e["b"], W.QUEUE_RATIO * e["b"], hex_f32(e["alpha"]), hex_f32(e["beta"]), hex_f32(e["gamma"]),
                     hex_f32(e["delta"]), e["in"], e["out"], rate))
    c = cands(rows)
    t0 = time.time()
    res = W.analyze(c)
    t_w = time.time() - t0
    t0 = time.time()
    m, st = ctx.queue_analyze(queue_cfgs(wva, c), c["rate"])
    t_dev = time.time() - t0
    om, ost = oracle_analyze(wva, oracle, c)
    assert np.array_equal(st, ost) and (st == res["status"]).all()
    mm = m.view(F).reshape(-1, 8)
    assert mm.view(np.uint32).tobytes() == om.view(np.uint32).tobytes()
    w = res["witnessed"]
    assert W.inside(res, mm)[w].all()
    print("hard_rounding: %d entries, %d witnessed, %d not witnessed, %d bit-determined; witness %.1f s, device %.2f s"
          % (len(c), w.sum(), ((st == W.OK) & ~w).sum(), W.singleton(res)[w].all(axis=1).sum(), t_w, t_dev))
    assert w.sum() >= 300


# ---- 4. wva_queue_size and the pair records ----------------------------------------------------------------------------

def test_queue_size_properties(wva, ctx):
    """Size's metrics inside the witness at the rate it analysed (min of the three target rates), achieved values
    from those metrics, every rate <= RateRange.Max"""
    c = random_analyze_items(1500, 11)
    c = c[c["b"] + c["q"] >= 2]
    rng = np.random.default_rng(12)
    n = len(c)
    ttft0 = c["gamma"] + c["delta"] * c["in"]
    itl0 = c["alpha"] + c["beta"]
    combo = rng.integers(0, 8, n)
    t = np.zeros((n, 3), F)
    t[:, 0] = np.where(combo & 1, ttft0 * np.exp(rng.uniform(-1, 4, n)), 0)
    t[:, 1] = np.where(combo & 2, itl0 * np.exp(rng.uniform(-0.5, 3, n)), 0)
    t[:, 2] = np.where(combo & 4, rng.uniform(1, 5000, n), 0)
    t0 = time.time()
    rates, m, ach, st = ctx.queue_size(queue_cfgs(wva, c), t)
    t_dev = time.time() - t0
    ok = st == 0
    rmax = np.array([rate_max(int(x["b"]), int(x["q"]), x["alpha"], x["beta"], x["gamma"], x["delta"], int(x["in"]),
                              int(x["out"])) for x in c], F)
    assert (rates[ok] <= rmax[ok, None]).all()
    mm = m.view(F).reshape(-1, 8)
    with np.errstate(all="ignore"):
        assert (ach[ok, 0].view(np.uint32) == (mm[ok, 2] + mm[ok, 4]).view(np.uint32)).all()
        assert (ach[ok, 1].view(np.uint32) == mm[ok, 5].view(np.uint32)).all()
        assert (ach[ok, 2].view(np.uint32) == (mm[ok, 0] * c["out"][ok].astype(F)).view(np.uint32)).all()
    at = c[ok].copy()
    at["rate"] = rates[ok].min(axis=1)
    t0 = time.time()
    res = W.analyze(at)
    t_w = time.time() - t0
    assert (res["status"] == W.OK).all()
    w = res["witnessed"]
    assert W.inside(res, mm[ok])[w].all(), np.flatnonzero(w & ~W.inside(res, mm[ok]).all(axis=1))[:5]
    print("queue_size: %d items, %d sized, %d witnessed, %d bit-determined; witness %.1f s, device %.2f s" % (
        n, ok.sum(), w.sum(), W.singleton(res)[w].all(axis=1).sum(), t_w, t_dev))
    assert ok.sum() > 0.2 * n and w.sum() > 0.8 * ok.sum()


def test_pair_records_properties(wva, ctx):
    """each feasible pair record: rateStar (Size's throughput on the pair's queue) gives max_arrv_rate_per_replica and
    numReplicas = max(ceil(f64(totalRate) / f64(rateStar)), minReplicas); its ITL, TTFT and rho lie inside the witness
    of Analyze(totalRate / numReplicas)"""
    img = wva.synth.make_system(80, 4, seed=31, n_types=2)
    ctx.upload(img)
    t0 = time.time()
    rec, feas = ctx.analyze_pairs()
    t_dev = time.time() - t0
    A = img.A
    rows, targets, meta = [], [], []
    for i in np.flatnonzero(feas):
        s, a = divmod(int(i), A)
        if img.srv_arrival_rpm[s] == 0 or img.srv_out_tokens[s] == 0:
            continue
        pi = int(img.srv_model[s]) * A + a
        N = int(rec.batch_size[i])
        rows.append((N, W.QUEUE_RATIO * N, img.perf_alpha[pi], img.perf_beta[pi], img.perf_gamma[pi], img.perf_delta[pi],
                     int(img.srv_in_tokens[s]), int(img.srv_out_tokens[s]), F(0)))
        targets.append((img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s]))
        meta.append((int(i), s))
    c = cands(rows)
    t0 = time.time()
    _, sm, _, sst = ctx.queue_size(queue_cfgs(wva, c), np.array(targets, F))
    t_dev += time.time() - t0
    assert (sst == 0).all()
    rate_star = sm["throughput"]
    for j, (i, s) in enumerate(meta):
        out = int(img.srv_out_tokens[s])
        total = F(img.srv_arrival_rpm[s]) / F(60) if img.srv_slo_tps[s] == 0 else F(img.srv_slo_tps[s]) / F(out)
        n_rep = max(int(math.ceil(float(total) / float(rate_star[j]))), int(img.srv_min_replicas[s]))
        assert rec.num_replicas[i] == n_rep, (i, rec.num_replicas[i], n_rep)
        assert rec.max_arrv_rate_per_replica[i] == F(rate_star[j] / F(1000)), i
        c["rate"][j] = F(total / F(n_rep))
    t0 = time.time()
    res = W.analyze(c)
    t_w = time.time() - t0
    assert (res["status"] == W.OK).all()
    w = res["witnessed"]
    idx = np.array([i for i, _ in meta])
    lo, hi = res["lo"], res["hi"]
    itl = rec.itl[idx]
    ttft_lo, ttft_hi = lo[:, 2] + lo[:, 4], hi[:, 2] + hi[:, 4]          # float32 addition is monotone
    ttft = rec.ttft[idx]
    assert ((itl >= lo[:, 5]) & (itl <= hi[:, 5]))[w].all()
    assert ((ttft >= ttft_lo) & (ttft <= ttft_hi))[w].all()
    assert ((rec.rho[idx] >= lo[:, 7]) & (rec.rho[idx] <= hi[:, 7]))[w].all()
    print("pair records: %d feasible with load, %d witnessed; witness %.1f s, device %.2f s" % (len(c), w.sum(), t_w,
                                                                                                 t_dev))
    assert len(c) > 100 and w.sum() > 0.9 * len(c)
