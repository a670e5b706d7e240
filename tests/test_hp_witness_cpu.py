"""The high-precision witness (hp_witness.py) against the oracle, without a GPU: every oracle output lies inside the
witness's intervals and every status equals its prediction, on fixtures that reach the branches a shared misreading
of the reference would hide in; the share of bit-exact (one-float) intervals, with floors; and seven one-line
mutants of the witness, each of which must reject the unmodified oracle.  The fixtures and the helpers are shared
with test_hp_witness_gpu.py."""
import importlib
import os
import sys
import time

import numpy as np
import pytest

import hp_witness as W

F = np.float32
PROFILES = [            # (alpha, beta, gamma, delta)
    (7.470, 0.044, 15.415, 0.000337),
    (20.0, 0.5, 100.0, 0.02),
    (3.0, 0.05, 40.0, 0.004),
    (12.0, 0.2, 5.0, 0.0005),
]
TOKENS = [(128, 128), (2000, 200), (0, 1), (0, 64), (512, 1), (64, 16)]
EDGE_B = (1, 31, 32, 33, 63, 65)
ERR_PAIR = 2                       # WVA_CAND_ERR_PAIR: the pair lookups fail (a pair rule, not Analyze's)
LOADS = (1e-4, 0.01, 0.1, 0.5, 0.9, 0.99)            # fractions of RateRange.Max; 1 (r = 0.999) is added below


def rate_max(b, q, al, be, ga, de, inn, out):
    return W.rate_range(W.rate_table(al, be, ga, de, inn, out, b), b)[1]


def cands(rows):
    """a CAND_DTYPE array from (b, q, alpha, beta, gamma, delta, in, out, rate) tuples"""
    out = np.zeros(len(rows), W.CAND_DTYPE)
    for i, r in enumerate(rows):
        out[i] = r
    return out


def _loads(row, loads, top=True):
    """the row at each load fraction of RateRange.Max, and at Max itself and one float below (r = 0.999)"""
    rmax = rate_max(*row)
    rates = [F(float(rmax) * x) for x in loads]
    if top:
        rates += [rmax, np.nextafter(rmax, F(0))]
    return [row + (r,) for r in rates]


def fixture(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    rows = []
    if name == "chunk_edges":                     # b at the scan kernels' chunk edges, q = 0, 1, 10 b
        for b in EDGE_B:
            for q in (0, 1, 10 * b):
                for p in PROFILES[:3]:
                    for inn, out in TOKENS[:3]:
                        rows += _loads((b, q) + p + (inn, out), LOADS)
    elif name == "tokens":                        # in = 0 / out = 1, in = 0, out = 1 with in > 0
        for b in (1, 2, 8, 64, 512):
            for q in (0, 10 * b):
                for p in PROFILES:
                    for inn, out in TOKENS[2:5]:
                        rows += _loads((b, q) + p + (inn, out), LOADS)
    elif name == "die_out":                       # light loads on large b: the chain dies out long before N
        for b in (256, 512, 2048):
            for p in PROFILES:
                for inn, out in TOKENS[:2]:
                    rows += _loads((b, 10 * b) + p + (inn, out), (1e-5, 1e-3, 0.01, 0.05), top=False)
    elif name == "large_b":                       # b up to 8192
        for b in (1024, 4096, 8192):
            for q in (0, 1, 10 * b):
                for p in PROFILES[:2]:
                    rows += _loads((b, q) + p + (128, 128), (0.01, 0.5), top=True)
    elif name == "random":                        # test_size_fuzz's ranges
        for _ in range(400):
            b = int(np.exp(rng.uniform(0, np.log(2048))))
            q = int(rng.choice([0, 1, 3 * b, 10 * b, int(rng.integers(0, 4 * b + 1))]))
            p = (F(rng.uniform(1, 30)), F(rng.uniform(0.001, 1)), F(rng.uniform(0, 250)), F(rng.uniform(0, 0.1)))
            tok = (int(rng.integers(0, 4000)), int(rng.integers(1, 1000)))
            rows += _loads((b, q) + p + tok, (float(np.exp(rng.uniform(np.log(1e-4), 0))),), top=False)
    elif name == "statuses":                      # every error status, and K = 1
        for p in PROFILES[:2]:
            for inn, out in TOKENS[:3]:
                row = (8, 80) + p + (inn, out)
                rmax = rate_max(*row)
                rows += [row + (F(0),), row + (F(-1),), row + (np.nextafter(rmax, F(np.inf)),), row + (F(3e38),)]
                rows += [(0, 0) + p + (inn, out, F(1)), (4, -1) + p + (inn, out, F(1)), (4, 4) + p + (-1, out, F(1)),
                         (4, 4) + p + (inn, 0, F(1))]
                rows += _loads((1, 0) + p + (inn, out), (0.5,))
    return cands(rows)


FIXTURES = ("chunk_edges", "tokens", "die_out", "large_b", "random", "statuses")


# ---- the oracle's side -----------------------------------------------------------------------------------------------

def queue_cfgs(wva, c):
    q = np.zeros(len(c), wva.abi.QUEUE_CONFIG_DTYPE)
    for k in ("alpha", "beta", "gamma", "delta"):
        q[k] = c[k]
    q["max_batch_size"], q["max_queue_size"] = c["b"], c["q"]
    q["avg_input_tokens"], q["avg_output_tokens"] = c["in"], c["out"]
    return q


def oracle_analyze(wva, oracle, c):
    m, st = oracle.queue_analyze(queue_cfgs(wva, c), c["rate"], threads=max(1, oracle.hardware_threads()))
    return m.view(F).reshape(len(c), 8), st


def oracle_p_block(oracle, c, idx):
    """float32 of the oracle's normalised p[K] after Analyze on a fresh analyzer"""
    out = np.full(len(c), np.nan, F)
    for i in idx:
        x = c[i]
        a = oracle.Analyzer(int(x["b"]), int(x["q"]), x["alpha"], x["beta"], x["gamma"], x["delta"], int(x["in"]),
                            int(x["out"]))
        st, _ = a.analyze(F(x["rate"]))
        assert st == W.OK
        out[i] = F(a.probabilities()[int(x["b"] + x["q"])])
    return out


def image_cands(img, s, a, r, b):
    """the sweep's candidates (s, a, r, b) of an image as witness inputs: NewQueueAnalyzer({b, 10 b}) and
    Analyze(totalRate / r)"""
    A = img.A
    pi = img.srv_model[s] * A + a
    c = np.zeros(len(s), W.CAND_DTYPE)
    c["b"], c["q"] = b, W.QUEUE_RATIO * np.asarray(b)
    c["alpha"], c["beta"] = img.perf_alpha[pi], img.perf_beta[pi]
    c["gamma"], c["delta"] = img.perf_gamma[pi], img.perf_delta[pi]
    c["in"], c["out"] = img.srv_in_tokens[s], img.srv_out_tokens[s]
    c["rate"] = [W.sweep_rate(img.srv_arrival_rpm[si], img.srv_slo_tps[si], img.srv_out_tokens[si], ri)
                 for si, ri in zip(s, r)]
    return c


def image_feasible(img, res, c, s, r):
    return W.feasible(res, img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s], c["rate"], r,
                      img.srv_min_replicas[s])


def check(res, metrics, status, p_block=None, what=""):
    """statuses equal; every witnessed candidate's metrics (and p_block) inside its intervals"""
    bad = np.flatnonzero(res["status"] != status)
    assert len(bad) == 0, (what, "status", bad[:5], res["status"][bad[:5]], status[bad[:5]])
    w = res["witnessed"]
    ins = W.inside(res, metrics)
    bad = np.flatnonzero(w & ~ins.all(axis=1))
    assert len(bad) == 0, (what, "metrics", bad[:5], [W.FIELDS[j] for j in np.flatnonzero(~ins[bad[0]])])
    if p_block is not None:
        pb = p_block[w]
        ok = (pb >= res["pb_lo"][w]) & (pb <= res["pb_hi"][w])
        assert ok.all(), (what, "p_block", np.flatnonzero(w)[~ok][:5])
    return int(w.sum())


def fractions(res):
    w = res["witnessed"]
    return W.singleton(res)[w].mean(axis=0) if w.any() else np.zeros(9)


def report(what, res, t):
    fr = fractions(res)
    print("%s: %d candidates, %d witnessed, %d not witnessed (status OK), witness %.1f s; singleton %%: %s" % (
        what, len(res["status"]), res["witnessed"].sum(), ((res["status"] == W.OK) & ~res["witnessed"]).sum(), t,
        " ".join("%s %.1f" % (k, 100 * v) for k, v in zip(W.FIELDS + ("p_block",), fr))))
    return fr


# the singleton floors of each fixture, set from a run of these tests (percent; fields of AnalysisMetrics, p_block)
FLOORS = {
    "chunk_edges": (100, 100, 98, 97, 98, 98, 100, 97, 100),
    "tokens": (100, 100, 96, 95, 98, 98, 100, 95, 100),
    "die_out": (100, 100, 45, 38, 42, 40, 100, 38, 100),
    "large_b": (100, 100, 88, 80, 82, 84, 100, 80, 100),
    "random": (100, 100, 88, 85, 85, 88, 100, 85, 100),
    "statuses": (0,) * 9,                       # error statuses and K = 1 only: nothing to witness
}


@pytest.fixture(scope="module")
def fixtures():
    return {name: fixture(name) for name in FIXTURES}


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_inside_witness(wva, oracle, fixtures, name):
    """every oracle status equals the witness's, every metric and p_block lies inside its interval, and the share of
    one-float intervals is at its floor"""
    c = fixtures[name]
    t0 = time.time()
    res = W.analyze(c)
    t = time.time() - t0
    m, st = oracle_analyze(wva, oracle, c)
    pb = oracle_p_block(oracle, c, np.flatnonzero(res["witnessed"]))
    n = check(res, m, st, pb, name)
    assert n >= 0.8 * (st == W.OK).sum(), name
    fr = report(name, res, t)
    floor = np.array(FLOORS[name], float) / 100
    assert (fr >= floor).all(), (name, fr)


def test_fixtures_reach_branches(fixtures):
    """q = 0 (K = N, no tail), in = 0 / out = 1 (numDecode = 1), out = 1 with in > 0 (numDecode = 0), r = 0.999 (a rate
    at RateRange.Max), chains that die out, b = 1, 31, 32, 33, 63, 65, b up to 8192, every status"""
    allc = np.concatenate([fixtures[n] for n in FIXTURES])
    res = W.analyze(allc)
    w = res["witnessed"]
    assert (w & (allc["q"] == 0) & (allc["b"] > 1)).any()
    assert (w & (allc["in"] == 0) & (allc["out"] == 1)).any()
    assert (w & (allc["in"] > 0) & (allc["out"] == 1)).any()
    at_max = np.array([bool(w[i]) and x["rate"] == rate_max(int(x["b"]), int(x["q"]), x["alpha"], x["beta"],
                                                            x["gamma"], x["delta"], int(x["in"]), int(x["out"]))
                       for i, x in enumerate(allc)])
    assert (w & at_max).sum() >= 100
    for b in EDGE_B + (8192,):
        assert (w & (allc["b"] == b)).any(), b
    assert set(np.unique(res["status"])) == {W.OK, W.ERR_CONFIG, W.ERR_RATE_LE0, W.ERR_RATE_MAX, W.ERR_MODEL}
    # died out: at least 99.99 % of the mass below b / 8 requests in service
    d = fixtures["die_out"]
    rd = W.analyze(d)
    assert (rd["witnessed"] & (rd["hi"][:, 3] < d["b"] / 8)).sum() >= 50


def test_sweep_image_inside_witness(wva, oracle):
    """a small sweep image whole (in = 0 / out = 1 and TPS-target servers among them): statuses, metrics and the
    feasible bits the witness determines, against the oracle's sweep"""
    img = sweep_image(wva)
    R, B = 4, 70
    best, cube, status, _ = oracle.analyze_grid(img, R, B, threads=max(1, oracle.hardware_threads()))
    s, a, r, b = grid_ids(img, R, B)
    c = image_cands(img, s, a, r, b)
    usable = (status & 0xFE) != ERR_PAIR
    res = W.analyze(c[usable])
    check(res, cube.view(F).reshape(-1, 8)[usable], status[usable] & 0xFE, what="sweep")
    fe = image_feasible(img, res, c[usable], s[usable], r[usable])
    got = status[usable] & 1
    det = fe >= 0
    assert (fe[det] == got[det]).all()
    assert det.mean() > 0.99 and (fe == 1).any()
    report("sweep image", res, 0)


def sweep_image(wva, S=12, A=3, seed=5):
    img = wva.synth.make_system(S, A, seed=seed, n_types=2)
    img.perf_valid[:] = 1
    img.srv_target_valid[:] = 1
    img.srv_arrival_rpm[img.srv_arrival_rpm == 0] = F(900)
    img.srv_in_tokens[0], img.srv_out_tokens[0] = 0, 1
    img.srv_in_tokens[1] = 0
    img.srv_out_tokens[2] = 1
    img.srv_slo_tps[3] = F(800)
    img.srv_slo_tps[4] = F(60)
    return img


def grid_ids(img, R, B, s0=0, s1=None):
    s1 = img.S if s1 is None else s1
    idx = np.arange((s1 - s0) * img.A * R * B)
    b = (idx % B + 1).astype(np.int32)
    r = ((idx // B) % R + 1).astype(np.int32)
    a = ((idx // (B * R)) % img.A).astype(np.int32)
    s = (idx // (B * R * img.A) + s0).astype(np.int32)
    return s, a, r, b


# ---- mutants ---------------------------------------------------------------------------------------------------------

MUTANTS = {   # name -> (line of hp_witness.py, its replacement)
    "i_eq_num_minus_1": ("        split = N ", "        split = N - 1 "),
    "no_decode_only_rule": ("nd = 1 if (inn == 0 and out == 1) else out - 1", "nd = out - 1"),
    "tail_at_servRate_N": ("        rho = ratio[N - 1] ", "        rho = ratio[N] "),
    "K_minus_1": ("    return q + b\n", "    return q + b - 1\n"),
    "lambda_float64": ("        lam32 = F(F(rate) / F(1000))", "        lam32 = np.float64(rate) / 1000.0"),
    "no_wait_clamp": ("    wait = _wait_clamp(_op(lambda x, y: x - y, resp, serv))", "    wait = _op(lambda x, y: x - y, resp, serv)"),
    "throughput_without_1000": ("    thr1000 = _op(lambda x: x * F(1000), thr)", "    thr1000 = thr"),
}


def load_mutant(name, where):
    """a copy of hp_witness.py with one line changed, importable by worker processes"""
    old, new = MUTANTS[name]
    src = open(W.__file__).read()
    assert src.count(old) == 1, name
    mod = "hp_witness_" + name
    with open(os.path.join(where, mod + ".py"), "w") as f:
        f.write(src.replace(old, new))
    if where not in sys.path:
        sys.path.insert(0, where)
    return importlib.import_module(mod)


def mutant_fixture():
    """the inputs each mutant is run on: the branch fixtures (without the b > 2048 rows) and the error statuses"""
    c = np.concatenate([fixture(n) for n in ("chunk_edges", "tokens", "statuses")])
    return c


def rejects(M, wva, oracle, c):
    """how the mutant's witness rejects the oracle: (status mismatches, metric fields outside, p_block outside)"""
    res = M.analyze(c)
    m, st = oracle_analyze(wva, oracle, c)
    n_st = int((res["status"] != st).sum())
    w = res["witnessed"] & (st == W.OK)
    outside = (~M.inside(res, m))[w].sum(axis=0)
    pb = oracle_p_block(oracle, c, np.flatnonzero(w))[w]
    n_pb = int((~((pb >= res["pb_lo"][w]) & (pb <= res["pb_hi"][w]))).sum())
    return n_st, outside, n_pb


# Mutants the oracle still satisfies, and why: each changes the float64 rounding of the reference's loop but not the
# real number it computes, and the witness bounds that rounding instead of predicting it.
WEAK = {
    # sum_{i<=N-1} i p_i + N (1 - sum_{i<=N-1} p_i) = sum_{i<=N} i p_i + N (1 - sum_{i<=N} p_i): the term i = N is N p_N
    # either way, so both readings of mm1modelstatedependent.go:52 give the same inServ
    "i_eq_num_minus_1",
    # inSys >= inServ exactly (sum i p_i >= sum min(i, N) p_i), so resp - serv < 0 comes from rounding alone, and
    # only where inSys = inServ exactly (q = 0, or a tail of zero mass) -- there the interval of resp - serv holds 0
    "no_wait_clamp",
}


@pytest.mark.parametrize("name", sorted(set(MUTANTS) - WEAK))
def test_mutant_rejects_oracle(wva, oracle, tmp_path, name):
    """each one-line mutant of the witness rejects the unmodified oracle on the fixtures"""
    M = load_mutant(name, str(tmp_path))
    c = mutant_fixture()
    n_st, outside, n_pb = rejects(M, wva, oracle, c)
    print("%s: %d statuses differ; outside per field %s; p_block outside %d" % (
        name, n_st, dict(zip(W.FIELDS, outside.tolist())), n_pb))
    assert n_st + outside.sum() + n_pb > 0, name


@pytest.mark.parametrize("name", sorted(WEAK))
def test_weak_mutant_moves_rounding_only(wva, oracle, tmp_path, name):
    """a weak mutant's intervals overlap the witness's own on every candidate: what it changes lies inside the
    rounding the witness bounds (see WEAK)"""
    M = load_mutant(name, str(tmp_path))
    c = mutant_fixture()
    res, mres = W.analyze(c), M.analyze(c)
    assert (res["status"] == mres["status"]).all()
    w = res["witnessed"] & mres["witnessed"]
    assert w.sum() > 0.9 * res["witnessed"].sum()
    assert ((mres["lo"][w] <= res["hi"][w]) & (res["lo"][w] <= mres["hi"][w])).all(), name
    n_st, outside, n_pb = rejects(M, wva, oracle, c)
    print("%s (weak): %d statuses differ, %d fields outside, %d p_block outside" % (name, n_st, outside.sum(), n_pb))
