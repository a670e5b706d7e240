"""Inputs for the tests of the public analyzer API (wva_queue_analyze, wva_queue_size, wva_model_solve) and the
restatements that classify them.  Seeded and deterministic; shared by test_analyzer_api_cpu.py (which shows that every
fixture reaches its branch and that the oracle terminates on it) and test_analyzer_api_gpu.py (which compares the
device with the oracle on them).

  target edges   Size / BinarySearch targets derived from the oracle's own evaluations at lambdaMin and lambdaMax,
                 stepped with nextafter across the 1e-6 tolerance band (utils.go:12-20, 26-70)
  fault items    the overflow profile (beta = 1e-4, delta = 1e-7, b = 900 .. 3000, loads near RateRange.Max): chains
                 that overflow float64 and take the rescale of mm1modelstatedependent.go:84-89 on the materialised path
  model fixtures bare MM1ModelStateDependent inputs that take the chain rescale (:84-89) only, the sum rescale
                 (:95-104) only, both, and repeated rescales that flush p[0] to 0
  classifier     the inputs on which the reference never returns: a service rate of 0 or NaN reached by the chain, a
                 lambda of NaN or +Inf on a valid call, and what makes Analyze and Size run such a chain
  witness        the birth-death solution in mpmath from the float32 rates and lambda as exact values
"""
import numpy as np

import wva_import

abi = wva_import.load().abi
F = np.float32
TOL = F(1e-6)                 # utils.go:8
EPS = F(0.001)                # queueanalyzer.go:8
SAFETY = F(0.1)               # queueanalyzer.go:11
KINDS = (0, 1)                # EvalTTFT, EvalITL


# ---- float32 restatements ----------------------------------------------------------------------------------------------

def cfgs(rows):
    """a QUEUE_CONFIG_DTYPE array from (b, queue, alpha, beta, gamma, delta, in, out) tuples"""
    out = np.zeros(len(rows), dtype=abi.QUEUE_CONFIG_DTYPE)
    for i, (b, q, al, be, ga, de, inn, o) in enumerate(rows):
        out[i] = (b, q, al, be, ga, de, inn, o)
    return out


def config_ok(c):
    """Configuration.check + RequestSize.check (queueanalyzer.go:337-352)"""
    return not (c["max_batch_size"] <= 0 or c["max_queue_size"] < 0 or c["avg_input_tokens"] < 0
                or c["avg_output_tokens"] < 1)


def cfg_rate_table(c):
    """servRate[0 .. N-1] of BuildModel (queueanalyzer.go:102-113) in its operation order"""
    N, inn, out = int(c["max_batch_size"]), int(c["avg_input_tokens"]), int(c["avg_output_tokens"])
    al, be, ga, de = (F(c[k]) for k in ("alpha", "beta", "gamma", "delta"))
    fn = np.arange(1, N + 1, dtype=F)
    with np.errstate(all="ignore"):
        pre = np.zeros(N, F) if inn == 0 else ga + (de * F(inn)) * fn
        nd = 1 if (inn == 0 and out == 1) else out - 1
        dec = F(nd) * (al + be * fn)
        return fn / (pre + dec)


def lambda_range(c):
    """(lambdaMin, lambdaMax) of Size: RateRange / 1000 (queueanalyzer.go:116-118, 192-193)"""
    tab = cfg_rate_table(c)
    with np.errstate(all="ignore"):
        rmin = (tab[0] * EPS) * F(1000)
        rmax = (tab[-1] * (F(1) - EPS)) * F(1000)
        return rmin / F(1000), rmax / F(1000), rmax


def _bad_table(tab):
    return bool(((tab == 0) | np.isnan(tab)).any())


def chain_hangs(tab, lam):
    """computeProbabilities (mm1modelstatedependent.go:77-90) never returns: a reached rate of 0 or NaN makes p[n+1]
    Inf or NaN for any p[n] (0/0 once rescaling has flushed p[n]); lambda NaN or +Inf does the same (0 * Inf).  A
    negative rate ends after a few rescales with p[n+1] = -0.  The chain of K >= N states reaches every entry."""
    lam = F(lam)
    return _bad_table(tab) or bool(np.isnan(lam) or np.isinf(lam))


def analyze_hangs(c, rate):
    """QueueAnalyzer.Analyze(rate) on a fresh analyzer runs a chain that never ends"""
    if not config_ok(c):
        return False
    rate = F(rate)
    _, _, rmax = lambda_range(c)
    if rate <= 0 or rate > rmax:
        return False
    if int(c["max_batch_size"]) + int(c["max_queue_size"]) < 2:      # fresh rho = 1 >= K: the model is invalid
        return False
    with np.errstate(all="ignore"):
        return chain_hangs(cfg_rate_table(c), rate / F(1000))


def size_hangs(c, t, y_at_min=None):
    """QueueAnalyzer.Size(targets t) runs a chain that never ends.  y_at_min(kind) gives EvalTTFT / EvalITL at
    lambdaMin (finite there; only asked for when lambdaMax is not finite and the table is good): a search whose value
    at lambdaMin is within tolerance returns before it evaluates lambdaMax."""
    if not config_ok(c):
        return False
    t = [F(x) for x in t]
    if any(x < 0 for x in t):
        return False
    if int(c["max_batch_size"]) + int(c["max_queue_size"]) < 2:
        return False
    tab = cfg_rate_table(c)
    lmin, lmax, rmax = lambda_range(c)
    searches = [k for k in KINDS if t[k] > 0]
    if _bad_table(tab):                                              # the first chain hangs, if one runs
        if searches:
            return not (lmin > lmax)
        with np.errstate(all="ignore"):
            lam = lmax if not t[2] > 0 else np.minimum(lmax, lmax * (F(1) - SAFETY))
            rate = lam * F(1000)
        return not (rate <= 0 or rate > rmax)
    if np.isfinite(lmax):
        return False                                                 # every lambda evaluated is finite
    for k in searches:                                               # xMin <= NaN / +Inf is never rejected
        if not np.isfinite(lmin):
            return True
        if not within_tolerance(y_at_min(k), t[k]):
            return True
    return not searches                                              # only lambdaMin was used, or lambdaMax itself


def within_tolerance(x, v, tol=TOL):
    """WithinTolerance (utils.go:12-20)"""
    x, v = F(x), F(v)
    if x == v:
        return True
    if v == 0 or tol < 0:
        return False
    with np.errstate(all="ignore"):
        q = (x - v) / v
    return bool(abs(float(q)) <= float(tol))


def model_call_hangs(K, serv, lam, mu, p0):
    """MM1ModelStateDependent.Solve(lam, mu) on a model whose last p[0] is p0 never returns"""
    rho = F(1) - F(p0)
    if rho < 0 or rho >= F(K) or F(lam) < 0 or F(mu) <= 0:
        return False                                                 # invalid: nothing is computed
    if K == 0:
        return False
    serv = np.asarray(serv, F)
    reached = serv[:min(len(serv), K)]
    return chain_hangs(reached, lam)


# ---- target edges ------------------------------------------------------------------------------------------------------

def step_out(y, direction):
    """the last float32 target within tolerance of y stepping from y towards `direction` and the first one outside"""
    t = F(y)
    while True:
        nxt = np.nextafter(t, F(direction))
        if not within_tolerance(y, nxt):
            return t, nxt
        t = nxt


EDGE_PROFILES = [        # (alpha, beta, gamma, delta, in, out): TTFT and ITL strictly increasing in lambda
    (7.470, 0.044, 15.415, 0.000337, 128, 128),
    (20.0, 0.5, 100.0, 0.02, 512, 64),
    (3.0, 0.05, 40.0, 0.004, 2000, 200),
    (12.0, 0.2, 5.0, 0.0005, 64, 16),
]
EDGE_BATCHES = [(2, 0), (8, 80), (48, 480), (200, 2000)]
EDGE_CLASSES = ("at_min", "in_min", "out_min", "at_max", "in_max", "out_max", "inside", "nan", "inf")


def edge_targets(oracle, c):
    """{(kind, class): target} for one config; the outcomes BinarySearch must report are in EDGE_OUTCOME"""
    a = oracle.Analyzer(*[c[k] for k in ("max_batch_size", "max_queue_size", "alpha", "beta", "gamma", "delta",
                                         "avg_input_tokens", "avg_output_tokens")])
    lmin, lmax, _ = lambda_range(c)
    out = {}
    for k in KINDS:
        y0, y1 = a.eval(k, lmin), a.eval(k, lmax)
        assert y0 is not None and y1 is not None and y0 < y1 and not within_tolerance(y1, y0)
        in_min, out_min = step_out(y0, -np.inf)
        in_max, out_max = step_out(y1, np.inf)
        out.update({(k, "at_min"): y0, (k, "in_min"): in_min, (k, "out_min"): out_min,
                    (k, "at_max"): y1, (k, "in_max"): in_max, (k, "out_max"): out_max,
                    (k, "inside"): F(np.sqrt(float(y0) * float(y1))), (k, "nan"): F(np.nan), (k, "inf"): F(np.inf)})
    return out


EDGE_OUTCOME = {          # class -> (x, ind) of BinarySearch; "mid": strictly inside; "nan": nan_search_x
    "at_min": ("min", 0), "in_min": ("min", 0), "out_min": ("min", -1),
    "at_max": ("max", 0), "in_max": ("max", 0), "out_max": ("max", +1),
    "inside": ("mid", 0), "nan": ("nan", 0), "inf": ("max", +1),
}


def nan_search_x(lmin, lmax):
    """the x a NaN target ends on: no test is ever true, so xMin moves to the midpoint 100 times"""
    lo, hi = F(lmin), F(lmax)
    x = F(0)
    for _ in range(100):
        x = F(0.5) * (lo + hi)
        lo = x
    return x


# (alpha, target) with float32((alpha - target) / target) = +-1e-6 exactly: WithinTolerance's `<=` decides.  With
# beta = 0 EvalITL is alpha at every lambda, so an ITL search for the target returns lambdaMin (ind 0); a strict `<`
# would give ind -1 (target above) or +1 (below).
TOL_EDGE = [(9.536733627319336, 9.5367431640625), (9.536752700805664, 9.5367431640625),
            (11.444080352783203, 11.444091796875), (11.444103240966797, 11.444091796875)]


def tol_edge_cfg(alpha):
    return (48, 480, alpha, 0.0, 40.0, 0.004, 2000, 200)


BUDGET_CFG = (512, 5120, 7.470, 0.044, 15.415, 0.000337, 128, 128)   # test_pairs_iteration_budget's pair
BUDGET_TARGETS = (1000.0, 10.0, 0.0)     # the TTFT search never meets the tolerance: all 100 iterations


def edge_outcome_ok(cls, x, ind, lmin, lmax):
    want_x, want_ind = EDGE_OUTCOME[cls]
    if ind != want_ind:
        return False
    return {"min": x == lmin, "max": x == lmax, "mid": lmin < x < lmax, "nan": x == nan_search_x(lmin, lmax)}[want_x]


# ---- fault items (chains that overflow float64 under Analyze / Size) ---------------------------------------------------

OVERFLOW = dict(alpha=20.0, beta=1e-4, gamma=10.0, delta=1e-7, in_tok=64, out_tok=8)


def overflow_cfg(b, q):
    o = OVERFLOW
    return (b, q, o["alpha"], o["beta"], o["gamma"], o["delta"], o["in_tok"], o["out_tok"])


def overflow_rate(c, frac):
    """a request rate (req/s) at frac * RateRange.Max"""
    _, _, rmax = lambda_range(c)
    return F(float(rmax) * frac)


TAME = (20.0, 0.5, 100.0, 0.02, 512, 64)


def tame_cfg(b, q):
    return (b, q) + TAME


# ---- bare-model fixtures -----------------------------------------------------------------------------------------------
# name -> (K, service rates, lambda); what each one does in the oracle is asserted by test_analyzer_api_cpu.py

MODEL_FIXTURES = {
    "chain_only": (40, [1e-37] * 5 + [1e38], 1e37),                   # p[5] overflows once; a falling tail after it
    "sum_only": (400, [1e-38] * 8 + [1e-2, 1.0], 1.0),                # 391 entries near 1e306 under ratio 1
    "sum_only_long": (30000, [1e-38] * 8 + [1.0], 1.0),
    "both": (400, [1e-38] * 16 + [1e-4, 1.0], 1.0),                   # an overflow, then a flat run whose sum overflows
    "flush_p0": (100, [3e-38, 3e-38, 1.0], 3e38),                     # rescales at every early step: p[0] -> 0
    "flush_p0_long": (2000, [1e-38] * 40 + [1.0], 1.0),
}
FLUSHED = {"flush_p0", "flush_p0_long", "both"}                   # fixtures whose p[0] ends at 0


def witness(K, serv, lam, prec=200):
    """normalised p[0..K] of the birth-death chain p[n+1] = p[n] lam / servRate[min(n, len-1)], in mpmath with the
    float32 inputs as exact values (positive finite rates and lambda only)"""
    import mpmath
    mpmath.mp.prec = prec
    serv = [mpmath.mpf(float(F(s))) for s in serv]
    lam = mpmath.mpf(float(F(lam)))
    r = [mpmath.mpf(1)]
    for n in range(K):
        r.append(r[-1] * lam / serv[min(n, len(serv) - 1)])
    s = mpmath.fsum(r)
    return [x / s for x in r]


def witness_check(p, w, K, floor=2.0 ** -900, ulps=None):
    """the largest relative error of p against the witness over entries >= floor, and the bound it must meet: each
    entry passes through at most 2K chain operations, a few rescales, the (K+1)-term sum and the final division"""
    import mpmath
    bound = 4 * (K + 2) * 2.0 ** -53 if ulps is None else ulps
    worst = 0.0
    n = 0
    for pi, wi in zip(p, w):
        if wi < floor:
            continue
        n += 1
        worst = max(worst, float(abs((mpmath.mpf(float(pi)) - wi) / wi)))
    return worst, bound, n
