"""An independent high-precision witness of the reference's queueing model: for a candidate (profile alpha beta gamma
delta, in, out, maxBatch b, maxQueue q, request rate) it gives the status Analyze returns and a float32 interval for
each of the 8 AnalysisMetrics fields and for p_block = float32 of the normalised p[K].

It was written from the reference's Go source alone -- pkg/analyzer/queueanalyzer.go, mm1modelstatedependent.go,
queuemodel.go, mm1kmodel.go and pkg/core/allocation.go:77-150 -- without reading this project's oracle or kernels, so
that a misreading shared by those two cannot pass through it.  It imports neither.  Citations are file:line of those
Go files.  The one rule that is not the reference's is the sweep's SLO test (`feasible`), which restates the sweep
this project adds (include/wva_b200.h, wva_analyze_grid).

Float32 scalars exactly as Go computes them (numpy float32, one IEEE round-to-nearest per operator, Go's operand
order; Go on amd64 does not fuse a*b+c):
  servRate[n-1] = n / (PrefillTime(in, n) + float32(numDecode) * DecodeTime(n))        queueanalyzer.go:103-113
  PrefillTime = 0 if in == 0 else gamma + (delta * float32(in)) * n                      :257-262
  DecodeTime = alpha + beta * n                                                          :264-266
  numDecode = out - 1, except 1 when in == 0 and out == 1                                :106-110
  RateRange = {(servRate[0] * Eps) * 1000, (servRate[b-1] * (1 - Eps)) * 1000}           :116-118
  K = MaxQueueSize + MaxBatchSize                                                        :121
  lambda = float32(requestRate / 1000)                                                   :146
  sweep: totalRate = ArrivalRate / 60, or TPS / float32(K_tokens) with a TPS target;
         rate = totalRate / float32(r)                                                   allocation.go:134-148
Statuses (exact predictions): NewQueueAnalyzer's checks (queueanalyzer.go:305-319) -> ERR_CONFIG; rate <= 0 -> ERR_RATE_LE0
(:135); rate > RateRange.Max -> ERR_RATE_MAX (:140); then the validity test of queuemodel.go:31 with the rho that
ComputeRho (mm1modelstatedependent.go:33-35) takes from the p[0] the model holds when Solve is entered.  A fresh
analyzer's p[] is all zeros (mm1kmodel.go:22), so rho = 1 and the model is invalid exactly when float32(K) <= 1 ->
ERR_MODEL.

The exact chain (mpmath, PREC bits) from the float32 rates and lambda taken as exact values:
  p_0 = 1, p_n = prod_{k<n} lambda / servRate[min(k, b-1)]                 mm1modelstatedependent.go:73-90
so for n <= N = b the p_n are a product (shared by every candidate of a row with the same profile and lambda: the
ramp), and above N the ratio rho = lambda / servRate[N-1] is constant, so with m = q:
  sum_{k=1..m} rho^k = rho (1 - rho^m) / (1 - rho),  sum_{k=1..m} k rho^k = rho (1 - (m+1) rho^m + m rho^(m+1)) / (1 - rho)^2
(m and m (m+1) / 2 at rho = 1), p_K = p_N rho^m.  With S = sum p_n the normalised aggregates are
  q_K = p_K / S,  inSys = sum_{i=1..K} i p_i / S,  inServ = sum_{i<=N} i p_i / S + N sum_{i>N} p_i / S
inServ is what :49-55 compute -- avgNumInSystem at i == num plus (1 - sumP) num -- written without the cancellation.

The interval the reference's float64 loop can produce around them.  u = 2^-53, g(k) = k u / (1 - k u), and
(1 + t_k) stands for a factor with |t_k| <= g(k) (products and quotients of such factors compose as in Higham, Lemma
3.3: (1+t_j)(1+t_k) = 1+t_{j+k}, (1+t_j)/(1+t_k) = 1+t_{j+2k}).  While no value leaves the normal range:
  * p[n+1] = (p[n] * lambda) / sRate (:83) is two roundings per step: pp_n = p_n (1 + t_{2n}), n <= K;
  * sum (:94-95) adds pp_0 .. pp_K in order; every term is positive and meets at most K additions:
    SS = S (1 + t_{3K});
  * p[n] /= sum (:110): qq_n = q_n (1 + t_{2K+1}) / (1 + t_{3K}) = q_n (1 + t_{8K+1});
  * avgNumInSystem (:50) adds fl(i qq_i), one more rounding each, K additions: inSys (1 + t_{9K+2}), and the partial
    sum at i = N likewise: A_N (1 + t_{9K+2});
  * sumP (:48, :51) at i = N: s_N (1 + t_{9K+1}), so 1 - sumP = t_N - e with |e| <= g(9K+1) s_N: the absolute
    term of (1 - sumP) num is at most N (g(2) t_N + (1 + g(2)) g(9K+1) s_N) -- of order K N u;
  * avgNumInServers = fl(A + fl(fl(1 - sumP) N)) (:53): one more relative u on the whole;
  * float32(p[K]) reads qq_K: q_K (1 + t_{8K+1}).
Terms below the normal range: each chain step, product and quotient then adds an absolute error of at most 2^-1075
(2^-1075 / sRate for the product before the division).  While every ratio lambda / sRate from the first such step on
is <= 1 these do not grow, so each pp_n is off by at most n (1 + 1 / min sRate) 2^-1074 (1 + g(2K)); the sum, the
normalisation and the i p products carry that through at most K terms each.  ABS = (K + 1)^3 (2 + 1 / min sRate)
2^-1072 bounds all of it, and is added to every aggregate (N ABS to inServ).  A chain whose ratio exceeds 1 after such
a step could amplify it, and is marked not witnessed.
Not witnessed either (counted; the oracle tests cover them): a chain that would meet a rescale predicate of :84-104
(an unnormalised p[n], p[n] lambda or sum >= 2^1000), a non-positive or non-finite rate or lambda.  mpmath's own
error (PREC = 256 bits; the closed forms lose at most ~2 log2(m / (1 - rho)) < 160 bits) is covered by a relative
2^-80.

Each aggregate interval is rounded outward to float64 and then to float32 at both ends (round-to-nearest is monotone,
so the reference's float32(x) lies between the float32 of the ends), and the float32 epilogue of Analyze
(mm1modelstatedependent.go:56-66, queueanalyzer.go:153-172, 296-302) runs on intervals: each Go float32 operator is
applied to every combination of endpoints with round-to-nearest and the result is the smallest and largest of
them (this takes the crossed ends for subtraction and division); the clamps apply to both ends.  Where every input
interval is one float32 the result is one float32: a bit-exact prediction.
"""
import concurrent.futures as cf
import itertools
import multiprocessing
import os

import mpmath
import numpy as np

F = np.float32
PREC = 256
U = 2.0 ** -53
EPS = F(0.001)                  # queueanalyzer.go:8
SAFETY = F(0.1)                 # queueanalyzer.go:11
QUEUE_RATIO = 10                # the sweep's MaxQueueSize = 10 b (config.MaxQueueToBatchRatio, allocation.go:87)

# status bytes of this project's C-ABI (include/wva_b200.h)
OK, FEASIBLE, ERR_CONFIG, ERR_RATE_LE0, ERR_RATE_MAX, ERR_MODEL = 0, 1, 4, 6, 8, 10
FIELDS = ("throughput", "avg_resp_time", "avg_wait_time", "avg_num_in_serv", "avg_prefill_time", "avg_token_time",
          "max_rate", "rho")
CAND_DTYPE = np.dtype([("b", "<i8"), ("q", "<i8"), ("alpha", "<f4"), ("beta", "<f4"), ("gamma", "<f4"),
                       ("delta", "<f4"), ("in", "<i8"), ("out", "<i8"), ("rate", "<f4")])

# ---- float32 scalars in Go's order -----------------------------------------------------------------------------------

def rate_table(al, be, ga, de, inn, out, n):
    """servRate[0 .. n-1] (queueanalyzer.go:103-113)"""
    al, be, ga, de = F(al), F(be), F(ga), F(de)
    fn = np.arange(1, n + 1, dtype=np.float64).astype(F)
    with np.errstate(all="ignore"):
        pre = np.zeros(n, F) if inn == 0 else ga + (de * F(inn)) * fn                   # :257-262
        nd = 1 if (inn == 0 and out == 1) else out - 1                                  # :106-110
        dec = F(nd) * (al + be * fn)                                                    # :111, :264-266
        return fn / (pre + dec)


def rate_range(tab, b):
    """(RateRange.Min, RateRange.Max) (queueanalyzer.go:116-118)"""
    with np.errstate(all="ignore"):
        return (tab[0] * EPS) * F(1000), (tab[b - 1] * (F(1) - EPS)) * F(1000)


def config_ok(b, q, inn, out):
    """Configuration.check and RequestSize.check (queueanalyzer.go:305-319)"""
    return b > 0 and q >= 0 and inn >= 0 and out >= 1


def sweep_rate(arrival, slo_tps, out, r):
    """the rate one replica of r analyses: totalRate / float32(r) (allocation.go:134-148)"""
    with np.errstate(all="ignore"):
        total = F(arrival) / F(60) if F(slo_tps) == 0 else F(slo_tps) / F(out)
        return total / F(r)


def rate_target_tps(rate_max):
    """TargetRate.RateTargetTPS of Size: (lambdaMax (1 - 0.1)) 1000 with lambdaMax = Max / 1000 (queueanalyzer.go:194,
    231-234, 246)"""
    with np.errstate(all="ignore"):
        return ((F(rate_max) / F(1000)) * (F(1) - SAFETY)) * F(1000)


# ---- float32 interval arithmetic -------------------------------------------------------------------------------------

def _op(f, *ivs):
    """[min, max] over every combination of endpoints of f (float32 round-to-nearest operators)"""
    with np.errstate(all="ignore"):
        vals = [F(f(*c)) for c in itertools.product(*ivs)]
    if any(np.isnan(v) for v in vals):
        return (F(np.nan), F(np.nan))
    return (min(vals), max(vals))


def _clamp(iv, lo, hi):
    """Go's min(max(x, lo), hi) on both ends"""
    return tuple(F(min(max(x, lo), hi)) for x in iv)


def _wait_clamp(iv):
    """if avgWaitTime < 0 { avgWaitTime = 0 } (mm1modelstatedependent.go:63-65) on both ends"""
    return tuple(F(0) if x < 0 else x for x in iv)


def _f32_iv(lo, hi, floor=-np.inf):
    """float32 round-to-nearest of every value in [lo, hi] (mpmath values; outward to float64 first); floor: a lower
    bound the value has whatever the error (0 for sums of non-negative terms)"""
    lo64 = np.nextafter(float(lo), -np.inf)
    hi64 = np.nextafter(float(hi), np.inf)
    return F(max(lo64, floor)), F(hi64)


def epilogue(c, lam32, rate_max, qK, inSys, inServ):
    """computeStatistics' float32 tail and Analyze (mm1modelstatedependent.go:56-66, queueanalyzer.go:153-172) on the
    float32 intervals of p[K], avgNumInSystem and avgNumInServers -> (8 metric intervals, p_block interval)"""
    al, be, ga, de = F(c["alpha"]), F(c["beta"]), F(c["gamma"]), F(c["delta"])
    inn, out, b = int(c["in"]), int(c["out"]), int(c["b"])
    lam = (lam32, lam32)
    pk = qK                                                                         # float32(m.p[m.K]) (:59)
    thr = _op(lambda x, y: x * (F(1) - y), lam, pk)                                 # lambda (1 - float32(p[K])) (:59)
    resp = _op(lambda x, y: x / y, inSys, thr)                                      # (:60)
    serv = _op(lambda x, y: x / y, inServ, thr)                                     # (:61)
    wait = _wait_clamp(_op(lambda x, y: x - y, resp, serv))                         # (:62-65)
    tokens = F(out - 1)                                                             # queueanalyzer.go:297
    num = _op(lambda x: x - (ga + al * tokens), serv)                               # :298
    den = (de * F(inn)) + (be * tokens)                                             # :299
    conc = _clamp(_op(lambda x: x / den, num), F(0), F(b))                          # :300-301
    if inn == 0:
        prefill = (F(0), F(0))                                                      # :258-260
    else:
        prefill = _op(lambda x: ga + (de * F(inn)) * x, conc)                       # :261
    token = _op(lambda x: al + be * x, conc)                                        # :265
    rho = _clamp(_op(lambda x: x / F(b), inServ), F(0), F(1))                       # :159-160
    thr1000 = _op(lambda x: x * F(1000), thr)                                       # :164
    rmax = (F(rate_max), F(rate_max))
    return [thr1000, resp, wait, inServ, prefill, token, rmax, rho], pk


# ---- the exact chain -------------------------------------------------------------------------------------------------

def _g(k):
    return k * U / (1 - k * U)


def _row(task):
    """every candidate of one row (profile, in, out, lambda): [(index, witnessed, lo[9], hi[9])], field 8 = p_block"""
    (al, be, ga, de, inn, out, lam32, rmax_of, cands) = task
    mp = mpmath.mp
    mp.prec = PREC
    mpf = mpmath.mpf
    bmax = max(b for _, b, _ in cands)
    tab = rate_table(al, be, ga, de, inn, out, bmax + 1)
    nan9 = [np.nan] * 9
    if not (lam32 > 0 and np.isfinite(lam32)) or not (np.all(tab[:bmax] > 0) and np.all(np.isfinite(tab[:bmax]))):
        return [(i, False, nan9, nan9) for i, _, _ in cands]
    big, tiny = mpf(2) ** 1000, mpf(2) ** -1000
    lam = mpf(float(lam32))
    with np.errstate(all="ignore"):
        ratio = [lam / mpf(float(s)) if s > 0 and np.isfinite(s) else mpf(0) for s in tab]
    ratio_f = np.array([float(x) for x in ratio])
    p, P, Q, pmax = [mpf(1)], [mpf(1)], [mpf(0)], [mpf(1)]
    first_low = None
    for n in range(bmax):
        nxt = p[n] * ratio[n]
        if first_low is None and (p[n] * lam < tiny or nxt < tiny):
            first_low = n
        p.append(nxt)
        P.append(P[n] + nxt)
        Q.append(Q[n] + (n + 1) * nxt)
        pmax.append(max(pmax[n], nxt))
    lam_hi = max(lam, mpf(1))
    slack = mpf(2) ** -80
    smin = float(np.min(tab[:bmax]))
    out_rows = []
    for idx, b, q in cands:
        N = b
        K = K_of(b, q)
        m = K - N
        split = N                      # computeStatistics sets avgNumInServers at i == num (mm1modelstatedependent.go:52)
        rho = ratio[N - 1]             # above N the chain divides by servRate[num-1] (mm1modelstatedependent.go:80-82)
        pN = p[N]
        if rho == 1:
            T0, T1 = mpf(m), mpf(m) * (m + 1) / 2
        else:
            rm = rho ** m
            T0 = rho * (1 - rm) / (1 - rho)
            T1 = rho * (1 - (m + 1) * rm + m * rm * rho) / (1 - rho) ** 2
        pK = pN * rho ** m if m >= 0 else pN / rho ** (-m)
        S = P[N] + pN * T0
        tail_max = pN * max(mpf(1), rho ** m if m >= 0 else mpf(1))
        if max(pmax[N], tail_max) * lam_hi >= big or S >= big:
            out_rows.append((idx, False, nan9, nan9))
            continue
        tail_low = m > 0 and min(pN, pK) * min(lam, mpf(1)) < tiny
        if (first_low is not None and first_low < N and ratio_f[first_low:N].max() > 1 - 1e-12) or \
                (tail_low and float(rho) > 1 - 1e-12):
            out_rows.append((idx, False, nan9, nan9))
            continue
        qK = pK / S
        in_sys = (Q[N] + pN * (N * T0 + T1)) / S
        A_split, s_split = Q[split] / S, P[split] / S
        t_split = 1 - s_split
        in_serv = A_split + N * t_split
        ABS = mpf((K + 1) ** 3) * (2 + 1 / mpf(smin)) * mpf(2) ** -1072
        e_qK = qK * (_g(8 * K + 1) + slack) + ABS
        e_sys = in_sys * (_g(9 * K + 2) + slack) + ABS
        e_serv = (U * abs(in_serv) + (1 + U) * (_g(9 * K + 2) * A_split + _g(2) * N * abs(t_split)
                                                + (1 + _g(2)) * _g(9 * K + 1) * N * s_split)
                  + slack * (A_split + N) + N * ABS)
        ivs = [_f32_iv(v - e, v + e, f) for v, e, f in ((qK, e_qK, 0.0), (in_sys, e_sys, 0.0), (in_serv, e_serv, -np.inf))]
        c = dict(alpha=al, beta=be, gamma=ga, delta=de, b=b, q=q)
        c["in"], c["out"] = inn, out
        metrics, pk = epilogue(c, lam32, rmax_of[b], *ivs)
        lo = [float(x[0]) for x in metrics] + [float(pk[0])]
        hi = [float(x[1]) for x in metrics] + [float(pk[1])]
        ok = not any(np.isnan(lo) | np.isnan(hi))
        out_rows.append((idx, ok, lo, hi))
    return out_rows


def _lambda(rate):
    """lambda = requestRate / 1000 in float32 (queueanalyzer.go:146)"""
    with np.errstate(all="ignore"):
        lam32 = F(F(rate) / F(1000))
    return lam32


def _profile(c):
    return (F(c["alpha"]), F(c["beta"]), F(c["gamma"]), F(c["delta"]), int(c["in"]), int(c["out"]))


def _default_procs():
    return max(1, min(32, os.cpu_count() or 1))


def analyze(cands, procs=None):
    """the witness of QueueAnalyzer(b, q).Analyze(rate) on a fresh analyzer for every candidate of a CAND_DTYPE array.
    Returns a dict: status (int8, exact), witnessed (bool: the metric intervals hold), lo / hi (float32 [n, 8], the
    AnalysisMetrics fields in order), pb_lo / pb_hi (float32 [n], p_block), rate_max (RateRange.Max)."""
    cands = np.asarray(cands, dtype=CAND_DTYPE)
    n = len(cands)
    status = np.zeros(n, np.int8)
    lo = np.full((n, 9), np.nan, F)
    hi = np.full((n, 9), np.nan, F)
    witnessed = np.zeros(n, bool)
    rmax_all = np.full(n, np.nan, F)
    rows, tables = {}, {}
    for c in cands:
        k = _profile(c)
        tables[k] = max(tables.get(k, 1), int(c["b"]))
    tables = {k: rate_table(*k, n) for k, n in tables.items()}
    for i, c in enumerate(cands):
        b, q, inn, out = int(c["b"]), int(c["q"]), int(c["in"]), int(c["out"])
        if not config_ok(b, q, inn, out):
            status[i] = ERR_CONFIG
            continue
        rate = F(c["rate"])
        _, rmax = rate_range(tables[_profile(c)], b)
        rmax_all[i] = rmax
        if rate <= 0:
            status[i] = ERR_RATE_LE0
            continue
        if rate > rmax:
            status[i] = ERR_RATE_MAX
            continue
        status[i] = ERR_MODEL if F(K_of(b, q)) <= F(1) else OK        # queuemodel.go:31, rho = 1 - float32(0)
        lam32 = _lambda(rate)
        key = (float(c["alpha"]), float(c["beta"]), float(c["gamma"]), float(c["delta"]), inn, out, float(lam32))
        rows.setdefault(key, {"lam": lam32})
        rows[key].setdefault("c", []).append((i, b, q))
        rows[key].setdefault("rmax", {})[b] = float(rmax)
    tasks = [(F(k[0]), F(k[1]), F(k[2]), F(k[3]), k[4], k[5], v["lam"], v["rmax"], v["c"]) for k, v in rows.items()]
    procs = _default_procs() if procs is None else procs
    if procs <= 1 or len(tasks) < 4:
        results = map(_row, tasks)
    else:
        ex = cf.ProcessPoolExecutor(procs, mp_context=multiprocessing.get_context("spawn"))
        tasks.sort(key=lambda t: -max(b for _, b, _ in t[8]) * len(t[8]))
        results = ex.map(_row, tasks, chunksize=max(1, len(tasks) // (8 * procs)))
    try:
        for res in results:
            for idx, ok, l, h in res:
                witnessed[idx] = ok
                lo[idx], hi[idx] = l, h
    finally:
        if procs > 1 and len(tasks) >= 4:
            ex.shutdown()
    witnessed &= status == OK
    return dict(status=status, witnessed=witnessed, lo=lo[:, :8], hi=hi[:, :8],
                pb_lo=lo[:, 8], pb_hi=hi[:, 8], rate_max=rmax_all)


def K_of(b, q):
    """occupancyUpperBound (queueanalyzer.go:121)"""
    return q + b


def inside(res, metrics, mask=None):
    """bool [n, 8]: each float32 field of `metrics` (a METRICS-shaped [n, 8] float32 array) lies in its interval"""
    m = np.asarray(metrics, F).reshape(len(res["lo"]), 8)
    ok = (m >= res["lo"]) & (m <= res["hi"])
    return ok if mask is None else ok[mask]


def singleton(res):
    """bool [n, 9]: the interval is one float32 (fields of AnalysisMetrics, then p_block)"""
    lo = np.concatenate([res["lo"], res["pb_lo"][:, None]], axis=1)
    hi = np.concatenate([res["hi"], res["pb_hi"][:, None]], axis=1)
    return lo.view(np.uint32) == hi.view(np.uint32)


def feasible(res, slo_ttft, slo_itl, slo_tps, rate, r, min_replicas):
    """the sweep's feasible bit where the intervals decide it: 1, 0, or -1 (undetermined).  A candidate is feasible
    when Analyze succeeds, TTFT = wait + prefill <= SLO_TTFT and ITL <= SLO_ITL (each when its SLO is > 0), the rate is
    <= RateTargetTPS (with a TPS target) and r >= the server's minimum replicas (include/wva_b200.h).  Float32
    addition is monotone in each operand, so the TTFT interval is the sums of the ends."""
    lo, hi = res["lo"], res["hi"]
    slo_ttft, slo_itl, slo_tps = (np.asarray(x, F) for x in (slo_ttft, slo_itl, slo_tps))
    with np.errstate(all="ignore"):
        ttft = (lo[:, 2] + lo[:, 4], hi[:, 2] + hi[:, 4])
        fixed = (~(slo_tps > 0) | (np.asarray(rate, F) <= rate_target_tps(res["rate_max"]))) & \
            (np.asarray(r) >= np.asarray(min_replicas))
        yes = np.ones(len(lo), bool)
        no = ~fixed | (res["status"] != OK)
        for (l, h), slo in ((ttft, slo_ttft), ((lo[:, 5], hi[:, 5]), slo_itl)):
            yes &= ~(slo > 0) | (h <= slo)
            no |= (slo > 0) & (l > slo)
    out = np.full(len(lo), -1, np.int8)
    out[res["witnessed"] & yes] = 1
    out[res["witnessed"] & no] = 0
    out[~fixed | (res["status"] != OK)] = 0
    return out
