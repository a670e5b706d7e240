"""Inputs for the tests of pair sizing at BinarySearch's edges (test_pair_edges_cpu.py, test_pair_edges_gpu.py), and a
float32 restatement of the two bisections of QueueAnalyzer.Size (queueanalyzer.go:185-255, utils.go:26-70) together with
what size_pair_warp (csrc/wva_kernels.cuh) does around them.  Seeded and deterministic.

size_pair_warp does not run the reference's loop: it evaluates 3 tree levels speculatively in the first round and 4 in
every later round, skips nodes beyond the 100-iteration budget, takes a midpoint that rounds onto an endpoint from a memo,
evaluates a walked node whose certificate failed exactly, and runs the trailing Analyze under the guess throughput =
lambda * 1000.  The image built here puts one pair of each server at a chosen target class so that each of those paths
is taken:

  edge     edge_targets' classes (at / in / out of the band at both ends, inside, NaN, +Inf), TTFT or ITL alone.  A NaN
           target is skipped by Size like a zero one (`target > 0` is false), so it runs no search at all
  top      the first target below the value at lambdaMax outside its band: the search walks towards lambdaMax, where the
           certified tail's precondition M (1 - lambda / s_N) >= 0.3 fails for N = 2 and 8
  depth    target = y(x_d), x_d the d-th midpoint of the inside search: the search ends after exactly d iterations, in the
           first round, on its last level, in the first node of round 2 and across later round boundaries
  gap      a TTFT target strictly between y(x) and y(x+) for adjacent float32 x, outside the band of both: the interval
           collapses onto [x, x+] and the rest of the 100 iterations come from the memo
  mixed    a gap TTFT search (all 100 iterations) beside an ITL search that ends in round 1 (at_min or +Inf), with and
           without a TPS target
  tol      TOL_EDGE's flat-ITL pairs (a tolerance quotient of exactly 1e-6) and BUDGET_CFG's pair
  arrival  copies of a few pairs with arrival rates that put totalRate / rateStar, and totalRate / (lambda * 1000) (the
           kernel's guess), on an integer and one ulp either side

Every server has 3 accelerators: the targeted pair (accelerator s % 3) and two bystanders with make_system's profiles,
sized at the same SLOs and compared like the rest.
"""
import collections

import numpy as np

import analyzer_api_cases as ac
from test_pairs_loads_cpu import boundary_rates

F = np.float32
MAXIT = 100                               # utils.go:9
NS = (1, 2, 8, 48, 200)                   # srv_max_batch of the fixtures (N = 1: no certificate)
CERT_FAIL_NS = (2, 8)                     # M (1 - r) < 0.3 over the top of the range
DEPTHS = (1, 2, 3, 4, 5, 7, 8, 11, 12)
A = 3
TPS_ON = F(100.0)

Path = collections.namedtuple("Path", "x ind iters mids memo ivals")


# ---- float32 restatement -----------------------------------------------------------------------------------------------

def bisect_path(an, kind, lo, hi, target):
    """BinarySearch (utils.go:26-70) in float32 over an.eval (EvalTTFT / EvalITL) -> Path: the x and ind it returns,
    the iterations of its loop (0 for an exit at either end), the midpoints visited, whether a midpoint equalled an
    endpoint of its interval, and the interval before each iteration.  None where an evaluation is invalid."""
    lo, hi, target = F(lo), F(hi), F(target)
    if lo > hi:
        return None
    yb = []
    for x in (lo, hi):
        y = an.eval(kind, x)
        if y is None:
            return None
        if ac.within_tolerance(y, target):
            return Path(x, 0, 0, [], False, [])
        yb.append(y)
    inc = yb[0] < yb[1]
    if (inc and target < yb[0]) or (not inc and target > yb[0]):
        return Path(lo, -1, 0, [], False, [])
    if (inc and target > yb[1]) or (not inc and target < yb[1]):
        return Path(hi, +1, 0, [], False, [])
    mids, ivals, memo = [], [], False
    x = F(0)
    for _ in range(MAXIT):
        ivals.append((lo, hi))
        x = F(F(0.5) * F(lo + hi))
        memo = memo or x == lo or x == hi
        mids.append(x)
        y = an.eval(kind, x)
        if y is None:
            return None
        if ac.within_tolerance(y, target):
            break
        if (inc and target < y) or (not inc and target > y):
            hi = x
        else:
            lo = x
    return Path(x, 0, len(mids), mids, memo, ivals)


def node_x(lo, hi, node):
    """bisect_node_x: x of heap node `node` (children 2j: xMax = x, 2j+1: xMin = x) of the tree over [lo, hi], and
    whether its midpoint rounds onto an endpoint of its own interval"""
    lo, hi = F(lo), F(hi)
    depth = node.bit_length() - 1
    x = F(F(0.5) * F(lo + hi))
    for l in range(depth - 1, -1, -1):
        if (node >> l) & 1:
            lo = x
        else:
            hi = x
        x = F(F(0.5) * F(lo + hi))
    return x, bool(x == lo or x == hi)


def kernel_rounds(iters):
    """size_pair_warp's rounds for one search of `iters` iterations (0 for an end exit, None for no search): the first
    round walks 3 levels, every later one 4"""
    if iters is None:
        return 0
    return 1 + max(0, -(-(iters - 3) // 4))


def speculative_nodes(path, lo, hi):
    """x of every tree node size_pair_warp evaluates speculatively for this search: nodes 1..7 over [lo, hi] in round 1,
    nodes 1..15 over the interval reached after 3 + 4 (r - 2) iterations in round r >= 2; none deeper than the budget
    left, none whose midpoint rounds onto an endpoint (the memo resolves those)"""
    out = []
    for r in range(1, kernel_rounds(path.iters) + 1):
        it = 0 if r == 1 else 3 + 4 * (r - 2)
        l, h = (F(lo), F(hi)) if r == 1 else path.ivals[it]
        for node in range(1, 8 if r == 1 else 16):
            if node.bit_length() - 1 >= MAXIT - it:
                continue
            x, onto = node_x(l, h, node)
            if not onto:
                out.append(x)
    return out


def cert_precondition(lam, s_n, N):
    """cert_eval's preconditions at lambda (float32) with tail rate s_N (float32): N >= 2, K = 11 N <= 2^20,
    1 - r in [2^-11, 1) and M (1 - r) >= 0.3, M = K - N, 1 - r formed in float64 as cert_eval does"""
    if N < 2 or 11 * N > (1 << 20):
        return False
    s, l = float(s_n), float(lam)
    one_r = (s - l) / s
    return (one_r >= 2.0 ** -11) and (one_r < 1.0) and (10.0 * N * one_r >= 0.3)


def cfg_row(img, s, a, N=None):
    """the queue configuration (b, queue, alpha, beta, gamma, delta, in, out) CreateAllocation builds for pair (s, a)"""
    N = int(img.srv_max_batch[s]) if N is None else N
    m = int(img.srv_model[s]) * img.A + a
    return (N, 10 * N, img.perf_alpha[m], img.perf_beta[m], img.perf_gamma[m], img.perf_delta[m],
            int(img.srv_in_tokens[s]), int(img.srv_out_tokens[s]))


Sizing = collections.namedtuple("Sizing", "paths lam request rmax nil rounds")


def size_pair(an, c, targets):
    """QueueAnalyzer.Size's searches and range test for one pair: Sizing(paths {kind: Path or None for no search},
    lambda, requestRate, RateRange.Max, nil: Size fails, rounds size_pair_warp takes)"""
    lmin, lmax, rmax = ac.lambda_range(c)
    paths, lam = {}, []
    nil = False
    for k in ac.KINDS:
        t = F(targets[k])
        if not t > 0:
            paths[k] = None
            lam.append(lmax)
            continue
        p = bisect_path(an, k, lmin, lmax, t)
        paths[k] = p
        if p is None or p.ind < 0:
            nil = True
        lam.append(lmax if p is None else p.x)
    lam.append(lmax * (F(1) - ac.SAFETY) if F(targets[2]) > 0 else lmax)
    lam = F(min(lam))
    req = F(lam * F(1000))
    nil = nil or req <= 0 or req > rmax
    rounds = max(kernel_rounds(None if p is None else p.iters) for p in paths.values())
    return Sizing(paths, lam, req, rmax, nil, rounds)


def guess_miss(an, sz, total, min_rep):
    """whether size_pair_warp's trailing Analyze under the guess throughput = x1 * 1000 misses (its counter adds 100):
    the guessed per-replica rate differs from the real one or falls outside (0, RateRange.Max]"""
    x1 = F(sz.request / F(1000))
    guess = F(x1 * F(1000))
    rep_g = max(int(np.ceil(np.float64(total) / np.float64(guess))), int(min_rep))
    rate2_g = F(F(total) / F(rep_g))
    ok_g = not (rate2_g <= 0) and not (rate2_g > sz.rmax)
    _, m = an.analyze(sz.request)
    star = F(m.throughput)
    rep = max(int(np.ceil(np.float64(total) / np.float64(star))), int(min_rep))
    rate2 = F(F(total) / F(rep))
    return not (ok_g and rate2 == rate2_g), star, guess


def total_rate(img, s):
    """totalRate of CreateAllocation (allocation.go:128-133)"""
    if img.srv_slo_tps[s] == 0:
        return F(F(img.srv_arrival_rpm[s]) / F(60))
    return F(F(img.srv_slo_tps[s]) / F(int(img.srv_out_tokens[s])))


def zero_load(img, s):
    return img.srv_arrival_rpm[s] == 0 or img.srv_out_tokens[s] == 0


# ---- fixture targets ---------------------------------------------------------------------------------------------------

def _analyzer(oracle, row):
    return oracle.Analyzer(*row)


def gap_targets(an, c, kind=0, n=3):
    """up to n targets strictly between y(x) and y(x+) for adjacent float32 x, outside the band of both: the lowest,
    one in the middle and the highest gap found on a scan of the range that is dense near lambdaMax"""
    lmin, lmax, _ = ac.lambda_range(c)
    fr = np.concatenate([np.linspace(0.0, 1.0, 200), 1.0 - np.logspace(-1, -7, 60)])
    xs = sorted({F(lmin + (lmax - lmin) * F(f)) for f in fr} | {np.nextafter(lmax, F(0))})
    found = []
    for x in xs:
        if not lmin <= x < lmax:
            continue
        xp = np.nextafter(x, F(np.inf))
        y0, y1 = an.eval(kind, x), an.eval(kind, xp)
        t = F(np.sqrt(float(y0) * float(y1)))
        if y0 < t < y1 and not ac.within_tolerance(y0, t) and not ac.within_tolerance(y1, t):
            p = bisect_path(an, kind, lmin, lmax, t)        # a crossing elsewhere inside the band would end it early
            if p.iters == MAXIT and p.ivals[-1] == (x, xp):
                found.append((x, t))
    if len(found) <= n:
        return found
    return [found[0], found[len(found) // 2], found[-1]]


def top_target(an, c, kind):
    """the first target below y(lambdaMax) outside its tolerance band"""
    _, lmax, _ = ac.lambda_range(c)
    return ac.step_out(an.eval(kind, lmax), -np.inf)[1]


Item = collections.namedtuple("Item", "N prof cls kind targets arrival")


def _items(oracle):
    """the targeted pairs: (N, profile row, class, kind, (TTFT, ITL, TPS) targets, arrival rpm or None)"""
    out = []
    for i, N in enumerate(NS):
        for p in (i % 4, (i + 1) % 4):
            prof = ac.EDGE_PROFILES[p]
            c = ac.cfgs([(N, 10 * N) + prof])[0]
            an = _analyzer(oracle, (N, 10 * N) + prof)
            kinds = (0,) if N == 1 else ac.KINDS            # N = 1: EvalITL is flat (effective concurrency 1)
            tg = ac.edge_targets(oracle, c) if N > 1 else None
            for k in kinds:
                for cls in ac.EDGE_CLASSES:
                    t = tg[k, cls] if tg else _edge_ttft_only(oracle, c)[cls]
                    out.append(Item(N, prof, cls, k, _one(k, t), None))
                out.append(Item(N, prof, "top", k, _one(k, top_target(an, c, k)), None))
        # depth targets on a third profile: TTFT everywhere, ITL where its range is wide enough that x_11, x_12 are
        # not within tolerance of each other
        prof = ac.EDGE_PROFILES[(i + 2) % 4]
        c = ac.cfgs([(N, 10 * N) + prof])[0]
        an = _analyzer(oracle, (N, 10 * N) + prof)
        lmin, lmax, _ = ac.lambda_range(c)
        for k in ((0, 1) if N >= 48 else (0,)):
            y0, y1 = an.eval(k, lmin), an.eval(k, lmax)
            inside = bisect_path(an, k, lmin, lmax, F(np.sqrt(float(y0) * float(y1))))
            for d in DEPTHS:
                out.append(Item(N, prof, "depth%d" % d, k, _one(k, an.eval(k, inside.mids[d - 1])), None))
        # gap targets (TTFT only: EvalITL moves too little per float32 step) and the mixed pairs
        for p in range(4):
            prof = ac.EDGE_PROFILES[p]
            if N < 8 or (N == 8 and p not in (0, 3)):
                continue
            c = ac.cfgs([(N, 10 * N) + prof])[0]
            an = _analyzer(oracle, (N, 10 * N) + prof)
            gaps = gap_targets(an, c)
            if N == 8 or p % 2 == i % 2:
                for _, t in gaps:
                    out.append(Item(N, prof, "gap", 0, (t, F(0), F(0)), None))
                tg = ac.edge_targets(oracle, c)
                for cl in ("at_min", "inf"):
                    for tps in (F(0), TPS_ON):
                        out.append(Item(N, prof, "mixed_" + cl, 0, (gaps[-1][1], tg[1, cl], tps), None))
    for alpha, t in ac.TOL_EDGE:
        out.append(Item(48, ac.tol_edge_cfg(alpha)[2:], "tol", 1, (F(0), F(t), F(0)), None))
    out.append(Item(512, ac.BUDGET_CFG[2:], "budget", 0, tuple(F(x) for x in ac.BUDGET_TARGETS), None))
    return out


def _one(kind, t):
    return (F(t), F(0), F(0)) if kind == 0 else (F(0), F(t), F(0))


def _edge_ttft_only(oracle, c):
    """edge_targets' TTFT classes for N = 1 (edge_targets asserts an increasing EvalITL, which N = 1 does not have)"""
    an = _analyzer(oracle, tuple(c[k] for k in c.dtype.names))
    lmin, lmax, _ = ac.lambda_range(c)
    y0, y1 = an.eval(0, lmin), an.eval(0, lmax)
    in_min, out_min = ac.step_out(y0, -np.inf)
    in_max, out_max = ac.step_out(y1, np.inf)
    return {"at_min": y0, "in_min": in_min, "out_min": out_min, "at_max": y1, "in_max": in_max, "out_max": out_max,
            "inside": F(np.sqrt(float(y0) * float(y1))), "nan": F(np.nan), "inf": F(np.inf)}


# classes whose copies get arrival rates on the replica-count boundaries
ARRIVAL_FROM = (("inside", 0, 48), ("inf", 0, 8), ("depth7", 0, 200), ("top", 1, 2))


def _place(img, s, it, rng):
    a = s % A
    m = int(img.srv_model[s]) * A + a
    al, be, ga, de, inn, o = it.prof
    img.perf_alpha[m], img.perf_beta[m], img.perf_gamma[m], img.perf_delta[m] = al, be, ga, de
    img.srv_in_tokens[s], img.srv_out_tokens[s] = inn, o
    img.srv_max_batch[s] = it.N
    img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s] = it.targets
    img.srv_arrival_rpm[s] = it.arrival if it.arrival is not None else F(np.exp(rng.uniform(np.log(10.0), np.log(6e4))))


_CACHE = {}


def edge_image(wva, oracle):
    """(image, items): server s holds items[s] on accelerator s % 3"""
    if "img" in _CACHE:
        return _CACHE["img"]
    items = _items(oracle)
    # arrival copies: rates on the boundaries of rateStar and of the kernel's guess
    extra = []
    for cls, kind, N in ARRIVAL_FROM:
        it = next(x for x in items if x.cls == cls and x.kind == kind and x.N == N)
        c = ac.cfgs([(it.N, 10 * it.N) + it.prof])[0]
        an = _analyzer(oracle, (it.N, 10 * it.N) + it.prof)
        sz = size_pair(an, c, it.targets)
        assert not sz.nil, (cls, kind, N)
        _, star, guess = guess_miss(an, sz, F(1), 0)
        rates = np.unique(np.concatenate([boundary_rates(star), boundary_rates(guess)]))
        extra += [it._replace(arrival=F(r)) for r in rates]
    items = items + extra
    S = len(items)
    img = wva.synth.make_system(S, A, seed=4242, n_types=A, tps_fraction=0.0, zero_load_fraction=0.0,
                                keep_fraction=0.0, edge_fraction=0.0)
    img.perf_valid[:] = 1
    img.srv_target_valid[:] = 1
    img.srv_keep_acc[:] = 0
    rng = np.random.default_rng(4243)
    for s, it in enumerate(items):
        _place(img, s, it, rng)
    _CACHE["img"] = (img, items)
    return img, items


def restated(wva, oracle, img):
    """size_pair for every pair of the image: {(s, a): (Sizing, analyzer, config)}"""
    key = ("restated", id(img))
    if key not in _CACHE:
        out = {}
        for s in range(img.S):
            t = (img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s])
            for a in range(img.A):
                row = cfg_row(img, s, a)
                an = _analyzer(oracle, row)
                c = ac.cfgs([row])[0]
                out[s, a] = (size_pair(an, c, t), an, c)
        _CACHE[key] = out
    return _CACHE[key]


def oracle_pairs(oracle, img):
    key = ("oracle", id(img))
    if key not in _CACHE:
        _CACHE[key] = oracle.analyze_pairs(img, threads=oracle.hardware_threads())
    return _CACHE[key]
