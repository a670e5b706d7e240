"""Pair sizing and the default candidate sweep against the oracle on performance profiles that synth.make_system never
produces.  make_system draws every coefficient from a narrow positive range, so every service-rate table it makes is
tame, every chain stays inside the float64 value window and no chain overflows.  Real profiles are not that polite: the
ConfigMap adapters turn a NaN, Inf or unparsable value into 0 (DESIGN §9.1), and a fitted profile with a tiny or a
negative term parses like any other.  Each family below keeps the sweep's shapes and changes the numbers in the
profiles so that they select branches of k_scan_prep / k_scan_cert / k_scan_lean that tame tables never take:

  zero        every subset of {alpha, beta, gamma, delta} set to 0, in in {0, 200}, out in {1, 2, 64}: tot(n) = 0 makes
              the rate +Inf (bad table entries, nGood < B -> literal list); EffectiveConcurrency's denominator
              delta*in + beta*(out-1) = 0 -> the epilogue's plain float32 division (pc.denOk false)
  tiny        coefficients in [1e-30, 1e-20) and float32 subnormals: non-tame tables (no died-out rule, the scan ramp
              leaves the value window -> deferred exact chains), denominators below 2^-60, rates up to +Inf
  huge        coefficients in (1e6, 1e30]: non-tame, denominators above 2^60, lambda below 2^-100 (row broken at b = 1)
  negative    a small negative delta or beta with tot(n) > 0, and pairs whose tot(n) crosses 0 inside the table:
              negative rates (literal list, status RATE_MAX behind the crossing)
  overflow    the profile of test_pairs_overflow_rescale_path swept to b = 2048: chains that overflow float64 and take
              the rescale branches (mm1modelstatedependent.go:84-89, 96-104) on the literal list with p[] in HBM
  load_edges  tame profiles, b_max = 300: lambda just below / above 2^-100 and subnormal, lambda in [2^-100, 2^-60)
              (k_scan_lean's plain division of the throughput), a b = 30 candidate a few ulps under RateRange.Max
              (the certificate's M(1-r) >= 0.3 test on both sides), 10 b (1-r) on both sides of 140 (its exp/log1p
              term), exact stops at b = 32c and 32c+1

The CPU tests show that each fixture reaches its branch -- a float32 restatement of BuildModel's rate table and of
scan_row_exact's stop rule, and the oracle -- and that the oracle terminates on it.  The GPU tests compare every pair
record and the whole metric cube with the oracle and check that the branch did run.  No profile holds a NaN and no
table holds a 0 rate: the reference's rescale loop never ends on those.  Nor does it size a pair whose RateRange.Max
is +Inf (unsizable_pairs); the pair tests leave those pairs out, the sweep keeps them.
"""
import struct

import numpy as np
import pytest

F = np.float32
B_CAP = 1 << 31
WIN_LO, WIN_SPAN = 0x0DF00000, 0x7DD00000 - 0x0DF00000      # high words of 2^-800 and 2^990 (wva_device.cuh)
FAMILIES = ["zero", "tiny", "huge", "negative", "overflow", "load_edges"]


# ---- float32 / float64 restatements -----------------------------------------------------------------------------------

def _hi(x):
    """high 32-bit word of a float64"""
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0] >> 32


def _coeffs(img, s, a):
    m = int(img.srv_model[s]) * img.A + a
    return img.perf_alpha[m], img.perf_beta[m], img.perf_gamma[m], img.perf_delta[m]


def rate_table(img, s, a, n):
    """servRate[0 .. n-1] of pair (s, a) in float32, in BuildModel's operation order (queueanalyzer.go:102-113)"""
    al, be, ga, de = _coeffs(img, s, a)
    inn, out = int(img.srv_in_tokens[s]), int(img.srv_out_tokens[s])
    fn = np.arange(1, n + 1, dtype=F)
    with np.errstate(all="ignore"):
        pre = np.zeros(n, F) if inn == 0 else ga + (de * F(inn)) * fn
        nd = 1 if (inn == 0 and out == 1) else out - 1
        dec = F(nd) * (al + be * fn)
        return fn / (pre + dec)


def ec_denominator(img, s, a):
    """EffectiveConcurrency's denominator delta*in + beta*(out-1) (queueanalyzer.go:296-302)"""
    al, be, ga, de = _coeffs(img, s, a)
    with np.errstate(all="ignore"):
        return de * F(int(img.srv_in_tokens[s])) + be * F(int(img.srv_out_tokens[s]) - 1)


def is_tame(img, s, a):
    """tame_parms (wva_device.cuh): every coefficient 0 or in [1e-20, 1e6]"""
    return all(x == 0 or (F(1e-20) <= x <= F(1e6)) for x in _coeffs(img, s, a))


def n_good(tab, B):
    """table entries [0, nGood) are positive and finite (k_scan_prep)"""
    bad = np.flatnonzero(~((tab[:B] > 0) & (tab[:B] < np.inf)))
    return int(bad[0]) if len(bad) else B


def row_lambda(img, s, r):
    """lambda of sweep row (s, *, r) in float32: (arrival / 60) / r / 1000"""
    return F(F(F(img.srv_arrival_rpm[s]) / F(60)) / F(r)) / F(1000)


def rate_max(tab):
    """RateRange.Max of every batch size (queueanalyzer.go:116-118)"""
    return (tab * (F(1) - F(0.001))) * F(1000)


def scan_row_stop(tab, B, good, tame, lam):
    """scan_row_exact's (stopB, brokenB), None for 'never': the exact ramp of one row and its died-out rule"""
    lam_d = float(lam)
    if not (2.0 ** -100 <= lam_d <= 2.0 ** 20):
        return None, 1
    n_end = min(good, B)
    if not tame or not (lam <= F(0.998) * tab[max(n_end - 1, 0)]):
        return None, None
    p = total = 1.0
    thr, hmin = 0, 0x3ff00000
    for n in range(n_end):
        pn = (p * lam_d) / float(tab[n])
        hq = _hi(pn)
        if (hq - WIN_LO) % (1 << 32) >= WIN_SPAN:
            return None, n + 1
        total += pn
        p = pn
        if n == 0 and pn >= 2.0 ** -400:
            thr = _hi((2.0 ** -68 * min(1.0, pn)) / float(11 * B))
        hmin = min(hmin, hq)
        if hq < thr and lam <= F(0.998) * tab[n] and total <= 2.0 ** 400:
            if (hmin >> 20) - (_hi(total) >> 20) < -1000:
                return None, n + 1
            return n + 1, None
    return None, None


def cert_x(tab, lam, b):
    """10 b (1 - r) of candidate b, r = lambda / servRate[b-1] (cert_eval_fast's x)"""
    s = float(tab[b - 1])
    return 10.0 * b * ((s - float(lam)) * (1.0 / s))


def _arrival_for_lambda(lam_target, below):
    """the float32 arrival rate whose row-1 lambda is the last one below (below=True) or the first one at or above
    lam_target"""
    a = F(float(lam_target) * 60000.0)
    lam = lambda x: F(F(x / F(60)) / F(1)) / F(1000)
    while lam(a) >= lam_target:
        a = np.nextafter(a, F(0))
    while lam(np.nextafter(a, F(np.inf))) < lam_target:
        a = np.nextafter(a, F(np.inf))
    return a if below else np.nextafter(a, F(np.inf))


# ---- fixture builder ---------------------------------------------------------------------------------------------------

def _base(wva, S, A, seed, max_batch_hi=129):
    """a make_system image with every pair usable, no TPS target and a server-level batch bound for pair sizing"""
    img = wva.synth.make_system(S, A, seed=seed, zero_load_fraction=0.0, keep_fraction=0.0, tps_fraction=0.0,
                                edge_fraction=0.0)
    rng = np.random.default_rng(seed + 1000)
    img.perf_valid[:] = 1
    img.srv_target_valid[:] = 1
    img.srv_slo_tps[:] = 0.0
    img.srv_max_batch[:] = rng.integers(8, max_batch_hi, S)
    return img, rng


def _loguniform(rng, lo, hi, n=None):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n))


def _zero(wva):
    S, A = 24, 4
    img, rng = _base(wva, S, A, 301)
    io = [(0, 1), (0, 2), (0, 64), (200, 1), (200, 2), (200, 64)]
    for s in range(S):
        img.srv_in_tokens[s], img.srv_out_tokens[s] = io[s % 6]
        for a in range(A):
            subset = (s // 6) * A + a                     # 16 subsets per (in, out) combination
            m = int(img.srv_model[s]) * A + a
            for bit, arr in enumerate((img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta)):
                if subset >> bit & 1:
                    arr[m] = 0.0
    img.srv_arrival_rpm[:] = _loguniform(rng, 1.0, 3000.0, S).astype(F)
    return img, 4, 100


def _tiny(wva):
    S, A = 16, 2
    img, rng = _base(wva, S, A, 302)
    n = S * A
    tiny = lambda k: _loguniform(rng, 1e-30, 1e-20, k).astype(F)
    mode = np.arange(n) % 4
    for arr in (img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta):
        arr[mode == 0] = tiny(int((mode == 0).sum()))                     # all tiny: rates ~1e20 .. +Inf
    img.perf_beta[mode == 1] = tiny(int((mode == 1).sum()))               # normal alpha, gamma; tiny beta, delta
    img.perf_delta[mode == 1] = tiny(int((mode == 1).sum()))
    img.perf_beta[mode == 2] = F(1e-41)                                    # float32 subnormals beside normal terms
    img.perf_delta[mode == 2] = F(3e-45)
    for arr in (img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta):
        arr[mode == 3] = F(2e-42)                                          # all subnormal
    img.srv_in_tokens[::5] = 0
    img.srv_arrival_rpm[:] = _loguniform(rng, 1.0, 60000.0, S).astype(F)
    return img, 4, 128


def _huge(wva):
    S, A = 16, 2
    img, rng = _base(wva, S, A, 303)
    n = S * A
    for arr in (img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta):
        arr[:] = _loguniform(rng, 1.001e6, 1e30, n).astype(F)
    img.srv_in_tokens[:] = rng.integers(0, 2049, S)
    img.srv_out_tokens[:] = rng.integers(1, 257, S)
    img.srv_slo_itl[::2] = 0.0; img.srv_slo_ttft[::2] = 0.0       # no latency target: candidates feasible, winners exist
    # loads relative to the pair's own rates (a = 0), so that most candidates are analysed and not rejected by RateRange
    for s in range(S):
        tab = rate_table(img, s, 0, 128)
        b = int(rng.integers(1, 129))
        img.srv_arrival_rpm[s] = F(float(tab[b - 1]) * rng.uniform(0.05, 1.0) * 60000.0)
    return img, 4, 128


def _negative(wva):
    S, A = 16, 2
    img, rng = _base(wva, S, A, 304, max_batch_hi=97)
    for s in range(S):
        for a in range(A):
            m = int(img.srv_model[s]) * A + a
            if s < 8:                                                      # tot(n) stays positive
                if (s + a) % 2:
                    img.perf_delta[m] = F(-rng.uniform(1e-7, 1e-5))
                else:
                    img.perf_beta[m] = F(-rng.uniform(1e-5, 1e-3))
            else:                                                          # tot(n) crosses 0 at n0
                n0 = rng.uniform(40.0, 150.0)
                img.perf_alpha[m], img.perf_beta[m], img.perf_gamma[m] = 10.0, 0.1, 100.0
                img.perf_delta[m] = F(-(170.0 / n0 + 0.7) / 200.0)
        if s >= 8:
            img.srv_in_tokens[s], img.srv_out_tokens[s] = 200, 8
    img.srv_arrival_rpm[:] = _loguniform(rng, 1.0, 600.0, S).astype(F)
    return img, 4, 160


def _overflow(wva):
    """test_pairs_overflow_rescale_path's image: near-linear rate growth, so the chain of batch size b peaks near e^b"""
    img = wva.synth.make_system(6, 2, seed=5, max_pair_batch=0)
    img.perf_alpha[:] = 20.0; img.perf_beta[:] = 1e-4; img.perf_gamma[:] = 10.0; img.perf_delta[:] = 1e-7
    img.perf_valid[:] = 1; img.srv_target_valid[:] = 1
    img.srv_max_batch[:] = [900, 1500, 2500, 1200, 3000, 2000]
    img.srv_arrival_rpm[:] = [3e5, 6e5, 2e6, 1e3, 5e6, 9e5]
    img.srv_in_tokens[:] = 64; img.srv_out_tokens[:] = 8
    img.srv_slo_itl[:] = 200.0; img.srv_slo_ttft[:] = 2000.0; img.srv_slo_tps[:] = 0.0
    img.srv_keep_acc[:] = 0
    return img, 8, 2048


STOP_TARGETS = (32, 33, 64, 65)


def _arrival_for_stop(img, s, B, target):
    """an arrival rate whose row 1 (accelerator 0) stops exactly at b = target, or None"""
    tab = rate_table(img, s, 0, B)
    good = n_good(tab, B)

    def stop(a):
        return scan_row_stop(tab, B, good, True, F(F(F(a) / F(60)) / F(1)) / F(1000))[0] or B_CAP

    lo, hi = 1e-3, 0.998 * float(tab[good - 1]) * 60000.0    # from a row that stops within a few states to one that never does
    if stop(lo) >= target or stop(hi) < target:
        return None
    for _ in range(80):
        mid = F(np.sqrt(lo * hi))
        if mid in (F(lo), F(hi)):
            break
        if stop(mid) >= target:
            hi = float(mid)
        else:
            lo = float(mid)
    a = F(hi)
    return a if stop(a) == target else None


def _load_edges(wva):
    S, A, R, B = 32, 2, 8, 300
    img, rng = _base(wva, S, A, 306)
    img.srv_out_tokens[:] = rng.integers(2, 65, S)
    img.srv_in_tokens[:] = rng.integers(16, 1025, S)
    # lambda of row 1: just below 2^-100, just at/above it, a float32 subnormal, inside [2^-100, 2^-60)
    img.srv_arrival_rpm[0] = _arrival_for_lambda(F(2.0 ** -100), below=True)
    img.srv_arrival_rpm[1] = _arrival_for_lambda(F(2.0 ** -100), below=False)
    img.srv_arrival_rpm[2] = _arrival_for_lambda(F(2.0 ** -130), below=False)
    img.srv_arrival_rpm[3] = _arrival_for_lambda(F(2.0 ** -80), below=False)
    # row 1's b = 30 candidate k ulps under RateRange.Max (10 b (1 - r) ~ 0.3); arrival / 60 does not reach every
    # float32, so gamma moves by an ulp at a time until the rate k ulps under the limit is reachable
    for i, k in enumerate((0, 0, 1, 2, 3, 5)):
        s = 4 + i
        m = int(img.srv_model[s]) * A
        for _ in range(64):
            target = rate_max(rate_table(img, s, 0, 30))[29]
            for _ in range(k):
                target = np.nextafter(target, F(0))
            a = F(float(target) * 60.0)
            while F(a / F(60)) > target:
                a = np.nextafter(a, F(0))
            while F(np.nextafter(a, F(np.inf)) / F(60)) <= target:
                a = np.nextafter(a, F(np.inf))
            if F(a / F(60)) == target:
                break
            img.perf_gamma[m] = np.nextafter(img.perf_gamma[m], F(np.inf))
        img.srv_arrival_rpm[s] = a
    # row 1's candidate b* with 10 b* (1 - r) = 140
    for i, bstar in enumerate((40, 64, 100, 150, 200, 250)):
        s = 10 + i
        tab = rate_table(img, s, 0, B)
        img.srv_arrival_rpm[s] = F(float(tab[bstar - 1]) * (1.0 - 14.0 / bstar) * 60000.0)
    # exact stops at b = 32c and 32c + 1 (two servers per target where the table allows it)
    s = 16
    for target in STOP_TARGETS:
        found = 0
        while found < 2 and s < 24:
            a = _arrival_for_stop(img, s, B, target)
            if a is not None:
                img.srv_arrival_rpm[s] = a
                found += 1
            s += 1
    img.srv_arrival_rpm[24:] = _loguniform(rng, 1.0, 60000.0, S - 24).astype(F)
    return img, R, B


_BUILDERS = dict(zero=_zero, tiny=_tiny, huge=_huge, negative=_negative, overflow=_overflow, load_edges=_load_edges)
_CACHE = {}


def family(wva, name):
    """(image, r_max, b_max) of a profile family, built once per session from fixed seeds"""
    if name not in _CACHE:
        _CACHE[name] = _BUILDERS[name](wva)
    return _CACHE[name]


def unsizable_pairs(img):
    """pairs whose RateRange.Max is +Inf at the pair's batch size N (servRate[N-1] is +Inf, or above float32's largest
    value / 0.999 / 1000).  The sweep of such a table terminates (p[n+1] = p[n] lambda / servRate[n] with a finite
    lambda), but sizing it does not: Size's bisection evaluates lambda = RateRange.Max / 1000 = +Inf, whose first chain
    step is Inf / servRate[0] = Inf or Inf / Inf = NaN, and the rescale loop of computeProbabilities
    (mm1modelstatedependent.go:84-89) never ends on either."""
    with np.errstate(over="ignore"):
        return [(s, a) for s in range(img.S) for a in range(img.A)
                if np.isposinf(rate_max(rate_table(img, s, a, pair_n(img, s, a)))[-1])]


def pairs_image(wva, name):
    """the family's image for pair sizing: the pairs whose sizing does not terminate in the reference lose their perf row"""
    img, _, _ = family(wva, name)
    out = img.shard(0, img.S)
    for s, a in unsizable_pairs(img):
        out.perf_valid[int(img.srv_model[s]) * img.A + a] = 0
    return out


_ORACLE = {}


def oracle_grid(oracle, wva, name):
    """the oracle's sweep of a family: (best, cube, status, rescale events it took)"""
    if name not in _ORACLE:
        img, R, B = family(wva, name)
        e0 = oracle.rescale_events()
        got = oracle.analyze_grid(img, R, B, want_cube=True, threads=oracle.hardware_threads())
        _ORACLE[name] = got[:3] + (oracle.rescale_events() - e0,)
    return _ORACLE[name]


# ---- per-family facts the CPU tests assert -----------------------------------------------------------------------------

def pair_n(img, s, a):
    """the batch size N pair sizing uses (allocation.go:85: the server's override, else maxBatch * atTokens / outTokens)"""
    m = int(img.srv_model[s]) * img.A + a
    n = int(img.srv_max_batch[s]) or int(img.perf_max_batch[m]) * int(img.perf_at_tokens[m]) // max(int(img.srv_out_tokens[s]), 1)
    return max(n, 1)


def tables(img, B):
    """{(s, a): float32 rate table over max(B, pair-sizing N)}"""
    return {(s, a): rate_table(img, s, a, max(B, pair_n(img, s, a))) for s in range(img.S) for a in range(img.A)}


def literal_from_tables(img, R, B):
    """candidates behind a bad table entry: k_scan_cert lists every one of them on the literal path"""
    return sum(R * (B - n_good(t, B)) for t in tables(img, B).values())


def cube_mismatch(got, want):
    """index of the first cube float that differs bit for bit (a NaN on both sides counts as equal), or None"""
    g = np.ascontiguousarray(got).view(np.float32)
    w = np.ascontiguousarray(want).view(np.float32)
    if g.shape != w.shape:
        return -1
    same = (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w))
    bad = np.flatnonzero(~same)
    return None if len(bad) == 0 else int(bad[0])


# ---- CPU: each fixture reaches its branch, and the oracle terminates on it ---------------------------------------------

@pytest.mark.parametrize("name", FAMILIES)
def test_family_tables_are_usable_inputs(wva, name):
    """no table entry is 0 or NaN (the reference's rescale loop never ends on those) and no profile holds a NaN"""
    img, R, B = family(wva, name)
    for arr in (img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta, img.srv_arrival_rpm):
        assert not np.isnan(arr).any(), name
    for (s, a), t in tables(img, B).items():
        assert not (t == 0).any() and not np.isnan(t).any(), (name, s, a)


@pytest.mark.parametrize("name,tame", [("zero", True), ("tiny", False), ("huge", False), ("negative", False),
                                       ("overflow", True), ("load_edges", True)])
def test_family_tameness(wva, name, tame):
    """zero, overflow and load_edges keep tame tables; tiny, huge and negative are non-tame on every pair"""
    img, _, _ = family(wva, name)
    flags = {is_tame(img, s, a) for s in range(img.S) for a in range(img.A)}
    assert flags == {tame}, name


def test_zero_family_branches(wva):
    """zero: all 16 subsets x in {0, >0} x out {1, 2, >>1}; tot = 0 everywhere (+Inf rates, nGood = 0) and a zero
    EffectiveConcurrency denominator both occur, next to ordinary pairs"""
    img, R, B = family(wva, "zero")
    combos = set()
    for s in range(img.S):
        for a in range(img.A):
            zeros = tuple(bool(x == 0) for x in _coeffs(img, s, a))
            combos.add((zeros, int(img.srv_in_tokens[s]) > 0, int(img.srv_out_tokens[s])))
    assert len(combos) == 16 * 2 * 3
    tabs = tables(img, B)
    goods = [n_good(t, B) for t in tabs.values()]
    assert goods.count(0) >= 6 and goods.count(B) > len(goods) // 2
    dens = [ec_denominator(img, s, a) for s, a in tabs]
    assert sum(d == 0 for d in dens) >= 16
    assert literal_from_tables(img, R, B) == R * sum(B - g for g in goods) > 0


def test_tiny_family_branches(wva):
    """tiny: coefficients below 1e-20 and float32 subnormals; rates finite or +Inf; EffectiveConcurrency denominators
    below 2^-60 (the epilogue's plain division); light rows that leave the value window"""
    img, R, B = family(wva, "tiny")
    c = np.concatenate([img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta])
    assert ((c > 0) & (c < F(1.1754944e-38))).any() and ((c >= F(1e-30)) & (c < F(1e-20))).any()
    tabs = tables(img, B)
    assert any(np.isinf(t[:B]).any() for t in tabs.values())
    dens = [ec_denominator(img, s, a) for s, a in tabs]
    assert sum(0 < d < 2.0 ** -60 for d in dens) >= 4


def test_huge_family_branches(wva):
    """huge: coefficients in (1e6, 1e30], tot(n) finite everywhere, denominators above 2^60, rows with lambda < 2^-100"""
    img, R, B = family(wva, "huge")
    c = np.concatenate([img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta])
    assert (c > 1e6).all() and (c <= F(1e30)).all()
    tabs = tables(img, B)
    for t in tabs.values():
        assert (t > 0).all() and np.isfinite(t).all()          # tot = +Inf would make a rate 0
    dens = [ec_denominator(img, s, a) for s, a in tabs]
    assert sum(d > 2.0 ** 60 for d in dens) >= 4
    lams = [float(row_lambda(img, s, r)) for s in range(img.S) for r in range(1, R + 1)]
    assert sum(0 < x < 2.0 ** -100 for x in lams) > 0 and sum(x >= 2.0 ** -100 for x in lams) > 0


def test_negative_family_branches(wva):
    """negative: a negative delta or beta with positive tables, and tables whose tot(n) crosses 0 inside the sweep
    (negative rates from there on: nGood < B)"""
    img, R, B = family(wva, "negative")
    assert (img.perf_delta < 0).any() and (img.perf_beta < 0).any()
    tabs = tables(img, B)
    crossing = [(s, a) for (s, a), t in tabs.items() if (t[:B] < 0).any()]
    positive = [(s, a) for (s, a), t in tabs.items() if (t > 0).all() and np.isfinite(t).all()]
    assert len(crossing) >= 8 and len(positive) >= 8
    for s, a in crossing:
        g = n_good(tabs[s, a], B)
        assert 30 < g < B and (tabs[s, a][g:B] < 0).any()
    assert literal_from_tables(img, R, B) > 0


def test_overflow_family_rescales(wva, oracle):
    """overflow: the oracle's sweep takes the rescale branches"""
    img, R, B = family(wva, "overflow")
    assert 1024 <= B <= 2048 and R == 8
    *_, events = oracle_grid(oracle, wva, "overflow")
    assert events > 0


def test_load_edges_family_branches(wva):
    """load_edges: lambda below / at 2^-100, subnormal and in [2^-100, 2^-60); a b = 30 candidate under RateRange.Max
    with 10 b (1-r) on both sides of 0.3 and candidates with it on both sides of 140, before their rows' stops; b_max
    not a multiple of 32; exact stops at 32c and 32c + 1"""
    img, R, B = family(wva, "load_edges")
    assert B % 32 != 0
    lam1 = [row_lambda(img, s, 1) for s in range(4)]
    assert float(lam1[0]) < 2.0 ** -100 <= float(lam1[1]) and float(np.nextafter(lam1[1], F(0))) < 2.0 ** -100
    assert 0 < lam1[2] < F(1.1754944e-38)
    assert 2.0 ** -100 <= float(lam1[3]) < 2.0 ** -60
    tabs = tables(img, B)
    near03, near140, stops = set(), set(), set()
    for (s, a), t in tabs.items():
        good = n_good(t, B)
        rmax = rate_max(t)
        for r in range(1, R + 1):
            lam = row_lambda(img, s, r)
            rate = F(F(img.srv_arrival_rpm[s]) / F(60)) / F(r)
            stop, broken = scan_row_stop(t, B, good, True, lam)
            if stop is not None:
                stops.add(stop)
            if (stop, broken) == (None, 1):
                continue
            last = min(stop or B_CAP, broken or B_CAP, good + 1, B + 1)      # candidates before the stop: the certificate
            for b in range(1, last):
                if not (rate <= rmax[b - 1]):
                    continue
                x = cert_x(t, lam, b)
                if b <= 30 and abs(x - 0.3) < 1e-3:
                    near03.add(x >= 0.3)
                if abs(x - 140.0) < 1.0:
                    near140.add(x >= 140.0)
    assert near03 == {False, True}, near03
    assert near140 == {False, True}, near140
    assert {32, 33, 64, 65} <= stops, sorted(stops)


@pytest.mark.parametrize("name", FAMILIES)
def test_oracle_terminates_on_family(wva, oracle, name):
    """the oracle sizes every pair and sweeps the whole cube of each family (the GPU tests compare with these)"""
    img, R, B = family(wva, name)
    _, _, status, _ = oracle_grid(oracle, wva, name)
    pairs, feas, _ = oracle.analyze_pairs(pairs_image(wva, name), threads=oracle.hardware_threads())
    assert len(status) == img.S * img.A * R * B
    assert ((status & 0xfe) == 0).sum() > 0                     # some candidates are analysed, not only rejected
    print("%s: %d candidates, %d analysed, %d feasible; %d pairs feasible" %
          (name, len(status), int(((status & 0xfe) == 0).sum()), int((status & 1).sum()), int(feas.sum())))


# ---- GPU: pair records and the whole cube against the oracle, and the branch did run ----------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", FAMILIES)
def test_family_pairs_match_oracle(wva, oracle, ctx, name):
    """both pair kernels (one thread per pair, one warp per pair) against Server.Calculate on every pair whose sizing
    terminates in the reference"""
    img = pairs_image(wva, name)
    want, wfe, _ = oracle.analyze_pairs(img, threads=oracle.hardware_threads())
    for warp_max in (0, 1 << 22):
        ctx.pairs_set_warp_max(warp_max)
        try:
            ctx.upload(img)
            got, gfe = ctx.analyze_pairs()
        finally:
            ctx.pairs_set_warp_max(1 << 22)
        assert np.array_equal(gfe, wfe), (name, warp_max)
        ok, field = got.equal_bits(want)
        assert ok, (name, warp_max, field)
    print("%s pairs: %d of %d feasible" % (name, int(wfe.sum()), len(wfe)))


def _sweep_and_compare(wva, oracle, ctx, name):
    img, R, B = family(wva, name)
    ctx.upload(img)
    best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
    lists, counters = ctx.grid_list_sizes(), ctx.grid_counters()
    w_best, w_cube, w_status, events = oracle_grid(oracle, wva, name)
    assert np.array_equal(status, w_status), (name, int(np.flatnonzero(status != w_status)[0]))
    assert best.tobytes() == w_best.tobytes(), name
    bad = cube_mismatch(cube, w_cube)
    assert bad is None, (name, bad // 8 if bad >= 0 else bad, bad % 8 if bad >= 0 else None)
    ok = int(((w_status & 0xfe) == 0).sum())
    assert counters["candidates_ok"] == ok, name
    print("%s sweep: deferred %d, literal %d, candidates_ok %d of %d, oracle rescale events %d" %
          (name, lists["deferred"], lists["literal"], ok, len(w_status), events))
    return img, R, B, lists


# families whose rows reach the exact-chain list (non-tame tables, lambda outside the exact ramp's window) and families
# whose candidates reach the literal list (bad table entries, overflow); where every literal candidate sits behind a
# bad table entry the count is exact
DEFERRED = {"tiny", "huge", "negative", "load_edges"}
LITERAL = {"zero", "negative", "overflow"}
LITERAL_EXACT = {"zero", "negative"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", FAMILIES)
def test_family_sweep_matches_oracle(wva, oracle, ctx, name):
    """the default sweep (k_scan_prep -> k_scan_cert || k_scan_lean -> exact-chain and literal lists): status bytes,
    winners and every cube float against the oracle, and the family's branch did run"""
    img, R, B, lists = _sweep_and_compare(wva, oracle, ctx, name)
    if name in DEFERRED:
        assert lists["deferred"] > 0, name
    if name in LITERAL:
        assert lists["literal"] > 0, name
    if name in LITERAL_EXACT:
        assert lists["literal"] == literal_from_tables(img, R, B), name
    if name == "overflow":
        assert oracle_grid(oracle, wva, name)[3] > 0


@pytest.mark.gpu
def test_zero_family_exact_chains_only(wva, oracle, ctx):
    """the zero family with certified tails off (exact chains only) against the oracle as well"""
    ctx.set_certified_tails(0)
    try:
        _sweep_and_compare(wva, oracle, ctx, "zero")
    finally:
        ctx.set_certified_tails(1)
