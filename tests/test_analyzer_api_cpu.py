"""CPU side of the analyzer API tests (test_analyzer_api_gpu.py): every fixture of analyzer_api_cases.py reaches the
branch it is built for, the oracle terminates on it, and the oracle's p[] agrees with an independent high-precision
solution.  No device is needed."""
import time

import numpy as np
import pytest

import analyzer_api_cases as ac
import test_profile_edges_gpu as pe

F = np.float32


def _analyzer(oracle, c):
    return oracle.Analyzer(*[c[k] for k in c.dtype.names])


# ---- the threaded Size oracle ------------------------------------------------------------------------------------------

def test_queue_size_mt_equals_single_thread(oracle):
    """wvao_queue_size_mt is byte-equal to the sequential loop for 1, 3 and all threads"""
    rng = np.random.default_rng(71)
    n = 300
    rows = [(int(rng.integers(1, 200)), int(rng.integers(0, 4)) * 10, *ac.EDGE_PROFILES[i % 4]) for i in range(n)]
    c = ac.cfgs(rows)
    c["max_queue_size"] *= c["max_batch_size"] // 10 + 1
    t = np.stack([rng.choice([0.0, 300.0, 2000.0], n), rng.choice([0.0, 20.0, 60.0], n),
                  rng.choice([0.0, 10.0], n)], 1).astype(F)
    t[:4] = [[-1, 0, 0], [np.nan, 0, 0], [0, np.inf, 0], [0, 0, 0]]
    c["max_batch_size"][4] = 0
    want = oracle.queue_size(c, t)
    for th in (1, 3, oracle.hardware_threads()):
        got = oracle.queue_size(c, t, threads=th)
        for g, w in zip(got, want):
            assert np.ascontiguousarray(g).tobytes() == np.ascontiguousarray(w).tobytes(), th
    assert 0 < int((want[3] == 0).sum()) < n


# ---- target edges ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("prof", range(len(ac.EDGE_PROFILES)))
def test_binary_search_target_edges(oracle, prof):
    """for the TTFT and the ITL search alike: a target equal to the value at lambdaMin or lambdaMax returns that end,
    the last target inside the tolerance band returns it too, the first one outside gives ind = -1 / +1, a target in
    between converges inside, NaN runs the 100 iterations to the restated end point and +Inf gives lambdaMax"""
    for b, q in ac.EDGE_BATCHES:
        c = ac.cfgs([(b, q) + ac.EDGE_PROFILES[prof]])[0]
        lmin, lmax, _ = ac.lambda_range(c)
        a = _analyzer(oracle, c)
        assert a.rate_range()[0] / F(1000) == lmin and a.rate_range()[1] / F(1000) == lmax
        tg = ac.edge_targets(oracle, c)
        assert {cl for _, cl in tg} == set(ac.EDGE_CLASSES)
        for (k, cl), t in tg.items():
            x, ind, err = a.binary_search(k, lmin, lmax, t)
            assert err == 0 and ac.edge_outcome_ok(cl, x, ind, lmin, lmax), (prof, b, k, cl, x, ind)
        for k in ac.KINDS:                                  # the band edges are one float32 step apart
            assert np.nextafter(tg[k, "in_min"], F(-np.inf)) == tg[k, "out_min"]
            assert np.nextafter(tg[k, "in_max"], F(np.inf)) == tg[k, "out_max"]


def test_binary_search_iteration_budget(oracle):
    """test_pairs_iteration_budget's pair: the TTFT search ends inside the interval with its last midpoint outside the
    tolerance (all 100 iterations), the ITL search converges"""
    c = ac.cfgs([ac.BUDGET_CFG])[0]
    lmin, lmax, _ = ac.lambda_range(c)
    a = _analyzer(oracle, c)
    x, ind, err = a.binary_search(0, lmin, lmax, ac.BUDGET_TARGETS[0])
    assert err == 0 and ind == 0 and lmin < x < lmax
    assert not ac.within_tolerance(a.eval(0, x), ac.BUDGET_TARGETS[0])
    x, ind, err = a.binary_search(1, lmin, lmax, ac.BUDGET_TARGETS[1])
    assert err == 0 and ind == 0 and ac.within_tolerance(a.eval(1, x), ac.BUDGET_TARGETS[1])


def test_tolerance_boundary_targets(oracle):
    """TOL_EDGE: |float32((alpha - t) / t)| is exactly 1e-6, EvalITL is alpha at both ends, and the ITL search returns
    lambdaMin with ind 0 -- only because the tolerance test is `<=`"""
    for alpha, t in ac.TOL_EDGE:
        alpha, t = F(alpha), F(t)
        assert abs((alpha - t) / t) == ac.TOL and ac.within_tolerance(alpha, t)
        c = ac.cfgs([ac.tol_edge_cfg(alpha)])[0]
        lmin, lmax, _ = ac.lambda_range(c)
        a = _analyzer(oracle, c)
        assert a.eval(1, lmin) == alpha and a.eval(1, lmax) == alpha
        assert a.binary_search(1, lmin, lmax, t) == (lmin, 0, 0)


def test_size_target_classes(oracle):
    """Size on the edge targets: ind = -1 is an error, ind = +1 sizes at lambdaMax; a TPS target alone gives
    0.9 lambdaMax, all targets zero give lambdaMax, a NaN target is skipped like a zero one"""
    c = ac.cfgs([(48, 480) + ac.EDGE_PROFILES[1]])
    lmin, lmax, _ = ac.lambda_range(c[0])
    tg = ac.edge_targets(oracle, c[0])
    cases = [((tg[0, "out_min"], 0, 0), None), ((0, tg[1, "out_min"], 0), None),
             ((tg[0, "out_max"], 0, 0), lmax), ((0, tg[1, "out_max"], 0), lmax),
             ((tg[0, "at_min"], 0, 0), lmin), ((0, 0, 0), lmax), ((0, 0, 5.0), lmax * (F(1) - ac.SAFETY)),
             ((np.nan, np.nan, 0), lmax), ((np.inf, np.inf, 0), lmax)]
    rates, _, _, status = oracle.queue_size(np.repeat(c, len(cases)), np.array([t for t, _ in cases], F))
    for i, (t, lam) in enumerate(cases):
        if lam is None:
            assert status[i] == 1, t
        else:
            assert status[i] == 0 and F(rates[i].min()) == lam * F(1000), (t, rates[i])


# ---- fault items: the chain rescale under Analyze and Size -------------------------------------------------------------

FAULT_BATCHES = [(900, 9000), (1500, 15000), (2500, 0), (1200, 1), (3000, 30000), (2000, 7)]


def test_overflow_profile_takes_chain_rescale(oracle):
    """the overflow profile near RateRange.Max takes the chain rescale in Analyze and somewhere in Size; the tame
    controls never do, and no item of either takes the sum rescale"""
    for b, q in FAULT_BATCHES:
        c = ac.cfgs([ac.overflow_cfg(b, q)])
        c0 = oracle.rescale_counts()
        _, st = oracle.queue_analyze(c, [ac.overflow_rate(c[0], 0.98)])
        c1 = oracle.rescale_counts()
        assert st[0] == 0 and c1[0] > c0[0] and c1[1] == c0[1], (b, q)
        _, _, _, st = oracle.queue_size(c, np.array([[2000.0, 200.0, 0.0]], F))
        c2 = oracle.rescale_counts()
        assert c2[0] > c1[0], (b, q)
    for b, q in [(8, 80), (100, 1000), (1024, 0)]:
        c = ac.cfgs([ac.tame_cfg(b, q)])
        c0 = oracle.rescale_counts()
        oracle.queue_analyze(c, [ac.overflow_rate(c[0], 0.98)])
        oracle.queue_size(c, np.array([[2000.0, 200.0, 0.0]], F))
        assert oracle.rescale_counts() == c0, (b, q)


# ---- bare-model fixtures -----------------------------------------------------------------------------------------------

MODEL_BRANCHES = {"chain_only": (True, False), "sum_only": (False, True), "sum_only_long": (False, True),
                  "both": (True, True), "flush_p0": (True, False), "flush_p0_long": (True, False)}


@pytest.mark.parametrize("name", sorted(ac.MODEL_FIXTURES))
def test_model_fixture_branches(oracle, name):
    """each bare-model fixture takes exactly the rescale branches it is named for, counted apart; the flushing ones
    leave p[0] = 0, so the next call reads a stale rho of 1"""
    K, serv, lam = ac.MODEL_FIXTURES[name]
    m = oracle.Model(K, serv)
    c0 = oracle.rescale_counts()
    out = m.solve(lam, 1.0)
    c1 = oracle.rescale_counts()
    chain, summ = MODEL_BRANCHES[name]
    assert out["valid"] == 1
    assert (c1[0] > c0[0]) == chain and (c1[1] > c0[1]) == summ, (name, c0, c1)
    p = m.probabilities()
    assert abs(p.sum() - 1.0) < 1e-12
    if name in ac.FLUSHED:
        assert p[0] == 0.0
        nxt = m.solve(0.5, 0.0)                      # an invalid call reports the stale rho it tested
        assert nxt["valid"] == 0 and nxt["rho"] == 1.0
    if name.startswith("flush"):
        assert c1[0] - c0[0] >= 3                    # p[0] divided by MaxFloat64 / K at least three times


@pytest.mark.parametrize("name", sorted(ac.MODEL_FIXTURES))
def test_model_fixture_witness(oracle, name):
    """the oracle's normalised p[] against the mpmath birth-death solution: relative error <= 4 (K+2) 2^-53 on every
    entry >= 2^-900"""
    K, serv, lam = ac.MODEL_FIXTURES[name]
    m = oracle.Model(K, serv)
    m.solve(lam, 1.0)
    worst, bound, n = ac.witness_check(m.probabilities(), ac.witness(K, serv, lam), K)
    assert n > 0 and worst <= bound, (name, worst, bound)


def test_witness_is_sharp(oracle):
    """the witness notices a one-ulp change of a single service rate on a tame model"""
    serv = np.array([0.3, 0.7, 1.1, 1.6], F)
    m = oracle.Model(12, serv)
    m.solve(0.9, 1.0)
    serv2 = serv.copy()
    serv2[2] = np.nextafter(serv2[2], F(2))
    worst, bound, _ = ac.witness_check(m.probabilities(), ac.witness(12, serv2, 0.9), 12, ulps=2.0 ** -40)
    assert worst > bound


# ---- the non-terminating classifier ------------------------------------------------------------------------------------

def test_classifier_restated_table_matches_families(wva):
    """cfg_rate_table is BuildModel's table as test_profile_edges_gpu.rate_table restates it, on every family pair"""
    for name in pe.FAMILIES:
        img, _, B = pe.family(wva, name)
        for s in range(img.S):
            for a in range(img.A):
                c = family_cfg(img, s, a, B, 0)
                got, want = ac.cfg_rate_table(c), pe.rate_table(img, s, a, B)
                assert got.tobytes() == want.tobytes(), (name, s, a)


def family_cfg(img, s, a, b, q):
    al, be, ga, de = pe._coeffs(img, s, a)
    return ac.cfgs([(b, q, al, be, ga, de, int(img.srv_in_tokens[s]), int(img.srv_out_tokens[s]))])[0]


HANGING = [   # (config, rate or targets, which call): inputs the reference never returns from
    ((4, 4, 3e38, -5e37, 0.0, 0.0, 0, 3), "analyze_max"),          # tot(1), tot(2) = +Inf: service rates 0
    ((4, 4, np.nan, 1.0, 1.0, 0.0, 0, 64), "analyze"),             # service rate NaN
    ((4, 4, 1.0, 1.0, 1.0, 0.0, 0, 64), "analyze_nan"),            # lambda NaN
    ((64, 640, 1e-37, 1e-37, 1e-37, 1e-37, 10, 10), "size"),       # RateRange.Max = +Inf
]


def test_classifier_flags_hanging_inputs(oracle):
    """the classifier flags every input of HANGING and none of the fault items, tame controls or invalid configs"""
    for row, kind in HANGING:
        c = ac.cfgs([row])[0]
        if kind == "analyze":
            assert ac.analyze_hangs(c, 1e-3), row
        elif kind == "analyze_max":
            rmax = ac.lambda_range(c)[2]
            assert ac.analyze_hangs(c, rmax) and not ac.analyze_hangs(c, np.nextafter(rmax, F(1))), row
        elif kind == "analyze_nan":
            assert ac.analyze_hangs(c, np.nan) and not ac.analyze_hangs(c, 1e-3), row
        else:
            assert ac.size_hangs(c, (0, 0, 0)) and ac.size_hangs(c, (100.0, 0, 0), lambda k: F(5.0))
            assert not ac.size_hangs(c, (-1, 0, 0)) and not ac.size_hangs(c, (5.0, 0, 0), lambda k: F(5.0))
            assert not ac.analyze_hangs(c, 1.0)
    for b, q in FAULT_BATCHES:
        c = ac.cfgs([ac.overflow_cfg(b, q)])[0]
        assert not ac.analyze_hangs(c, ac.overflow_rate(c, 0.98)) and not ac.size_hangs(c, (2000.0, 200.0, 0.0))
    c = ac.cfgs([(1, 0, 3e38, 1.0, 1.0, 0.0, 0, 64)])[0]              # K = 1: the model is never valid
    assert not ac.analyze_hangs(c, 1e-3) and not ac.size_hangs(c, (0, 0, 0))
    c = ac.cfgs([(0, 4, np.nan, 1.0, 1.0, 0.0, 0, 64)])[0]            # invalid configuration
    assert not ac.analyze_hangs(c, 1e-3)


def test_classifier_on_families(wva, oracle):
    """no family pair hangs under Analyze at totalRate / r (no table holds 0 or NaN); under Size at the server's
    SLOs exactly the pairs test_profile_edges_gpu.unsizable_pairs names hang at their pair-sizing N"""
    for name in pe.FAMILIES:
        img, R, B = pe.family(wva, name)
        unsizable = set(pe.unsizable_pairs(img))
        for s in range(img.S):
            for a in range(img.A):
                n = pe.pair_n(img, s, a)
                c = family_cfg(img, s, a, n, 10 * n)
                rate = F(F(img.srv_arrival_rpm[s]) / F(60))
                assert not any(ac.analyze_hangs(c, rate / F(r)) for r in range(1, R + 1)), (name, s, a)
                t = (img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s])
                y = lambda k: _analyzer(oracle, np.array([c])[0]).eval(k, ac.lambda_range(c)[0])
                assert ac.size_hangs(c, t, y) == ((s, a) in unsizable), (name, s, a)


def test_model_classifier(oracle):
    """rates 0 / NaN reached, lambda NaN / +Inf hang; a negative rate, an unreached 0 rate, K = 0 and invalid calls
    do not, and the oracle returns on every one of those"""
    hang = [(10, [1.0, 0.0], 0.5), (10, [1.0, np.nan], 0.5), (10, [1.0], np.inf), (10, [1.0], np.nan)]
    for K, serv, lam in hang:
        assert ac.model_call_hangs(K, serv, lam, 1.0, 0.0), (K, serv, lam)
    ok = [(10, [1.0, -1.0], 0.5, 1.0), (1000, [2.0, -1e-30], 1e30, 1.0), (2, [1.0, 1.0, 0.0], 0.5, 1.0),
          (0, [1.0], np.nan, 1.0), (10, [0.0], 0.5, 0.0), (10, [0.0], -1.0, 1.0), (10, [np.nan], 0.5, -0.0)]
    for K, serv, lam, mu in ok:
        assert not ac.model_call_hangs(K, serv, lam, mu, 0.0), (K, serv, lam, mu)
        oracle.Model(K, serv).solve(lam, mu)
    assert ac.model_call_hangs(10, [1.0], np.nan, np.nan, 0.0)         # mu NaN is valid in the reference
    assert not ac.model_call_hangs(1, [0.0], 0.5, 1.0, 0.0)            # K = 1: the first call is invalid (rho = 1)


def test_oracle_size_time_at_large_b(oracle):
    """the threaded oracle keeps the Size fuzz of the GPU file affordable: time per item at b = 512, printed"""
    c = ac.cfgs([ac.BUDGET_CFG] * 32)
    t = np.tile(np.array(ac.BUDGET_TARGETS, F), (32, 1))
    t0 = time.time()
    oracle.queue_size(c, t, threads=oracle.hardware_threads())
    dt = (time.time() - t0) / 32
    print("oracle Size at b = 512: %.2f ms per item with %d threads" % (dt * 1e3, oracle.hardware_threads()))
