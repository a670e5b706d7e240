"""The public analyzer API on the device -- wva_queue_size (Size), wva_queue_analyze (Analyze) and wva_model_solve (the
bare MM1ModelStateDependent) -- against the oracle, bit for bit (float32 through bit patterns, NaN = NaN): a Size fuzz
over batch sizes 1 .. 8192, the target edges of BinarySearch, the profile families of test_profile_edges_gpu.py, the
materialised retry of both batched calls (items whose chain needs rescaling, relaunched over a fault list with
per-item p[] scratch rows) and the bare model on rescaling, flushing and non-terminating inputs.  The inputs and their
classification are in analyzer_api_cases.py; test_analyzer_api_cpu.py shows that they reach their branches."""
import ctypes as C
import time

import numpy as np
import pytest

import analyzer_api_cases as ac                 # loads the package (wva_import)
import test_profile_edges_gpu as pe

from inferno_autoscaler_b200 import binding    # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32


def _same(got, want):
    """bit-equal float32 arrays or records, a NaN on both sides counting as equal"""
    g = np.ascontiguousarray(got).view(np.float32).reshape(-1)
    w = np.ascontiguousarray(want).view(np.float32).reshape(-1)
    same = (g.view(np.uint32) == w.view(np.uint32)) | (np.isnan(g) & np.isnan(w))
    bad = np.flatnonzero(~same)
    return None if len(bad) == 0 else int(bad[0])


def _size_equal(got, want, idx=None):
    idx = slice(None) if idx is None else idx
    assert np.array_equal(got[3][idx], want[3][idx]), np.flatnonzero(got[3][idx] != want[3][idx])[:5]
    for g, w, what in zip(got[:3], want[:3], ("rates", "metrics", "achieved")):
        bad = _same(g[idx], w[idx])
        assert bad is None, (what, bad)


def _timed(what, f, *a, **k):
    t0 = time.time()
    out = f(*a, **k)
    print("%s: oracle %.1f s" % (what, time.time() - t0))
    return out


# ---- 1. Size fuzz ------------------------------------------------------------------------------------------------------

def test_size_fuzz(wva, oracle, ctx):
    """60 000 Size calls: b log-uniform in 1 .. 8192 (about 1 % above 2048), queue in {0, 1, 3, 10, 20} b or random,
    all 8 combinations of zero and non-zero TTFT / ITL / TPS targets drawn around the item's own scale, invalid
    configurations and negative targets"""
    rng = np.random.default_rng(2024)
    n = 60000
    b = np.exp(rng.uniform(0, np.log(2048), n)).astype(np.int32)
    big = rng.random(n) < 0.01
    b[big] = rng.integers(2049, 8193, int(big.sum()))
    c = np.zeros(n, dtype=wva.abi.QUEUE_CONFIG_DTYPE)
    c["max_batch_size"] = b
    mult = rng.choice([0, 1, 3, 10, 20, -1], n)
    c["max_queue_size"] = np.where(mult >= 0, mult * b, rng.integers(0, 4 * b + 1))
    c["alpha"] = rng.uniform(1, 30, n); c["beta"] = rng.uniform(0.001, 1, n)
    c["gamma"] = rng.uniform(0, 250, n); c["delta"] = rng.uniform(0, 0.1, n)
    c["avg_input_tokens"] = rng.integers(0, 4000, n); c["avg_output_tokens"] = rng.integers(1, 1000, n)
    ttft0 = c["gamma"] + c["delta"] * c["avg_input_tokens"]
    itl0 = c["alpha"] + c["beta"]
    combo = rng.integers(0, 8, n)
    t = np.zeros((n, 3), F)
    t[:, 0] = np.where(combo & 1, ttft0 * np.exp(rng.uniform(-1, 4, n)), 0)
    t[:, 1] = np.where(combo & 2, itl0 * np.exp(rng.uniform(-0.5, 3, n)), 0)
    t[:, 2] = np.where(combo & 4, rng.uniform(1, 5000, n), 0)
    bad = rng.choice(n, 400, replace=False)
    c["max_batch_size"][bad[:100]] = rng.integers(-3, 1, 100)
    c["max_queue_size"][bad[100:150]] = -1
    c["avg_output_tokens"][bad[150:200]] = 0
    t[bad[200:], rng.integers(0, 3, 200)] = -rng.uniform(0, 10, 200)
    want = _timed("Size fuzz (%d items)" % n, oracle.queue_size, c, t, threads=oracle.hardware_threads())
    got = ctx.queue_size(c, t)
    _size_equal(got, want)
    ok = want[3] == 0
    assert 0.2 * n < ok.sum() < n
    for k in range(8):
        assert ok[combo == k].any() and (~ok[combo == k]).any(), k


# ---- 2. target edges ---------------------------------------------------------------------------------------------------

def test_size_target_edges(wva, oracle, ctx):
    """every edge class of BinarySearch, for the TTFT and the ITL target, in every EDGE_PROFILE at every EDGE_BATCH,
    through wva_queue_size; plus the iteration-budget pair and targets exactly at the tolerance bound"""
    rows, targets = [], []
    for prof in ac.EDGE_PROFILES:
        for b, q in ac.EDGE_BATCHES:
            c = ac.cfgs([(b, q) + prof])[0]
            for (k, cl), y in ac.edge_targets(oracle, c).items():
                t = [0.0, 0.0, 0.0]
                t[k] = y
                rows.append((b, q) + prof); targets.append(t)
                t2 = list(t); t2[2] = 100.0                  # the same with a TPS target
                rows.append((b, q) + prof); targets.append(t2)
    rows.append(ac.BUDGET_CFG); targets.append(list(ac.BUDGET_TARGETS))
    for alpha, y in ac.TOL_EDGE:                             # WithinTolerance exactly at its bound
        rows.append(ac.tol_edge_cfg(alpha)); targets.append([0.0, y, 0.0])
    c, t = ac.cfgs(rows), np.array(targets, F)
    want = _timed("target edges", oracle.queue_size, c, t, threads=oracle.hardware_threads())
    got = ctx.queue_size(c, t)
    _size_equal(got, want)
    assert (want[3] == 1).any() and (want[3] == 0).any()


# ---- 3. profile families through the public API ------------------------------------------------------------------------

@pytest.mark.parametrize("name", pe.FAMILIES)
def test_family_public_api(wva, oracle, ctx, name):
    """every (server, accelerator) pair of the family becomes queue configs at b in {1, B / 2, B, N} and queue in
    {0, 1, 10} b: Analyze at totalRate / r for r = 1 .. R, Size at the server's SLOs.  Items that would not return
    in the reference are not sent to the oracle; the device must reject them and leave the others as the oracle has
    them"""
    img, R, B = pe.family(wva, name)
    rows, rates, trows, targets = [], [], [], []
    for s in range(img.S):
        for a in range(img.A):
            al, be, ga, de = pe._coeffs(img, s, a)
            for bb in sorted({1, max(1, B // 2), B, pe.pair_n(img, s, a)}):
                for qm in (0, 1, 10):
                    row = (bb, qm * bb, al, be, ga, de, int(img.srv_in_tokens[s]), int(img.srv_out_tokens[s]))
                    total = F(F(img.srv_arrival_rpm[s]) / F(60))
                    for r in range(1, R + 1):
                        rows.append(row); rates.append(total / F(r))
                    trows.append(row); targets.append((img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s]))
    c, rate = ac.cfgs(rows), np.array(rates, F)
    hang = np.array([ac.analyze_hangs(c[i], rate[i]) for i in range(len(c))])
    keep = ~hang
    want_m, want_s = _timed("%s Analyze (%d items)" % (name, keep.sum()), oracle.queue_analyze, c[keep], rate[keep],
                            threads=oracle.hardware_threads())
    got_m, got_s = ctx.queue_analyze(c, rate)
    assert np.array_equal(got_s[keep], want_s) and _same(got_m[keep], want_m) is None, name
    assert (got_s[hang] == wva.abi.CAND_ERR_MODEL).all(), name
    tc, t = ac.cfgs(trows), np.array(targets, F)
    y = lambda i: (lambda k: oracle.Analyzer(*[tc[i][f] for f in tc.dtype.names]).eval(k, ac.lambda_range(tc[i])[0]))
    shang = np.array([ac.size_hangs(tc[i], t[i], y(i)) for i in range(len(tc))])
    want = _timed("%s Size (%d items)" % (name, (~shang).sum()), oracle.queue_size, tc[~shang], t[~shang],
                  threads=oracle.hardware_threads())
    got = ctx.queue_size(tc, t)
    _size_equal([g[~shang] for g in got], want)
    assert (got[3][shang] == 1).all(), name
    print("%s: %d Analyze items (%d not terminating), %d Size items (%d not terminating)" %
          (name, len(c), hang.sum(), len(tc), shang.sum()))


# ---- 4. the materialised retry -----------------------------------------------------------------------------------------

def _oracle_chain_per_item(oracle, c, rate=None, t=None):
    """the oracle's chain-rescale count of every item, one item at a time"""
    out = np.zeros(len(c), np.int64)
    for i in range(len(c)):
        c0 = oracle.rescale_counts()[0]
        if rate is not None:
            oracle.queue_analyze(c[i:i + 1], rate[i:i + 1])
        else:
            oracle.queue_size(c[i:i + 1], t[i:i + 1])
        out[i] = oracle.rescale_counts()[0] - c0
    return out


FAULT_K = [(900, 9000), (1500, 15000), (2500, 0), (1200, 1), (3000, 30000), (2000, 7), (1000, 3), (2200, 11)]
HANG_ROWS = [(4, 4, 3e38, -5e37, 0.0, 0.0, 0, 3), (4, 4, np.nan, 1.0, 1.0, 0.0, 0, 64)]


def _retry_batch(n, positions, with_hangs):
    """n tame items (b <= 64) with fault items of pairwise different K at `positions`, optionally two
    non-terminating items after them"""
    rows = [ac.tame_cfg(8 + i % 57, (i % 4) * 10) for i in range(n)]
    for j, pos in enumerate(positions):
        rows[pos] = ac.overflow_cfg(*FAULT_K[j % len(FAULT_K)])
    hang_pos = []
    if with_hangs:
        free = [i for i in range(n) if i not in positions]
        hang_pos = free[1:3]
        for hp, row in zip(hang_pos, HANG_ROWS):
            rows[hp] = row
    c = ac.cfgs(rows)
    rate = np.array([ac.overflow_rate(c[i], 0.98) if i in positions else
                     (ac.lambda_range(c[i])[2] if i in hang_pos else ac.overflow_rate(c[i], 0.7)) for i in range(n)], F)
    return c, rate, np.array(hang_pos, int)


RETRY_CASES = {
    "edges": (300, [0, 127, 128, 255, 299], False),
    "all_faults": (8, list(range(8)), False),
    "one_item": (1, [0], False),
    "with_hangs": (200, [0, 50, 199], True),
}


def test_retry_follows_larger_call(wva, oracle, ctx):
    """a call with faults after a larger call on the same context: the staging buffers hold stale items"""
    c, rate, _ = _retry_batch(2000, [5, 1999], False)
    ctx.queue_analyze(c, rate)
    ctx.queue_size(c, np.tile(np.array([[2000.0, 200.0, 0.0]], F), (len(c), 1)))
    _check_retry(wva, oracle, ctx, *_retry_batch(130, [3, 129], False), positions=[3, 129])


@pytest.mark.parametrize("case", sorted(RETRY_CASES))
def test_materialised_retry(wva, oracle, ctx, case):
    """fault items at the batch edges, a batch of faults only, a one-item batch and faults beside non-terminating
    items, through both calls"""
    n, positions, hangs = RETRY_CASES[case]
    _check_retry(wva, oracle, ctx, *_retry_batch(n, positions, hangs), positions=positions)


def _check_retry(wva, oracle, ctx, c, rate, hang_pos, positions):
    n = len(c)
    keep = np.ones(n, bool); keep[hang_pos] = False
    t = np.tile(np.array([[2000.0, 200.0, 0.0]], F), (n, 1))
    # Analyze: launches +2 with faults; the oracle's chain rescale on exactly the fault items
    chain = _oracle_chain_per_item(oracle, c[keep], rate=rate[keep])
    fault = np.zeros(n, bool); fault[positions] = True
    assert np.array_equal(chain > 0, fault[keep])
    want_m, want_s = oracle.queue_analyze(c[keep], rate[keep])
    l0 = ctx.launch_count()
    got_m, got_s = ctx.queue_analyze(c, rate)
    assert ctx.launch_count() - l0 == 2
    assert np.array_equal(got_s[keep], want_s) and _same(got_m[keep], want_m) is None
    assert (got_s[fault] == 0).all() and (got_s[hang_pos] == wva.abi.CAND_ERR_MODEL).all()
    # Size
    chain = _oracle_chain_per_item(oracle, c[keep], t=t[keep])
    assert np.array_equal(chain > 0, fault[keep])
    want = oracle.queue_size(c[keep], t[keep])
    l0 = ctx.launch_count()
    got = ctx.queue_size(c, t)
    assert ctx.launch_count() - l0 == 2
    _size_equal([g[keep] for g in got], want)
    assert (got[3][hang_pos] == 1).all()
    # the tame items alone: one launch each
    tame = ~fault & keep
    if not tame.any():
        return
    l0 = ctx.launch_count()
    got_m2, got_s2 = ctx.queue_analyze(c[tame], rate[tame])
    ctx.queue_size(c[tame], t[tame])
    assert ctx.launch_count() - l0 == 2
    assert _same(got_m2, got_m[tame]) is None


# ---- 5. the bare model -------------------------------------------------------------------------------------------------

def _model_compare(oracle, ctx, K, serv, lam, mu):
    """ctx.model_solve against oracle.Model call by call; returns the device's p"""
    out, p = ctx.model_solve(K, serv, lam, mu)
    m = oracle.Model(K, serv)
    for i in range(len(lam)):
        want = m.solve(float(lam[i]), float(mu[i]))
        bad = _same(out[i], np.array([want[k] for k in oracle._SOLVE_KEYS], F))
        assert bad is None, (K, i, oracle._SOLVE_KEYS[bad])
    assert p.tobytes() == m.probabilities().tobytes() or _same(p.view(np.float32), m.probabilities().view(np.float32)) is None
    return p


@pytest.mark.parametrize("name", sorted(ac.MODEL_FIXTURES))
def test_model_fixtures(oracle, ctx, name):
    """every rescale fixture, followed by further calls on the same model (the flushed p[0] gives rho 1), and the
    device's p[] against the mpmath witness"""
    K, serv, lam = ac.MODEL_FIXTURES[name]
    lams = np.array([lam, lam, 0.5, lam], F)
    mus = np.array([1.0, 0.0, 1.0, 1.0], F)
    p = _model_compare(oracle, ctx, K, np.array(serv, F), lams[:1], mus[:1])
    worst, bound, cnt = ac.witness_check(p, ac.witness(K, serv, lam), K)
    assert cnt > 0 and worst <= bound, (worst, bound)
    if K <= 2000:
        _model_compare(oracle, ctx, K, np.array(serv, F), lams, mus)


MODEL_EDGES = [   # (K, rates, lambdas, mus)
    (0, [1.0], [0.5, -0.0, 0.0], [1.0, 1.0, 1.0]),
    (1, [1.0], [0.5, 0.2], [1.0, 1.0]),
    (2, [0.5, 1.5], [0.3, 1.0, 2.0, 0.0], [1.0, 1.0, -1.0, 1.0]),
    (10, [0.5, 1.5, 2.0], [0.3, 1.0, 2.0], [1.0, np.nan, np.inf]),                # n_rates < K, mu NaN and +Inf valid
    (3, [0.5, 1.5, 2.0, 7.0, 9.0], [0.3, 1.0], [1.0, 1.0]),                       # n_rates > K: i == num never hit
    (3, [0.5, 1.5, 2.0], [0.3, 1.0], [1.0, 1.0]),                                 # n_rates == K
    (20, [1e-45, 3e-40, 1.0], [1e-40, 0.5], [1.0, 1.0]),                          # subnormal rates
    (20, [1.0, np.inf, 2.0], [0.5, 0.7], [1.0, 1.0]),                             # +Inf rate: p[n+1] = 0
    (30, [0.7, 1.1], [1e-45, 3.4028235e38, -0.0, 0.0, 1e-40], [1.0] * 5),        # subnormal and MaxFloat32 lambda
    (12, [1.0, -1.0, 2.0], [0.5, 0.5], [1.0, 1.0]),                               # negative rate: ends, p = NaN
    (25, [0.5, 1.0], [0.3, -1.0, 0.6, 0.4], [0.0, 1.0, -0.0, 1.0]),              # invalid calls between valid ones
]


@pytest.mark.parametrize("case", range(len(MODEL_EDGES)))
def test_model_edges(oracle, ctx, case):
    """K in {0, 1, 2, ...}, n_rates below, at and above K, subnormal and +Inf rates, lambda in {+-0, subnormal,
    MaxFloat32}, mu in {0, -0, negative, NaN, +Inf} and mixes of valid and invalid calls"""
    K, serv, lam, mu = MODEL_EDGES[case]
    _model_compare(oracle, ctx, K, np.array(serv, F), np.array(lam, F), np.array(mu, F))


def test_model_large_k(oracle, ctx):
    """K = 10^6 on a chain with a chain rescale, against the oracle and the witness's first entries"""
    K, serv = 1000000, np.array([1e-38] * 9 + [1.0, 2.0], F)
    _model_compare(oracle, ctx, K, serv, np.array([1.0, 1.5], F), np.array([1.0, 1.0], F))


NONTERMINATING = [(10, [1.0, 0.0], 0.5), (10, [1.0, np.nan], 0.5), (10, [1.0], np.inf), (10, [1.0], np.nan)]


@pytest.mark.parametrize("case", range(len(NONTERMINATING)))
def test_model_nonterminating(wva, oracle, ctx, case):
    """a call the reference never returns from raises ENONFINITE, alone and after valid calls; the next call on the
    context equals the oracle.  K = 2^28 + 1 raises EINVAL."""
    K, serv, lam = NONTERMINATING[case]
    assert ac.model_call_hangs(K, serv, lam, 1.0, 0.0)
    for lams in ([lam], [0.3, lam, 0.4]):
        with pytest.raises(binding.WvaError) as e:
            ctx.model_solve(K, np.array(serv, F), np.array(lams, F), np.ones(len(lams), F))
        assert e.value.code == wva.abi.ENONFINITE
        _model_compare(oracle, ctx, 40, np.array([0.5, 1.0], F), np.array([0.3, 0.6], F), np.ones(2, F))
    one, out = np.ones(1, F), np.zeros(9, F)
    ptr = lambda a: wva.abi.ptr(a, C.c_float)
    rc = binding.lib().wva_model_solve(ctx._h, (1 << 28) + 1, ptr(one), 1, 1, ptr(one), ptr(one), ptr(out), None)
    assert rc == wva.abi.EINVAL
