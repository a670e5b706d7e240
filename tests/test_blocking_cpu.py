"""CPU: the oracle's blocking probability of sweep candidates (oracle_blocking.grid_candidates_blocking).

p_block is float32(p[K]) of the reference's computeProbabilities on NewQueueAnalyzer({b, 10 b}) at rate totalRate / r,
K = 11 b, for an analysed candidate; the quiet NaN otherwise.  The reference's throughput is lambda * (1 - float32(p[K]))
(mm1modelstatedependent.go:59) and Analyze reports it times 1000 (queueanalyzer.go:160), so on every analysed candidate

    cube.throughput == f32(f32(lambda * f32(1 - p_block)) * 1000),   lambda = f32(rate / 1000)

which ties p_block to an output the oracle has always had.
"""
import numpy as np
import pytest

from test_profile_edges_gpu import FAMILIES, family

F = np.float32
NAN_BITS = 0x7fc00000


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


def _threads(oracle):
    return max(1, oracle.hardware_threads())


def _random_candidates(img, R, B, n, seed):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, img.S, n), rng.integers(0, img.A, n), rng.integers(1, R + 1, n), rng.integers(1, B + 1, n))


def _rate(img, s, r):
    """totalRate / float32(r) in float32 (allocation.go:134-139)"""
    s = np.asarray(s)
    tps = img.srv_slo_tps[s]
    with np.errstate(all="ignore"):
        total = np.where(tps == F(0), img.srv_arrival_rpm[s] / F(60), tps / img.srv_out_tokens[s].astype(F)).astype(F)
        return (total / np.asarray(r).astype(F)).astype(F)


def check_throughput_identity(img, s, r, metrics, status, p_block):
    """cube.throughput == f32(f32(lambda * f32(1 - p_block)) * 1000) on every analysed candidate, NaN elsewhere.
    Returns the number of analysed candidates."""
    ok = (status & 0xfe) == 0
    assert np.array_equal(p_block[~ok].view(np.uint32), np.full(int((~ok).sum()), NAN_BITS, np.uint32))
    lam = (_rate(img, s, r) / F(1000)).astype(F)
    with np.errstate(all="ignore"):
        want = ((lam * (F(1) - p_block).astype(F)).astype(F) * F(1000)).astype(F)
    got = metrics["throughput"]
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    bad = np.flatnonzero(ok & ~same)
    assert len(bad) == 0, (int(bad[0]), float(got[bad[0]]), float(want[bad[0]]), float(p_block[bad[0]]))
    assert not np.isnan(p_block[ok]).any()
    assert ((p_block[ok] >= 0) & (p_block[ok] <= 1)).all()
    return int(ok.sum())


def test_p_block_is_the_analyzers_p_K(wva, oracle, ob):
    """p_block == float32(Analyzer.probabilities()[K]) after Analyze(totalRate / r), candidate by candidate"""
    img = wva.synth.make_system(12, 3, seed=11, n_types=2)
    s, a, r, b = _random_candidates(img, 16, 96, 400, seed=5)
    # a few heavily loaded candidates: the largest rate each pair accepts at b = 1, 2, 7
    s = np.concatenate([s, [0, 1, 2]]); a = np.concatenate([a, [0, 1, 2]]); r = np.concatenate([r, [1, 1, 1]])
    b = np.concatenate([b, [1, 2, 7]])
    metrics, status, p_block = ob.grid_candidates_blocking(img, s, a, r, b)
    o_metrics, o_status = oracle.grid_candidates(img, s, a, r, b)
    assert np.array_equal(status, o_status) and metrics.tobytes() == o_metrics.tobytes()
    rate = _rate(img, s, r)
    checked = 0
    for i in range(len(s)):
        if status[i] & 0xfe:
            assert p_block[i].view(np.uint32) == NAN_BITS
            continue
        m = int(img.srv_model[s[i]]) * img.A + int(a[i])
        an = oracle.Analyzer(int(b[i]), 10 * int(b[i]), img.perf_alpha[m], img.perf_beta[m], img.perf_gamma[m],
                             img.perf_delta[m], int(img.srv_in_tokens[s[i]]), int(img.srv_out_tokens[s[i]]))
        st, _ = an.analyze(rate[i])
        assert st == 0
        assert p_block[i].view(np.uint32) == F(an.probabilities()[11 * int(b[i])]).view(np.uint32), i
        checked += 1
    assert checked > 100


@pytest.mark.parametrize("config", [2, 3])
def test_throughput_identity_make_system(wva, oracle, ob, config):
    """the identity on random candidates of the generator's configurations (servers of config 3 thinned to 200)"""
    c = dict(wva.synth.CONFIGS[config])
    img = wva.synth.make_system(min(c["S"], 200), c["A"], seed=config, n_types=c["T"])
    s, a, r, b = _random_candidates(img, c["r_max"], c["b_max"], 20000, seed=config)
    metrics, status, p_block = ob.grid_candidates_blocking(img, s, a, r, b, threads=_threads(oracle))
    n_ok = check_throughput_identity(img, s, r, metrics, status, p_block)
    assert n_ok > 5000
    assert (p_block[(status & 0xfe) == 0] > 0).any()          # not every analysed candidate blocks nothing


@pytest.mark.parametrize("name", FAMILIES)
def test_throughput_identity_profile_families(wva, oracle, ob, name):
    """the identity on the performance-profile families of test_profile_edges_gpu (a random sample of each)"""
    img, R, B = family(wva, name)
    s, a, r, b = _random_candidates(img, R, B, 4000, seed=17)
    metrics, status, p_block = ob.grid_candidates_blocking(img, s, a, r, b, threads=_threads(oracle))
    o_metrics, o_status = oracle.grid_candidates(img, s, a, r, b, threads=_threads(oracle))
    assert np.array_equal(status, o_status) and metrics.tobytes() == o_metrics.tobytes()
    assert check_throughput_identity(img, s, r, metrics, status, p_block) > 0
