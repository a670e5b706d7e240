"""Candidates whose float32 result sits on a rounding boundary: the fixture tests/golden/hard_rounding.json, written by
tools/hard_rounding.py, checked here against the oracle alone.

Most candidates of the sweep and of the blocking plane never run the reference's chain.  A closed form computes a
value v, and v is accepted when v (1 - E) and v (1 + E) round to the same float32 (DESIGN §4 iii-v).  A bound E that is
too small can only show on a candidate whose reference float64 value lies within about E v of a float32 rounding
midpoint, which ordinary candidates almost never do.  The fixture holds candidates built to sit there.  d is the relative
distance of the REFERENCE's float64 value to the nearest float32 midpoint, in units of u = 2^-53:

  P   plane, must be listed for an exact chain: d(p[K] / sum) < E_blk / 2, E_blk = 10 K + 16384, with the closed
      form's preconditions met, so that only the width of the certificate decides
  Pf  plane, must be accepted: d >= 2 E_blk, the preconditions met with room to spare
  Pz  plane, at the certified zero's edge (block_certify: 0 when log2 p[N] + M log2 rho < -160): the two consecutive
      loads whose bound straddles -160 ('below' in [-161, -160), 'above' in [-160, -159]), and the lightest load
      whose p_block is not 0 ('subnormal': a nonzero float32 subnormal, which a looser threshold would turn into 0);
      compared bit for bit
  C   cube, must be deferred: d(inSys) < 32 K, or |inServ - m| < 32 K u inServ, or d(p[K]) < 64 K with 1 - f32 of
      the float32 values on either side of the midpoint differing; the certificate's preconditions met
  Cf  cube, must be certified: d >= 128 K on inSys and inServ, d >= 256 K on p[K]
  Q   pair records: a C candidate at the pair's own (replicas, N)

Each entry is one server of its own model on one accelerator.  The CPU tests re-derive every expected bit and every
class from the oracle (Analyzer.probabilities, Analyzer.solve, grid_candidates, grid_candidates_blocking) and check that
the float64 restatement below gives the oracle's values; the GPU tests are in test_hard_rounding_gpu.py.
"""
import json
import math
import os
import types

import numpy as np
import pytest

from test_profile_edges_gpu import rate_table as image_rate_table

F = np.float32
U = 2.0 ** -53
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hard_rounding.json")
B_VALUES = (1, 2, 3, 5, 8, 13, 31, 32, 33, 64, 100, 256, 512, 1024, 2048, 4096, 8192)
CLASSES = ("P", "Pf", "Pz", "C", "Cf", "Q")
MIN_COUNT = dict(P=64, C=64, Pf=16, Pz=16, Cf=16, Q=16)
WIN_LO, WIN_HI = 2.0 ** -800, 2.0 ** 990              # the scan ramp's value window (wva_device.cuh)


# ---- bit helpers ------------------------------------------------------------------------------------------------------

def f32_hex(x):
    return "%08x" % int(np.asarray(x, dtype=F).view(np.uint32))


def hex_f32(h):
    return np.uint32(int(h, 16)).view(F)


# ---- the fixture's images ---------------------------------------------------------------------------------------------

def entries_image(wva, entries):
    """one server per entry, each with a model of its own on the single accelerator; no current allocation, no TPS
    target; srv_max_batch is the entry's pair batch size N (0: the candidate is only swept)"""
    S = len(entries)
    img = wva.image.SystemImage(S, 1, S, 1)
    img.acc_cost[:] = 10.0
    img.acc_multiplicity[:] = 1
    img.acc_type[:] = 0
    for i, e in enumerate(entries):
        img.perf_alpha[i], img.perf_beta[i] = hex_f32(e["alpha"]), hex_f32(e["beta"])
        img.perf_gamma[i], img.perf_delta[i] = hex_f32(e["gamma"]), hex_f32(e["delta"])
        img.srv_arrival_rpm[i] = hex_f32(e["arrival"])
        img.srv_in_tokens[i], img.srv_out_tokens[i] = e["in"], e["out"]
        img.srv_slo_itl[i], img.srv_slo_ttft[i] = hex_f32(e["slo_itl"]), hex_f32(e["slo_ttft"])
        img.srv_max_batch[i] = e["n_pair"]
    img.perf_max_batch[:] = 256
    img.perf_at_tokens[:] = 128
    img.perf_acc_count[:] = 1
    img.perf_valid[:] = 1
    img.srv_model[:] = np.arange(S, dtype=np.int32)
    img.srv_target_valid[:] = 1
    img.srv_slo_tps[:] = 0.0
    return img


def load_fixture():
    with open(FIXTURE) as f:
        return json.load(f)


def groups(entries):
    """{b: [entry indices]} of the swept entries (Q entries are swept with their own image)"""
    out = {}
    for i, e in enumerate(entries):
        if e["cls"] != "Q":
            out.setdefault(e["b"], []).append(i)
    return out


# ---- float32 / float64 restatements -----------------------------------------------------------------------------------

def rate_table(alpha, beta, gamma, delta, inn, out, n):
    """servRate[0 .. n-1] in float32 of one profile: test_profile_edges_gpu.rate_table (BuildModel's operation order)
    on a one-pair view holding just the fields it reads"""
    pair = types.SimpleNamespace(A=1, srv_model=[0], srv_in_tokens=[inn], srv_out_tokens=[out],
                                 perf_alpha=np.array([alpha], F), perf_beta=np.array([beta], F),
                                 perf_gamma=np.array([gamma], F), perf_delta=np.array([delta], F))
    return image_rate_table(pair, 0, 0, n)


def row_lambda(arrival, r):
    """lambda of sweep row r and of a pair with r replicas: f32(f32(f32(arrival / 60) / r) / 1000)"""
    return F(F(F(arrival) / F(60)) / F(r)) / F(1000)


def chain(tab, b, lam):
    """The reference's computeProbabilities + computeStatistics (mm1modelstatedependent.go:38-112) in float64 for a
    vector of lambdas sharing one table, without rescaling: p[n+1] = (p[n] lambda) / s[n], sum = p[0] + ... + p[K] in
    index order, q[i] = p[i] / sum, inSys += i q[i], inServ = inSys + (1 - sumP) N at i == N.
    Returns a dict of float64 arrays: pN, sumN (sum up to p[N]), S, pK (= q[K]), in_sys, in_serv, pmin, pmax (over
    the ramp p[1..N])."""
    lam = np.asarray(lam, dtype=F).astype(np.float64)
    K = 11 * b
    s = tab[:b].astype(np.float64)
    p = np.ones_like(lam)
    tot = np.ones_like(lam)
    pmin, pmax = np.full_like(lam, np.inf), np.zeros_like(lam)
    pN = sumN = None
    with np.errstate(all="ignore"):
        for n in range(K):
            p = (p * lam) / s[min(n, b - 1)]
            tot = tot + p
            if n < b:
                pmin, pmax = np.minimum(pmin, p), np.maximum(pmax, p)
            if n == b - 1:
                pN, sumN = p, tot
        S = tot
        p = np.ones_like(lam)
        sumP = 1.0 / S
        in_sys = np.zeros_like(lam)
        in_serv = None
        q = sumP
        for i in range(1, K + 1):
            p = (p * lam) / s[min(i - 1, b - 1)]
            q = p / S
            in_sys = in_sys + float(i) * q
            sumP = sumP + q
            if i == b:
                in_serv = in_sys + (1.0 - sumP) * float(b)
    return dict(pN=pN, sumN=sumN, S=S, pK=q, in_sys=in_sys, in_serv=in_serv, pmin=pmin, pmax=pmax)


def _next_away(f, v):
    """the float32 neighbour of f on v's side"""
    return np.nextafter(f, np.where(v > f.astype(np.float64), F(np.inf), F(-np.inf)))


def midpoint(v):
    """the float32 rounding midpoint nearest to each float64 in v (exact in float64), and the float32 values on either
    side of it"""
    v = np.asarray(v, dtype=np.float64)
    f = v.astype(F)
    g = _next_away(f, v)
    m = (f.astype(np.float64) + g.astype(np.float64)) * 0.5
    return m, np.minimum(f, g), np.maximum(f, g)


def dist_u(v):
    """relative distance of v to its nearest float32 rounding midpoint, in units of u"""
    v = np.asarray(v, dtype=np.float64)
    m, _, _ = midpoint(v)
    with np.errstate(all="ignore"):
        return np.abs(v - m) / np.abs(v) / U


def block_terms(st, lam, tab, b):
    """the quantities block_certify tests (wva_block.cuh), in float64 numpy: 1 - r, log2 P, the zero bound
    log2 p[N] + M log2 rho, p[N] and p[N] lambda"""
    lamd = np.asarray(lam, dtype=F).astype(np.float64)
    s = float(tab[b - 1])
    M = 10 * b
    with np.errstate(all="ignore"):
        one_r = (s - lamd) / s
        rho = (lamd / s) * (1.0 + 2.0 ** -50)
        zero = np.log2(st["pN"]) + M * np.log2(rho)
        logP = np.log2(st["pN"]) + M * np.log2(lamd / s)
    return dict(one_r=one_r, zero=zero, logP=logP)


def zero_edge_case(st, lam, tab, b):
    """which edge of the certified zero (block_certify: bound log2 p[N] + M log2 rho < -160 -> 0) a candidate sits at:
    'below' (bound in [-161, -160): certified zero), 'above' (bound in [-160, -159]: the closed form or an exact chain
    decides), 'subnormal' (the reference's p_block is a nonzero float32 subnormal, so a zero certificate would be
    wrong), or ''"""
    z = block_terms(st, lam, tab, b)["zero"]
    pk = st["pK"].astype(F)
    return np.where((pk > 0) & (pk < F(2.0 ** -126)), "subnormal",
                    np.where((z >= -161.0) & (z < -160.0), "below", np.where((z >= -160.0) & (z <= -159.0), "above", "")))


def cube_x(lam, tab, b):
    """1 - r and x = M (1 - r) of cert_eval / cert_eval_fast"""
    s = float(tab[b - 1])
    one_r = (s - np.asarray(lam, dtype=F).astype(np.float64)) / s
    return one_r, 10.0 * b * one_r


def e_blk(b):
    return 10.0 * 11 * b + 16384.0


def cube_dists(st, b):
    """(d inSys, inServ distance relative to inServ, d p[K], 1 - f32 of p[K]'s two neighbours differ), units of u"""
    K = 11 * b
    d_sys = dist_u(st["in_sys"])
    m, _, _ = midpoint(st["in_serv"])
    with np.errstate(all="ignore"):
        d_serv = np.abs(st["in_serv"] - m) / np.abs(st["in_serv"]) / U
    d_pk = dist_u(st["pK"])
    _, lo, hi = midpoint(st["pK"])
    flip = (F(1) - lo) != (F(1) - hi)
    return d_sys, d_serv, d_pk, flip, K


def classify(cls, st, lam, tab, b, idx=Ellipsis):
    """whether the candidates (restated chain st) meet the definition of class cls"""
    K = 11 * b
    one_r, x = cube_x(lam, tab, b)
    pre_cube = (one_r >= 2.0 ** -11 * 1.01) & (x >= 0.3 * 1.01) & (st["pmin"] >= 2.0 ** -40) & \
               (st["pmax"] < 2.0 ** 980) & (st["S"] < 2.0 ** 990)
    bt = block_terms(st, lam, tab, b)
    pre_blk = (bt["one_r"] >= 2.0 ** -10) & (bt["logP"] > -190) & (st["pN"] < 2.0 ** 980) & (bt["zero"] > -150) & \
              (st["pmin"] >= WIN_LO) & (st["S"] < 2.0 ** 990) & (st["pN"] >= 2.0 ** -160)
    d_blk = dist_u(st["pK"])
    if cls == "P":
        return pre_blk & (d_blk < e_blk(b) / 2)
    if cls == "Pf":
        return pre_blk & (bt["one_r"] >= 2.0 ** -9) & (d_blk >= 2 * e_blk(b))
    if cls == "Pz":
        return (zero_edge_case(st, lam, tab, b) != "") & (bt["one_r"] >= 2.0 ** -10) & (st["pmin"] >= WIN_LO)
    d_sys, d_serv, d_pk, flip, _ = cube_dists(st, b)
    if cls in ("C", "Q"):
        return pre_cube & ((d_sys < 32 * K) | (d_serv < 32 * K) | ((d_pk < 64 * K) & flip))
    if cls == "Cf":
        m, _, _ = midpoint(st["in_serv"])
        serv_abs = np.abs(st["in_serv"] - m) / U
        return pre_cube & (d_sys >= 128 * K) & (serv_abs >= 128 * K * st["in_serv"] + 8.0 * K * b) & (d_pk >= 256 * K)
    raise ValueError(cls)


def class_distance(cls, st, lam, tab, b):
    """the distance the fixture records for an entry of class cls (units of u)"""
    if cls in ("P", "Pf", "Pz"):
        return dist_u(st["pK"])
    d_sys, d_serv, d_pk, flip, K = cube_dists(st, b)
    return np.minimum(np.minimum(d_sys, d_serv), np.where(flip, d_pk / 2, np.inf))


# ---- oracle views -----------------------------------------------------------------------------------------------------

def oracle_candidates(oracle, ob, img, r, b):
    """(metrics, status, p_block) of candidate (s, 0, r[s], b[s]) of every server s of img"""
    n = img.S
    s = np.arange(n, dtype=np.int32)
    m, st = oracle.grid_candidates(img, s, np.zeros(n, np.int32), np.asarray(r, np.int32), np.asarray(b, np.int32),
                                   threads=max(1, oracle.hardware_threads()))
    _, st2, pb = ob.grid_candidates_blocking(img, s, np.zeros(n, np.int32), np.asarray(r, np.int32),
                                             np.asarray(b, np.int32), threads=max(1, oracle.hardware_threads()))
    assert np.array_equal(st, st2)
    return m, st, pb


def oracle_chain(oracle, e):
    """(float64 normalised p[] of the oracle, its Analyzer.solve record) for entry e"""
    a = oracle.Analyzer(e["b"], 10 * e["b"], hex_f32(e["alpha"]), hex_f32(e["beta"]), hex_f32(e["gamma"]),
                        hex_f32(e["delta"]), e["in"], e["out"])
    lam = row_lambda(hex_f32(e["arrival"]), e["r"])
    rec = a.solve(lam)
    return a.probabilities(), rec


def stats_from_probabilities(p, N):
    """inSys and inServ of computeStatistics (mm1modelstatedependent.go:44-56) from the oracle's normalised p[]"""
    K = len(p) - 1
    i = np.arange(1, K + 1, dtype=np.float64)
    in_sys = np.cumsum(i * p[1:])                  # sequential, in index order
    sumP = np.cumsum(np.concatenate([[p[0]], p[1:]]))
    return float(in_sys[-1]), float(in_sys[N - 1] + (1.0 - sumP[N]) * N)


# ---- CPU tests --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def fixture():
    return load_fixture()


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


def test_fixture_coverage(fixture):
    """every class is populated, and P and C cover every batch size, r = 1 and r > 1, and at least 4 profiles"""
    E = fixture["entries"]
    count = {c: sum(e["cls"] == c for e in E) for c in CLASSES}
    for c, n in MIN_COUNT.items():
        assert count[c] >= n, (c, count)
    for c in ("P", "C"):
        mine = [e for e in E if e["cls"] == c]
        # P at b = 8192: with 1 - r >= 0.001 (RateRange.Max) p_block <= 0.999^81920 0.001 ~ 2^-128 is subnormal, and a
        # subnormal within E_blk / 2 of a midpoint takes ~2^12 loads to find among the few thousand that remain normal
        want = set(B_VALUES) - ({8192} if c == "P" else set())
        assert {e["b"] for e in mine} >= want, (c, sorted({e["b"] for e in mine}))
        assert {e["r"] == 1 for e in mine} == {True, False}, c
        assert len({(e["alpha"], e["beta"], e["gamma"], e["delta"], e["in"], e["out"]) for e in mine}) >= 4, c
    assert os.path.getsize(FIXTURE) < 1 << 20


def test_zero_edge_cases_present(fixture):
    """the Pz entries hold loads on both sides of the certified zero's threshold and nonzero subnormal p_blocks, each
    case at least 8 times, on the restated chain (whose p[K] / sum the next tests pin to the oracle's)"""
    seen = {"below": 0, "above": 0, "subnormal": 0}
    for e in fixture["entries"]:
        if e["cls"] != "Pz":
            continue
        b = e["b"]
        tab = rate_table(*[hex_f32(e[k]) for k in ("alpha", "beta", "gamma", "delta")], e["in"], e["out"], b)
        lam = np.array([row_lambda(hex_f32(e["arrival"]), e["r"])], dtype=F)
        case = str(zero_edge_case(chain(tab, b, lam), lam, tab, b)[0])
        assert case, e
        seen[case] += 1
        if case == "subnormal":
            assert 0 < int(e["p_block"], 16) < 0x00800000, e
    assert min(seen.values()) >= 8, seen


def test_expected_bits_match_oracle(wva, oracle, ob, fixture):
    """status, every metric and p_block of every entry, bit for bit, from the oracle's grid_candidates and
    grid_candidates_blocking"""
    E = fixture["entries"]
    img = entries_image(wva, E)
    m, st, pb = oracle_candidates(oracle, ob, img, [e["r"] for e in E], [e["b"] for e in E])
    for i, e in enumerate(E):
        assert int(st[i]) == e["status"], (i, e["cls"])
        assert [f32_hex(x) for x in m[i].tolist()] == e["metrics"], (i, e["cls"])
        assert f32_hex(pb[i]) == e["p_block"], (i, e["cls"])
    assert ((st & 0xfe) == 0).all()                 # every entry is a candidate Analyze accepts


def test_restatement_matches_oracle_and_classes_hold(oracle, fixture):
    """the float64 restatement gives the oracle's p[K] / sum bit for bit and its float32 inSys and inServ, and every
    entry meets its class's definition on the oracle's own float64 values"""
    E = fixture["entries"]
    by_key = {}
    for i, e in enumerate(E):
        by_key.setdefault((e["alpha"], e["beta"], e["gamma"], e["delta"], e["in"], e["out"], e["b"]), []).append(i)
    for key, idx in by_key.items():
        e0 = E[idx[0]]
        b = e0["b"]
        tab = rate_table(*[hex_f32(e0[k]) for k in ("alpha", "beta", "gamma", "delta")], e0["in"], e0["out"], b)
        lam = np.array([row_lambda(hex_f32(E[i]["arrival"]), E[i]["r"]) for i in idx], dtype=F)
        st = chain(tab, b, lam)
        for j, i in enumerate(idx):
            e = E[i]
            p, rec = oracle_chain(oracle, e)
            in_sys, in_serv = stats_from_probabilities(p, b)
            assert p[-1] == st["pK"][j], (i, e["cls"])
            assert F(in_sys) == rec["in_system"] == F(st["in_sys"][j]), (i, e["cls"])
            assert F(in_serv) == rec["in_servers"] == F(st["in_serv"][j]), (i, e["cls"])
            assert F(p[-1]) == hex_f32(e["p_block"]), (i, e["cls"])
            one = {k: v[j:j + 1] for k, v in st.items()}
            one.update(pK=np.array([p[-1]]), in_sys=np.array([in_sys]), in_serv=np.array([in_serv]))
            assert classify(e["cls"], one, lam[j:j + 1], tab, b)[0], (i, e["cls"])
            d = class_distance(e["cls"], one, lam[j:j + 1], tab, b)[0]
            if e["dist"] is None:
                assert not math.isfinite(d), (i, d)
            else:
                assert math.isclose(d, e["dist"], rel_tol=1e-9), (i, d, e["dist"])


def test_pair_entries_size_to_their_candidate(oracle, wva, fixture):
    """each Q entry's pair, sized by the oracle, has the entry's replicas and batch size"""
    Q = [e for e in fixture["entries"] if e["cls"] == "Q"]
    img = entries_image(wva, Q)
    pairs, feas, _ = oracle.analyze_pairs(img, threads=max(1, oracle.hardware_threads()))
    assert np.array_equal(pairs.num_replicas, [e["r"] for e in Q])
    assert np.array_equal(pairs.batch_size, [e["b"] for e in Q])
    assert np.array_equal(pairs.acc, np.zeros(len(Q)))
