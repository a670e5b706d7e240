"""CPU side of the pair-sizing edge tests (test_pair_edges_gpu.py): every fixture of pair_edge_cases.py reaches the class it
is built for, the float32 restatement of BinarySearch agrees with the oracle's, and the oracle terminates on the image
with its records nil exactly where the class says.  No device is needed."""
import numpy as np
import pytest

import analyzer_api_cases as ac
import pair_edge_cases as pc

F = np.float32


@pytest.fixture(scope="module")
def edge(wva, oracle):
    img, items = pc.edge_image(wva, oracle)
    return img, items, pc.restated(wva, oracle, img)


def _targeted(edge):
    img, items, rs = edge
    for s, it in enumerate(items):
        sz, an, c = rs[s, s % pc.A]
        yield s, it, sz, an, c


def test_restatement_equals_oracle_binary_search(edge):
    """on every pair of the image, each search's (x, ind) is the oracle's BinarySearch result"""
    img, items, rs = edge
    n = 0
    for (s, a), (sz, an, c) in rs.items():
        lmin, lmax, _ = ac.lambda_range(c)
        for k, p in sz.paths.items():
            if p is None:
                continue
            x, ind, err = an.binary_search(k, lmin, lmax, F((img.srv_slo_ttft, img.srv_slo_itl)[k][s]))
            assert err == 0 and (x, ind) == (p.x, p.ind), (s, a, k)
            n += 1
    assert n > len(items) * 2


def test_edge_classes_reach_their_outcome(edge):
    """the edge classes end where EDGE_OUTCOME says, except NaN: Size skips a NaN target (`target > 0` is false), so it
    sizes at lambdaMax as with the target off"""
    seen = set()
    for s, it, sz, an, c in _targeted(edge):
        if it.cls not in ac.EDGE_CLASSES:
            continue
        lmin, lmax, _ = ac.lambda_range(c)
        p = sz.paths[it.kind]
        if it.cls == "nan":
            assert p is None and sz.rounds == 0 and sz.lam == lmax, s
            x, ind, err = an.binary_search(it.kind, lmin, lmax, F(np.nan))
            assert err == 0 and ac.edge_outcome_ok("nan", x, ind, lmin, lmax)
        else:
            assert ac.edge_outcome_ok(it.cls, p.x, p.ind, lmin, lmax), (s, it.cls, p.x, p.ind)
            assert p.iters == 0 or it.cls == "inside"
        seen.add((it.N, it.kind, it.cls))
    assert len(seen) == 9 + 4 * 18          # N = 1 has TTFT classes only


def test_depth_targets_end_at_their_depth(edge):
    """target = y(x_d): exactly d iterations, ending on x_d, with every round boundary of the kernel covered"""
    rounds = set()
    for s, it, sz, an, c in _targeted(edge):
        if not it.cls.startswith("depth"):
            continue
        d = int(it.cls[5:])
        p = sz.paths[it.kind]
        assert p.iters == d and p.ind == 0 and not p.memo, (s, d, p.iters)
        rounds.add((d, pc.kernel_rounds(d)))
    assert {r for _, r in rounds} == {1, 2, 3, 4}
    assert {(3, 1), (4, 2), (7, 2), (8, 3), (11, 3), (12, 4)} <= rounds


def test_gap_targets_collapse_and_run_the_budget(edge):
    """gap and mixed targets: 100 iterations, the last interval two adjacent float32 values, the memo used; beside them
    the mixed pairs' ITL search ends in round 1"""
    n = 0
    for s, it, sz, an, c in _targeted(edge):
        if it.cls == "gap" or it.cls.startswith("mixed"):
            p = sz.paths[0]
            lo, hi = p.ivals[-1]
            assert p.iters == pc.MAXIT and p.memo and np.nextafter(lo, F(np.inf)) == hi, s
            assert not ac.within_tolerance(an.eval(0, p.x), F(img_slo(edge, s, 0)))
            assert sz.rounds == pc.kernel_rounds(pc.MAXIT) == 26
            n += 1
        if it.cls.startswith("mixed"):
            q = sz.paths[1]
            assert q.iters == 0 and q.ind == (0 if it.cls == "mixed_at_min" else 1), s
    assert n >= 30
    near_top = [it for s, it, sz, an, c in _targeted(edge) if it.cls == "gap" and
                sz.paths[0].x > ac.lambda_range(c)[1] * F(0.999)]
    assert near_top


def img_slo(edge, s, k):
    img = edge[0]
    return (img.srv_slo_ttft, img.srv_slo_itl)[k][s]


def test_tolerance_and_budget_pairs(edge):
    """TOL_EDGE's ITL searches return lambdaMin with ind 0 (a quotient of exactly 1e-6); BUDGET_CFG's TTFT search runs
    all 100 iterations without meeting the tolerance"""
    kinds = set()
    for s, it, sz, an, c in _targeted(edge):
        if it.cls == "tol":
            p = sz.paths[1]
            assert (p.x, p.ind, p.iters) == (ac.lambda_range(c)[0], 0, 0), s
            kinds.add("tol")
        if it.cls == "budget":
            p = sz.paths[0]
            assert p.iters == pc.MAXIT and not ac.within_tolerance(an.eval(0, p.x), F(ac.BUDGET_TARGETS[0]))
            kinds.add("budget")
    assert kinds == {"tol", "budget"}


def test_speculative_nodes_fail_the_certificate_near_the_top(edge):
    """the N = 2 and 8 top fixtures visit speculative nodes where cert_eval's preconditions fail (M (1 - r) < 0.3), so
    the certificate must fail there; N = 48 and 200 keep them over the same walk"""
    fails = {}
    for s, it, sz, an, c in _targeted(edge):
        if it.cls != "top":
            continue
        lmin, lmax, _ = ac.lambda_range(c)
        p = sz.paths[it.kind]
        assert p.iters >= 4, s                   # the walk goes past round 1, towards lambdaMax
        s_n = ac.cfg_rate_table(c)[-1]
        xs = pc.speculative_nodes(p, lmin, lmax)
        bad = sum(not pc.cert_precondition(x, s_n, it.N) for x in xs)
        fails.setdefault(it.N, []).append(bad)
    for N in pc.CERT_FAIL_NS:
        assert all(b > 0 for b in fails[N]), (N, fails[N])
    for N in (48, 200):
        assert all(b == 0 for b in fails[N]), (N, fails[N])
    assert not pc.cert_precondition(F(1.0), F(2.0), 1)                      # N = 1: no certificate at all


def test_round_trip_at_lambda_max_never_exceeds_rate_max(edge):
    """a search that ends at lambdaMax (out_max, +Inf, at_max, in_max) sizes at requestRate = (RateRange.Max / 1000) *
    1000, which is RateRange.Max itself: RateRange.Max is a float32 product by 1000, and for such a value the quotient
    by 1000 multiplied back is exact.  So Size's `requestRate > rateMax` test never fires after such a search; it is
    checked here on every fixture and on a million random rates across the float32 range rates take"""
    n = 0
    for s, it, sz, an, c in _targeted(edge):
        if it.cls in ("out_max", "inf", "at_max", "in_max"):
            _, lmax, rmax = ac.lambda_range(c)
            assert sz.lam == lmax and sz.request == rmax and not sz.nil, s
            n += 1
    assert n >= 80
    rng = np.random.default_rng(7)
    v = np.exp(rng.uniform(np.log(1e-30), np.log(1e30), 1_000_000)).astype(F)
    with np.errstate(all="ignore"):
        rmax = (v * F(1000)).astype(F)
        back = ((rmax / F(1000)).astype(F) * F(1000)).astype(F)
    fin = np.isfinite(rmax)
    assert (back[fin] == rmax[fin]).all()


def test_oracle_records_nil_where_the_class_says(wva, oracle, edge):
    """the oracle sizes every pair of the image; its record is nil exactly where the restated Size fails (and the
    targeted pair: out_min of either kind, and nowhere else)"""
    img, items, rs = edge
    _, fe, _ = pc.oracle_pairs(oracle, img)
    for (s, a), (sz, an, c) in rs.items():
        assert bool(fe[s * img.A + a]) == (not sz.nil), (s, a)
    for s, it, sz, an, c in _targeted(edge):
        assert sz.nil == (it.cls == "out_min"), (s, it.cls)
    assert 0 < int(fe.sum()) < len(fe)


def test_arrival_copies_step_the_replica_counts(oracle, edge):
    """the arrival copies put totalRate / rateStar and totalRate / guess on integers and one ulp either side: the
    kernel's guess misses on some of them and not on others"""
    img, items, rs = edge
    miss = []
    for s, it in enumerate(items):
        if it.arrival is None:
            continue
        sz, an, c = rs[s, s % pc.A]
        miss.append(pc.guess_miss(an, sz, pc.total_rate(img, s), img.srv_min_replicas[s])[0])
    assert len(miss) >= 24 and any(miss) and not all(miss)
