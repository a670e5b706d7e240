"""CPU: what pair sizing over arrival-rate scenarios (wva_analyze_pairs_loads) relies on, shown with the oracle alone --
TPS-target pairs do not depend on the rate, +0 / -0 / negative rates, the rates the reference still finishes on, and a
numpy restatement of numReplicas from QueueAnalyzer.Size's rateStar.  The helpers here are shared with
test_pairs_loads_gpu.py."""
import numpy as np
import pytest

from test_pairs_plane_cpu import rec_bytes, to_recs

F = np.float32
MIN_INT64 = np.iinfo(np.int64).min


def with_rates(img, rpm):
    """the image with ServerLoadSpec.ArrivalRate = rpm[s] on every server"""
    out = img.shard(0, img.S)
    out.srv_arrival_rpm[:] = np.asarray(rpm, dtype=F)
    return out


def oracle_loads(wva, oracle, img, rpm, threads=None):
    """the reference's records of every pair under every scenario column of rpm [S, n_l]: [S, n_l, A]"""
    threads = threads or oracle.hardware_threads()
    cols = []
    for j in range(rpm.shape[1]):
        allocs, fe, _ = oracle.analyze_pairs(with_rates(img, rpm[:, j]), threads=threads)
        cols.append(to_recs(wva, allocs, fe).reshape(img.S, img.A))
    return np.stack(cols, axis=1)


def pair_n(img, s, a):
    """N of CreateAllocation (allocation.go:81-86)"""
    if img.srv_max_batch[s] > 0:
        return int(img.srv_max_batch[s])
    pi = int(img.srv_model[s]) * img.A + a
    return max(int(img.perf_max_batch[pi]) * int(img.perf_at_tokens[pi]) // int(img.srv_out_tokens[s]), 1)


def rate_star(wva, oracle, img, s, a):
    """rateStar = Size's Analyze(requestRate).Throughput for pair (s, a), or None when Size fails"""
    n = pair_n(img, s, a)
    pi = int(img.srv_model[s]) * img.A + a
    cfg = np.array([(n, 10 * n, img.perf_alpha[pi], img.perf_beta[pi], img.perf_gamma[pi], img.perf_delta[pi],
                     img.srv_in_tokens[s], img.srv_out_tokens[s])], dtype=wva.abi.QUEUE_CONFIG_DTYPE)
    target = np.array([[img.srv_slo_ttft[s], img.srv_slo_itl[s], img.srv_slo_tps[s]]], dtype=F)
    _, metrics, _, status = oracle.queue_size(cfg, target)
    return None if status[0] else F(metrics["throughput"][0])


def go_int(x):
    """Go's int(float64) on amd64: out of range and NaN give MinInt64"""
    x = np.float64(x)
    return int(x) if np.isfinite(x) and -2.0 ** 63 <= x < 2.0 ** 63 else MIN_INT64


def num_replicas(rpm, rstar, min_rep):
    """allocation.go:135-141 for a server without a TPS target"""
    total = F(F(rpm) / F(60))
    return max(go_int(np.ceil(np.float64(total) / np.float64(rstar))), int(min_rep))


def rpm_for_total(total):
    """a float32 rate whose rpm / 60 is exactly `total` in float32, or None (then no float32 rate maps onto it)"""
    total = F(total)
    r0 = F(total * F(60))
    up, dn = r0, r0
    for _ in range(8):
        for r in (up, dn):
            if F(r / F(60)) == total:
                return r
        up, dn = np.nextafter(up, F(np.inf)), np.nextafter(dn, F(-np.inf))
    return None


def boundary_rates(rstar):
    """rates whose rpm / 60 is k * rateStar (k = 1, 2, 4), each with the rates one ulp either side"""
    out = []
    for k in (1, 2, 4):
        r = rpm_for_total(F(k) * rstar)
        if r is not None:
            out += [np.nextafter(r, F(-np.inf)), r, np.nextafter(r, F(np.inf))]
    return np.array(out, dtype=F)


def _image(wva):
    img = wva.synth.make_system(40, 3, seed=91, n_types=2, tps_fraction=0.3, zero_load_fraction=0.0)
    img.srv_keep_acc[:] = 0
    return img


def test_tps_target_pairs_do_not_depend_on_the_rate(wva, oracle):
    img = _image(wva)
    tps = img.srv_slo_tps > 0
    assert tps.sum() >= 5
    rows = []
    for rate in (F(1e-3), F(0.5), F(60.0), F(7e4), F(3e9)):
        allocs, fe, _ = oracle.analyze_pairs(with_rates(img, np.full(img.S, rate)), threads=oracle.hardware_threads())
        rows.append(to_recs(wva, allocs, fe).reshape(img.S, img.A)[tps])
    assert all(rec_bytes(r) == rec_bytes(rows[0]) for r in rows[1:])
    assert (rows[0]["feasible"] == 1).any()


def test_zero_and_negative_rates(wva, oracle):
    img = _image(wva)
    img.srv_min_replicas[:] = np.arange(img.S) % 2
    rpm = np.array([[0.0, -0.0, -1.0, -np.inf, -1e-40]] * img.S, dtype=F)
    recs = oracle_loads(wva, oracle, img, rpm)
    assert rec_bytes(recs[:, 0]) == rec_bytes(recs[:, 1])
    ones = img.srv_min_replicas == 1
    assert (recs[ones, 0]["feasible"] == 1).all() and (recs[ones, 0]["num_replicas"] == 1).all()
    assert (recs[ones, 0]["rho"] == 0).all()
    for j in (2, 3, 4):
        assert (recs[:, j]["feasible"] == 0).all() and (recs[:, j]["acc"] == -1).all()


def test_oracle_finishes_on_extreme_rates(wva, oracle):
    """+Inf and 3e38 overflow int64 in numReplicas (Go gives MinInt64, then MinNumReplicas wins); rates above 2^31
    replicas stay int64"""
    img = _image(wva)
    img.srv_slo_tps[:] = 0.0
    img.srv_min_replicas[:] = np.arange(img.S) % 3
    s, a = next((s, a) for s in range(img.S) for a in range(img.A) if rate_star(wva, oracle, img, s, a))
    rs = rate_star(wva, oracle, img, s, a)
    big = F(F(2.0 ** 33) * rs * F(60))
    rpm = np.array([[np.inf, 3e38, big]] * img.S, dtype=F)
    recs = oracle_loads(wva, oracle, img, rpm)
    for j in range(3):
        want = num_replicas(rpm[s, j], rs, img.srv_min_replicas[s])
        r = recs[s, j, a]
        if r["feasible"]:
            assert r["num_replicas"] == want
    assert num_replicas(rpm[s, 2], rs, 0) > 2 ** 31
    assert num_replicas(np.inf, rs, 2) == 2 and num_replicas(F(3e38), rs, 0) == 0


def test_num_replicas_restatement_on_boundaries(wva, oracle):
    img = _image(wva)
    img.srv_slo_tps[:] = 0.0
    found = 0
    for s, a in [(s, a) for s in range(0, img.S, 7) for a in range(img.A)]:
        rs = rate_star(wva, oracle, img, s, a)
        if rs is None:
            continue
        for k in (1, 2, 4):
            r = rpm_for_total(F(k) * rs)
            if r is not None:
                assert F(r / F(60)) == F(k) * rs
                found += 1
        rates = boundary_rates(rs)
        if not len(rates):
            continue                   # rpm / 60 skips over k * rateStar: no float32 rate lands on it
        sub = img.take([s] * len(rates))
        sub.srv_arrival_rpm[:] = rates
        allocs, fe, _ = oracle.analyze_pairs(sub, threads=oracle.hardware_threads())
        got = to_recs(wva, allocs, fe).reshape(len(rates), img.A)[:, a]
        want = [num_replicas(r, rs, img.srv_min_replicas[s]) for r in rates]
        ok = got["feasible"] == 1
        assert ok.any()
        assert list(got["num_replicas"][ok]) == [w for w, o in zip(want, ok) if o]
    assert found >= 6
