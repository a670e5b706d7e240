"""GPU: pair sizing at BinarySearch's edges (pair_edge_cases.py) against the oracle on every pair kernel, with device-side
evidence that size_pair_warp's branches ran; and the sweep's SLO test at equality.  Records are compared bit for bit
(feasibility, replicas, batch, six floats, a NaN equal to a NaN).  Every switch is put back to its default at the end."""
import numpy as np
import pytest

import pair_edge_cases as pc
from test_pairs_loads_cpu import oracle_loads
from test_pairs_plane_cpu import oracle_plane, rec_bytes, to_recs
from test_state_trace_gpu import DEFAULTS

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture
def restore(ctx):
    yield ctx
    ctx.pairs_set_pstore(DEFAULTS["pstore"])
    ctx.pairs_set_warp_max(DEFAULTS["warp_max"])
    ctx.set_certified_tails(DEFAULTS["certified"])


@pytest.fixture(scope="module")
def edge(wva, oracle):
    img, items = pc.edge_image(wva, oracle)
    allocs, fe, _ = pc.oracle_pairs(oracle, img)
    return img, items, to_recs(wva, allocs, fe), pc.restated(wva, oracle, img)


def _resident(wva, ctx, img):
    ctx.upload(img)
    allocs, fe = ctx.analyze_pairs()
    return to_recs(wva, allocs, fe)


def _first_bad(got, want):
    for i in range(len(want)):
        if rec_bytes(got[i:i + 1]) != rec_bytes(want[i:i + 1]):
            return i
    return None


@pytest.mark.parametrize("cert", [1, 0])
@pytest.mark.parametrize("pstore", [0, 1, 2, 3])
def test_warp_kernel_matches_oracle(wva, restore, edge, pstore, cert):
    """k_pairs_warp with and without the chain-value buffer and shared-memory tables, certified tails on and off: every
    record equals the oracle's; the per-pair round count is the restatement's; uncertain nodes are re-evaluated exactly
    on the N = 2 / 8 top fixtures with the certificate on; the trailing Analyze's guess misses and its x1 cache hits"""
    ctx = restore
    img, items, want, rs = edge
    ctx.set_certified_tails(cert)
    ctx.pairs_set_pstore(pstore | 4)
    got = _resident(wva, ctx, img)
    assert _first_bad(got, want) is None, (pstore, cert, _first_bad(got, want))
    dbg = ctx.pair_debug()
    rounds = (dbg[:, 1] >> np.uint64(32)).astype(np.int64)
    pend = ((dbg[:, 0] >> np.uint64(36)) & np.uint64(0xff)).astype(np.int64)
    expect = np.array([rs[s, a][0].rounds for s in range(img.S) for a in range(img.A)])
    bad = np.flatnonzero(rounds != expect)
    assert len(bad) == 0, [(int(i) // img.A, int(i) % img.A, int(rounds[i]), int(expect[i])) for i in bad[:8]]
    if cert:
        # every walked midpoint outside cert_eval's preconditions is a node whose speculative evaluation was uncertain
        for s, it in enumerate(items):
            if it.cls == "top" and it.N in pc.CERT_FAIL_NS:
                sz, an, c = rs[s, s % img.A]
                s_n = pc.ac.cfg_rate_table(c)[-1]
                need = sum(not pc.cert_precondition(x, s_n, it.N) for x in sz.paths[it.kind].mids)
                assert need > 0 and pend[s * img.A + s % img.A] >= need, (s, it.N, need, pend[s * img.A + s % img.A])
    cnt = ctx.pair_counters()
    assert cnt["rounds_sum"] == expect.sum() and cnt["rounds_max"] == expect.max() == 26
    miss, reach = 0, 0
    for s in range(img.S):
        for a in range(img.A):
            if want["feasible"][s * img.A + a] and not pc.zero_load(img, s):
                sz, an, c = rs[s, a]
                reach += 1
                miss += pc.guess_miss(an, sz, pc.total_rate(img, s), img.srv_min_replicas[s])[0]
    no_cache = cnt["trailing"] - 100 * miss
    assert miss > 0 and 0 <= no_cache < reach, (cnt["trailing"], miss, reach)


def test_uncertain_nodes_only_with_certified_tails(wva, restore, edge):
    """pendEvals with certified tails off is nowhere above its value with them on"""
    ctx = restore
    img = edge[0]
    got = {}
    for cert in (1, 0):
        ctx.set_certified_tails(cert)
        ctx.pairs_set_pstore(4)
        _resident(wva, ctx, img)
        got[cert] = ((ctx.pair_debug()[:, 0] >> np.uint64(36)) & np.uint64(0xff)).astype(np.int64)
    assert (got[0] <= got[1]).all() and got[1].sum() > got[0].sum()


def test_thread_kernel_matches_oracle(wva, restore, edge):
    """k_pairs (one thread per pair, warp_max 0)"""
    ctx = restore
    img, _, want, _ = edge
    ctx.pairs_set_warp_max(0)
    got = _resident(wva, ctx, img)
    assert _first_bad(got, want) is None, _first_bad(got, want)


def test_analyze_beside_the_sweep_matches_oracle(wva, restore, edge):
    """wva_analyze: pair sizing beside the candidate sweep"""
    ctx = restore
    img, _, want, _ = edge
    ctx.upload(img)
    ctx.analyze(4, 64)
    allocs, fe = ctx.pairs_fetch()
    got = to_recs(wva, allocs, fe)
    assert _first_bad(got, want) is None, _first_bad(got, want)


def test_batches_match_oracle(wva, oracle, restore, edge):
    """analyze_pairs_batches over {1} and every fixture N with N - 1 and N + 1: each column equals the oracle under that
    override, and column N equals the resident record on the servers whose own override is N"""
    ctx = restore
    img, _, want, _ = edge
    ns = sorted({int(n) for n in img.srv_max_batch})
    batch = sorted({1} | {n + d for n in ns for d in (-1, 0, 1) if n + d >= 1})
    ctx.upload(img)
    plane, _ = ctx.analyze_pairs_batches(batch)
    w = oracle_plane(wva, oracle, img, batch)
    bad = [b for j, b in enumerate(batch) if rec_bytes(plane[:, j]) != rec_bytes(w[:, j])]
    assert not bad, bad
    for j, b in enumerate(batch):
        own = np.repeat(img.srv_max_batch == b, img.A)
        if own.any():
            assert rec_bytes(plane[own, j]) == rec_bytes(want[own]), b


def test_loads_match_oracle(wva, oracle, restore, edge):
    """analyze_pairs_loads over the uploaded rate, 0.5x and 4x it, and the arrival copies' boundary rates on every
    server: each column equals the oracle on that column's image"""
    ctx = restore
    img, items, _, _ = edge
    base = img.srv_arrival_rpm.astype(F)
    rates = sorted({F(it.arrival) for it in items if it.arrival is not None})
    cols = [base, F(0.5) * base, F(4.0) * base] + [np.full(img.S, r, dtype=F) for r in rates]
    rpm = np.stack(cols, axis=1).astype(F)
    ctx.upload(img)
    plane, _ = ctx.analyze_pairs_loads(rpm)
    w = oracle_loads(wva, oracle, img, rpm)
    bad = [j for j in range(rpm.shape[1]) if rec_bytes(plane[:, j]) != rec_bytes(w[:, j])]
    assert not bad, bad


# ---- the sweep's SLO test at equality ----------------------------------------------------------------------------------

SWEEP_MODES = (1, 33, 0, 3, 5, 9, 17)
R_MAX, B_MAX = 8, 256


def _sweep_images(wva, oracle):
    img = wva.synth.make_system(64, 3, seed=4301, n_types=3, tps_fraction=0.0, zero_load_fraction=0.0)
    best, _, _, _ = oracle.analyze_grid(img, R_MAX, B_MAX, want_cube=False, threads=oracle.hardware_threads())
    won = np.flatnonzero(best["acc"] >= 0)
    assert len(won) >= 40
    out = {}
    for name, step in (("equal", None), ("below", -np.inf), ("above", np.inf)):
        im = img.shard(0, img.S)
        for s in won:
            if s % 2 == 0:
                v = F(best["ttft"][s])
                im.srv_slo_ttft[s] = v if step is None else np.nextafter(v, F(step))
            else:
                v = F(best["itl"][s])
                im.srv_slo_itl[s] = v if step is None else np.nextafter(v, F(step))
        out[name] = im
    return out, won


def test_sweep_slo_at_equality(wva, oracle, restore):
    """each server with a winner gets its winner's own TTFT (even servers) or ITL (odd) as the SLO, exactly and one ulp
    either side: winners and status bytes equal the oracle's in every sweep mode, and the oracle's winner changes
    between 'equal' and 'one ulp below' on most servers"""
    ctx = restore
    images, won = _sweep_images(wva, oracle)
    want = {k: oracle.analyze_grid(im, R_MAX, B_MAX, want_cube=True, threads=oracle.hardware_threads())
            for k, im in images.items()}
    for k, im in images.items():
        ctx.upload(im)
        for mode in SWEEP_MODES:
            ctx.set_certified_tails(mode)
            best, _, status = ctx.analyze_grid(R_MAX, B_MAX, want_cube=True)
            assert np.array_equal(status, want[k][2]), (k, mode, int(np.flatnonzero(status != want[k][2])[0]))
            assert best.tobytes() == want[k][0].tobytes(), (k, mode)
    eq, lo = want["equal"][0], want["below"][0]
    changed = sum(eq[s].tobytes() != lo[s].tobytes() for s in won)
    assert changed >= len(won) * 3 // 4, (changed, len(won))
