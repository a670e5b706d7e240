"""GPU: the sweep's and the blocking plane's certificates on the candidates of tests/golden/hard_rounding.json, whose
reference float32 results sit on rounding boundaries (classes in test_hard_rounding_cpu.py).

  * plane: every entry bit for bit against the oracle; every P entry listed for an exact chain, no Pf entry listed;
    the whole plane of every image the oracle can afford, else every listed candidate plus 10^4 random ones; one image
    again on a server slice;
  * cube, in every mode of set_certified_tails: status and metrics of every entry and every winner against the oracle;
    every C entry deferred to an exact chain wherever the kernel defers to a list, no Cf entry deferred by default;
  * pair records of the Q entries from both pair kernels, certified tails on and off, against the oracle.

Images hold one server per entry and are grouped by batch size, so that b_max is the group's b.
"""
import numpy as np
import pytest

from test_hard_rounding_cpu import entries_image, f32_hex, groups, load_fixture

pytestmark = pytest.mark.gpu

# set_certified_tails modes: 1 default (scan kernels), 33 scan kernels tuned for 3 blocks per SM, 0 no certificate,
# 3 one thread per candidate, 5 one thread per row, 9 one warp per row, 17 the automatic round-1 choice
MODES = (1, 33, 0, 3, 5, 9, 17)
PLANE_STEPS = 2e9                  # oracle chain steps the whole-plane comparison may cost


def _lists_deferred(mode, b_max):
    """whether this mode's sweep sends an uncertified candidate to the exact-chain list (grid_deferred): the scan
    kernels and one thread per row always do; one warp per row does while its table fits in shared memory
    (wva_b200.cu's wrowMode, restated here); k_grid (modes 3, 17 on small images, and 9 above that limit) runs such
    chains in place.  The caller asserts both outcomes, so a host change to this choice fails the test instead of
    switching its assertion off"""
    if mode in (1, 33, 5):
        return True
    if mode == 9:
        return b_max * 20 + 16 + 8 * (256 + 1 + 1 + 1024) * 8 <= 200 * 1024
    return False


@pytest.fixture(scope="module")
def ob(oracle):
    import oracle_blocking
    oracle_blocking.build()
    oracle_blocking.lib()
    return oracle_blocking


@pytest.fixture(scope="module")
def cases(wva):
    """[(name, image, r_max, b_max, entries)] : one image per batch size, and the pair entries' image"""
    E = load_fixture()["entries"]
    out = []
    for b, idx in sorted(groups(E).items()):
        es = [E[i] for i in idx]
        out.append(("b=%d" % b, entries_image(wva, es), max(e["r"] for e in es), b, es))
    Q = [e for e in E if e["cls"] == "Q"]
    out.append(("pairs", entries_image(wva, Q), max(e["r"] for e in Q), max(e["b"] for e in Q), Q))
    return out


def _threads(oracle):
    return max(1, oracle.hardware_threads())


def _ids(es, R, B):
    """cube index of each entry's candidate (server j of the image or slice, accelerator 0, r, b)"""
    return np.array([(j * R + e["r"] - 1) * B + e["b"] - 1 for j, e in enumerate(es)], dtype=np.int64)


def _mismatch(got, want):
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    bad = np.flatnonzero(~same)
    return None if len(bad) == 0 else int(bad[0])


def _decode(idx, R, B):
    idx = np.asarray(idx, dtype=np.int64)
    return (idx // (B * R)).astype(np.int32), ((idx // B) % R + 1).astype(np.int32), (idx % B + 1).astype(np.int32)


def _check_plane_ids(ob, oracle, img, p, ids, R, B, first=0):
    s, r, b = _decode(ids, R, B)
    _, _, want = ob.grid_candidates_blocking(img, s + first, np.zeros(len(ids), np.int32), r, b, threads=_threads(oracle))
    bad = _mismatch(p[ids], want)
    assert bad is None, (int(ids[bad]), float(p[ids][bad]), float(want[bad]))


def _plane_cost(img, R, B):
    return img.S * R * 11.0 * B * (B + 1) / 2


def _check_plane(ob, oracle, name, img, R, B, es, p, exact, first=0):
    ids = _ids(es, R, B)
    cls = np.array([e["cls"] for e in es])
    assert [f32_hex(x) for x in p[ids]] == [e["p_block"] for e in es], name
    _check_plane_ids(ob, oracle, img, p, ids, R, B, first)
    listed = np.isin(ids, exact)
    assert listed[cls == "P"].all(), (name, ids[(cls == "P") & ~listed])
    assert not listed[cls == "Pf"].any(), (name, ids[(cls == "Pf") & listed])
    return int((cls == "P").sum()), int((cls == "Pf").sum())


def test_plane_hard_candidates(wva, oracle, ob, ctx, cases):
    """p_block of every entry, the P entries listed and the Pf entries decided by the closed form; the whole plane, or
    every listed candidate and 10^4 random ones"""
    rng = np.random.default_rng(11)
    n_p = n_pf = closed = 0
    for name, img, R, B, es in cases:
        ctx.upload(img)
        ctx.analyze_grid(R, B, want_cube=False)
        p = ctx.grid_blocking()
        counts = ctx.grid_blocking_counts()
        exact, n_exact = ctx.grid_blocking_exact()
        assert n_exact == len(exact), name
        a, b = _check_plane(ob, oracle, name, img, R, B, es, p, exact)
        n_p, n_pf, closed = n_p + a, n_pf + b, closed + counts["closed_form"]
        if len(p) <= 10 ** 6 and _plane_cost(img, R, B) <= PLANE_STEPS:
            _, _, want = ob.grid_plane_blocking(img, R, B, threads=_threads(oracle))
            bad = _mismatch(p, want)
            assert bad is None, (name, bad, float(p[bad]), float(want[bad]))
        else:
            _check_plane_ids(ob, oracle, img, p, exact.astype(np.int64), R, B)
            _check_plane_ids(ob, oracle, img, p, np.sort(rng.choice(len(p), min(len(p), 10 ** 4), replace=False)), R, B)
        print("%s: blocking counts %s" % (name, counts))
    assert n_p >= 64 and n_pf >= 16
    assert closed >= n_pf


def test_plane_hard_candidates_server_slice(wva, oracle, ob, ctx, cases):
    """one image's plane on a server slice: ids are relative to the slice, the same entries are listed"""
    name, img, R, B, es = max(cases[:-1], key=lambda c: sum(e["cls"] == "P" for e in c[4]) if c[3] <= 512 else -1)
    first, count = 1, img.S - 2
    assert count >= 2
    ctx.upload(img)
    try:
        ctx.set_shard(first, count)
        ctx.analyze_grid(R, B, want_cube=False)
        p = ctx.grid_blocking()
        exact, _ = ctx.grid_blocking_exact()
    finally:
        ctx.upload(img)
    assert len(p) == count * R * B
    _check_plane(ob, oracle, name, img, R, B, es[first:first + count], p, exact, first=first)
    _, _, want = ob.grid_plane_blocking(img, R, B, s0=first, s1=first + count, threads=_threads(oracle))
    assert _mismatch(p, want) is None, name


_WINNERS = {}
WINNER_STEPS = 5e9                 # above this the oracle's sweep takes most of a minute: the uncertified sweep stands in


def _reference_winners(oracle, ctx, mode, name, img, R, B):
    """every server's winner from the oracle's sweep; for the b = 8192 image from the sweep with certified tails off
    (every candidate an exact chain, which the rest of the suite checks against the oracle)"""
    if _plane_cost(img, R, B) <= WINNER_STEPS:
        if name not in _WINNERS:
            _WINNERS[name] = oracle.analyze_grid(img, R, B, want_cube=False, threads=_threads(oracle))[0]
        return _WINNERS[name]
    ctx.set_certified_tails(0)
    try:
        return ctx.analyze_grid(R, B)[0]
    finally:
        ctx.set_certified_tails(mode)


@pytest.mark.parametrize("mode", MODES)
def test_cube_hard_candidates(wva, oracle, ctx, cases, mode):
    """status and metrics of every entry and every server's winner against the oracle; C entries deferred wherever
    the mode's kernel defers, Cf entries certified by the default sweep"""
    ctx.set_certified_tails(mode)
    try:
        for name, img, R, B, es in cases:
            ctx.upload(img)
            want_best = _reference_winners(oracle, ctx, mode, name, img, R, B)
            best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
            ids = _ids(es, R, B)
            assert [int(x) for x in status[ids]] == [e["status"] for e in es], (name, mode)
            got = [[f32_hex(x) for x in cube[i].tolist()] for i in ids]
            bad = [j for j, e in enumerate(es) if got[j] != e["metrics"]]
            assert not bad, (name, mode, bad[:4], es[bad[0]]["cls"])
            assert best.tobytes() == want_best.tobytes(), (name, mode)
            cls = np.array([e["cls"] for e in es])
            deferred, n_def = ctx.grid_deferred()
            assert n_def == len(deferred), (name, mode)
            listed = np.isin(ids, deferred.astype(np.int64))
            hard = (cls == "C") | (cls == "Q")
            # both ways, so that the test follows the host's kernel choice: a mode that defers lists every hard entry,
            # a certified mode that runs k_grid lists nothing (its uncertified chains run in place, and only the
            # results above check cert_eval there)
            if mode & 1 and _lists_deferred(mode, B):
                assert listed[hard].all(), (name, mode, ids[hard & ~listed])
            elif mode & 1:
                assert n_def == 0, (name, mode, n_def)
            if mode == 1:
                assert not listed[cls == "Cf"].any(), (name, ids[(cls == "Cf") & listed])
    finally:
        ctx.set_certified_tails(1)
        ctx.upload(cases[0][1])


def test_pair_records_hard_candidates(wva, oracle, ctx, cases):
    """both pair kernels, certified tails on and off, against Server.Calculate on every Q entry's pair"""
    name, img, _, _, es = cases[-1]
    want, wfe, _ = oracle.analyze_pairs(img, threads=_threads(oracle))
    assert list(want.num_replicas) == [e["r"] for e in es] and list(want.batch_size) == [e["b"] for e in es]
    try:
        for cert in (1, 0):
            for warp_max in (0, 1 << 22):
                ctx.set_certified_tails(cert)
                ctx.pairs_set_warp_max(warp_max)
                ctx.upload(img)
                got, gfe = ctx.analyze_pairs()
                assert np.array_equal(gfe, wfe), (cert, warp_max)
                ok, field = got.equal_bits(want)
                assert ok, (cert, warp_max, field)
    finally:
        ctx.set_certified_tails(1)
        ctx.pairs_set_warp_max(1 << 22)
