"""GPU parity at the sizes the speed claims are made on (VERDICT r01 item 1).

Everything here compares the CUDA path with the ORACLE (the CPU restatement of the reference API), never
GPU mode against GPU mode:

  * config 2: the entire 4 194 304-candidate cube, status bytes and winners;
  * configs 3, 4 (2 000-server slice) and 5 (A = 16 slice), generated exactly as bench.py generates them and
    swept by bench.py's default path (k_scan_prep -> k_scan_cert || k_scan_lean + the deferred exact-chain
    kernels): >= 1e6 random candidates, EVERY candidate the sweep handed to the exact-chain
    kernels, and every server's winner (its own record, plus an exhaustive proof that no candidate with a
    smaller key is feasible according to the oracle);
  * 1e7 random QueueAnalyzer.Analyze requests in certified mode, including the edges of the certificate's
    preconditions (r -> 0.9995, M(1-r) -> 0.3, K -> 2^20);
  * the un-tamed generator of SURVEY 8(d) (out_tokens from 1, no bound on N = maxBatch*atTokens/outTokens,
    reference pkg/core/allocation.go:85).

The oracle runs on all host threads of the box (the per-candidate work is independent; results do not
depend on the thread count).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
F = np.float32


def _threads(oracle):
    return max(1, oracle.hardware_threads())


def test_config2_entire_cube_vs_oracle(wva, oracle, ctx):
    """every one of the 4 194 304 candidates of BASELINE config 2, bit for bit, in the default (automatic) mode"""
    img, c = wva.synth.baseline_config(2)
    R, B = c["r_max"], c["b_max"]
    ctx.upload(img)
    best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
    o_best, o_cube, o_status, _ = oracle.analyze_grid(img, R, B, want_cube=True, threads=_threads(oracle))
    assert np.array_equal(status, o_status)
    assert cube.tobytes() == o_cube.tobytes()
    assert best.tobytes() == o_best.tobytes()
    assert int((status & 1).sum()) > 100000 and int(((status & 0xfe) == 0).sum()) > 1000000


def _decode(idx, A, R, B):
    b = (idx % B + 1).astype(np.int32)
    r = ((idx // B) % R + 1).astype(np.int32)
    pair = idx // (B * R)
    return (pair // A).astype(np.int32), (pair % A).astype(np.int32), r, b


def _check_sweep_against_oracle(wva, oracle, ctx, img, first, count, R, B, n_random, seed, also_fused=False):
    """Sweep servers [first, first+count) of `img` on the GPU (cube + status + winners) and check against the oracle:
    random candidates, all deferred candidates, and the winners exhaustively.  Returns counters for the report.
    also_fused: sweep a second time the way a repeated reconcile does when the deferred list is long (no stop at the host
    between the kernels, exact chains on SMs of their own): same bytes, and the oracle checks run on that second result."""
    th = _threads(oracle)
    A = img.A
    ctx.upload(img)
    ctx.set_shard(first, count)
    ctx.grid_set_fused(False)
    best, cube, status = ctx.analyze_grid(R, B, want_cube=True)
    assert ctx.grid_last_fused() == 0
    ctx.grid_set_fused(True)
    if also_fused:
        n0 = ctx.grid_list_sizes()["deferred"]
        assert n0 > 4096, "shard too small for the fused flow"
        best2, cube2, status2 = ctx.analyze_grid(R, B, want_cube=True)
        assert ctx.grid_last_fused() == 1
        assert ctx.grid_list_sizes()["deferred"] == n0
        assert best2.tobytes() == best.tobytes() and status2.tobytes() == status.tobytes() and cube2.tobytes() == cube.tobytes()
        best, cube, status = best2, cube2, status2
    lists = ctx.grid_list_sizes()
    deferred, n_def = ctx.grid_deferred(cap=1 << 24)
    assert n_def == len(deferred) == lists["deferred"]
    ncand = count * A * R * B
    assert len(cube) == ncand
    # (1) random candidates + (2) every deferred candidate
    rng = np.random.default_rng(seed)
    idx = np.unique(np.concatenate([rng.integers(0, ncand, n_random).astype(np.uint64), deferred]))
    s, a, r, b = _decode(idx.astype(np.int64), A, R, B)
    o_m, o_st = oracle.grid_candidates(img, s + first, a, r, b, threads=th)
    assert np.array_equal(o_st, status[idx.astype(np.int64)])
    assert o_m.tobytes() == cube[idx.astype(np.int64)].tobytes()
    # (3) winners
    (ls, la, lr), proof = prove_winners(wva, oracle, img, first + np.arange(count), best, R, B)
    # the GPU's own feasibility flags agree with that (cheap cross-check of the status cube)
    feas = (status & 1).reshape(count, A, R, B)
    assert int(feas[ls, la, lr].sum()) == 0
    ctx.set_shard(0, img.S)
    return dict(candidates=ncand, checked=len(idx), deferred=int(n_def), winners=int((best["acc"] >= 0).sum()),
                proof_candidates=proof, literal=lists["literal"])


def _row_values(oracle, img, R, srv):
    """oracle.grid_row_values of the listed servers, one call per run of consecutive ones -> [len(srv), A, R]"""
    out = np.empty((len(srv), img.A, R), dtype=F)
    for run in np.split(np.arange(len(srv)), np.flatnonzero(np.diff(srv) != 1) + 1):
        s0 = int(srv[run[0]])
        out[run] = oracle.grid_row_values(img, R, s0, s0 + len(run))
    return out


def prove_winners(wva, oracle, img, srv, best, R, B):
    """The sweep records `best` of servers `srv` (indices into img) against the oracle: each winner's own record, and no
    candidate with a smaller (value, a, r, b) key is feasible according to the oracle (a server without a winner has no
    feasible candidate at all).  Returns the (server position, a, r - 1) of the rows that precede a winner as a whole,
    and how many candidates the proof evaluated."""
    th = _threads(oracle)
    A = img.A
    srv = np.asarray(srv, dtype=np.int64)
    # own record ...
    has = best["acc"] >= 0
    ws = np.flatnonzero(has).astype(np.int32)
    w_m, w_st = oracle.grid_candidates(img, srv[ws], best["acc"][ws], best["replicas"][ws], best["batch"][ws], threads=th)
    assert (w_st == (wva.abi.CAND_OK | wva.abi.CAND_FEASIBLE)).all()
    assert np.array_equal((w_m["avg_wait_time"] + w_m["avg_prefill_time"]).astype(F).view(np.uint32), best["ttft"][ws].view(np.uint32))
    assert np.array_equal(w_m["avg_token_time"].view(np.uint32), best["itl"][ws].view(np.uint32))
    assert np.array_equal(w_m["rho"].view(np.uint32), best["rho"][ws].view(np.uint32))
    vals = _row_values(oracle, img, R, srv)                                # [len(srv), A, R]
    wv = vals[ws, best["acc"][ws], best["replicas"][ws] - 1]
    assert np.array_equal(wv.view(np.uint32), best["value"][ws].view(np.uint32))
    # ... and no candidate with a smaller (value, a, r, b) key is feasible according to the oracle
    a_ix = np.arange(A, dtype=np.int64)[None, :, None]
    r_ix = np.arange(R, dtype=np.int64)[None, None, :]
    rowkey = a_ix * R + r_ix                                               # (a, r) lexicographic rank
    v_win = np.where(has, best["value"], np.inf).astype(F)[:, None, None]
    k_win = np.where(has, best["acc"].astype(np.int64) * R + (best["replicas"] - 1), A * R)[:, None, None]
    with np.errstate(invalid="ignore"):
        lower = (vals < v_win) | ((vals == v_win) & (rowkey < k_win))      # NaN-valued rows are never selected
    ls, la, lr = np.nonzero(lower)
    rows_s = np.concatenate([srv[ls], srv[ws]]).astype(np.int32)
    rows_a = np.concatenate([la, best["acc"][ws]]).astype(np.int32)
    rows_r = np.concatenate([lr + 1, best["replicas"][ws]]).astype(np.int32)
    b_lo = np.ones(len(rows_s), dtype=np.int32)
    b_hi = np.concatenate([np.full(len(ls), B), best["batch"][ws] - 1]).astype(np.int32)
    nf = oracle.grid_rows_feasible(img, rows_s, rows_a, rows_r, b_lo, b_hi, threads=th)
    assert int(nf.sum()) == 0, "the oracle finds a feasible candidate that precedes a GPU winner"
    return (ls, la, lr), int((b_hi - b_lo + 1).clip(min=0).sum())


def test_config3_sweep_vs_oracle(wva, oracle, ctx):
    """BASELINE config 3 (bench.py's default workload): 1 000 servers x 8 accelerators x 64 x 512, swept in
    250-server shards (so that the host copy of the cube stays at 2.2 GB) by the default sweep kernels + deferred kernels."""
    img, c = wva.synth.baseline_config(3)
    tot = dict(checked=0, deferred=0, winners=0, proof_candidates=0)
    for first in range(0, img.S, 250):
        rep = _check_sweep_against_oracle(wva, oracle, ctx, img, first, 250, c["r_max"], c["b_max"], 260_000, seed=30 + first)
        for k in tot:
            tot[k] += rep[k]
    assert tot["checked"] >= 1_000_000 and tot["winners"] > 300 and tot["deferred"] > 0
    print("config 3:", tot)


def test_config3_fused_sweep_vs_oracle(wva, oracle, ctx):
    """500 servers of config 3 defer ~6 600 candidates: the second sweep takes the flow bench.py's steps take after the
    first one (all kernels launched without a host round trip, chain kernel on its own SMs); byte-equal to the
    stop-and-go sweep, and checked against the oracle like the others."""
    img, c = wva.synth.baseline_config(3)
    rep = _check_sweep_against_oracle(wva, oracle, ctx, img, 250, 500, c["r_max"], c["b_max"], 200_000, seed=35, also_fused=True)
    assert rep["deferred"] > 4096 and rep["winners"] > 100
    print("config 3, fused flow:", rep)


def test_config4_slice_vs_oracle(wva, oracle, ctx):
    """2 000 servers of BASELINE config 4, generated exactly as `bench.py --config 4` generates it."""
    c = wva.synth.CONFIGS[4]
    img = wva.synth.make_system(c["S"], c["A"], seed=4, n_types=c["T"])
    tot = dict(checked=0, deferred=0, winners=0, proof_candidates=0)
    for first in (0, 250, 5000, 5250, 9000, 9250, 9500, 9750):
        rep = _check_sweep_against_oracle(wva, oracle, ctx, img, first, 250, c["r_max"], c["b_max"], 130_000, seed=40 + first)
        for k in tot:
            tot[k] += rep[k]
    assert tot["checked"] >= 1_000_000 and tot["winners"] > 600
    print("config 4 slice:", tot)


def test_config5_slice_vs_oracle(wva, oracle, ctx):
    """1 000 servers of BASELINE config 5 (100 000 servers x 16 accelerators)."""
    c = wva.synth.CONFIGS[5]
    img = wva.synth.make_system(c["S"], c["A"], seed=5, n_types=c["T"])
    tot = dict(checked=0, deferred=0, winners=0, proof_candidates=0)
    for first in (0, 125, 33_300, 33_425, 66_600, 66_725, 99_750, 99_875):
        rep = _check_sweep_against_oracle(wva, oracle, ctx, img, first, 125, c["r_max"], c["b_max"], 130_000, seed=50 + first)
        for k in tot:
            tot[k] += rep[k]
    assert tot["checked"] >= 1_000_000 and tot["winners"] > 300
    print("config 5 slice:", tot)


def test_config3_pairs_and_decisions_vs_oracle(wva, oracle, ctx):
    """every pair record, assignment and per-type total of config 3 against the oracle (all 8 000 pairs)"""
    img, _ = wva.synth.baseline_config(3)
    ctx.upload(img)
    got, gfe = ctx.analyze_pairs()
    want, wfe, _ = oracle.analyze_pairs(img, threads=_threads(oracle))
    assert np.array_equal(gfe, wfe)
    ok, field = got.equal_bits(want)
    assert ok, field
    acc, chosen = ctx.solve(unlimited=True)
    w_acc, w_chosen = oracle.solve(img, want, wfe, unlimited=True)
    assert np.array_equal(acc, w_acc) and chosen.equal_bits(w_chosen)[0]
    cnt, cst = ctx.allocate_by_type()
    w_cnt, w_cst = oracle.allocate_by_type(img, w_acc, w_chosen)
    assert np.array_equal(cnt, w_cnt) and cst.tobytes() == w_cst.tobytes()


def _fuzz_configs(wva, rng, n):
    cfg = np.zeros(n, dtype=wva.abi.QUEUE_CONFIG_DTYPE)
    b = np.exp(rng.uniform(0, np.log(512), n)).astype(np.int32).clip(1, 512)
    cfg["max_batch_size"] = b
    cfg["max_queue_size"] = b * 10
    cfg["alpha"] = rng.uniform(1, 30, n); cfg["beta"] = rng.uniform(0.01, 1, n)
    cfg["gamma"] = rng.uniform(0, 250, n); cfg["delta"] = np.exp(rng.uniform(np.log(1e-4), np.log(0.1), n))
    cfg["avg_input_tokens"] = rng.integers(0, 4097, n); cfg["avg_output_tokens"] = rng.integers(1, 1025, n)
    return cfg


def _max_rates(wva, cfg):
    """RateRange.Max of every config in float32, as BuildModel computes it (queueanalyzer.go:112-118)."""
    n = cfg["max_batch_size"].astype(F)
    inn, out = cfg["avg_input_tokens"], cfg["avg_output_tokens"]
    pre = np.where(inn == 0, F(0), (cfg["gamma"] + (cfg["delta"] * inn.astype(F)).astype(F) * n).astype(F)).astype(F)
    nd = np.where((inn == 0) & (out == 1), 1, out - 1).astype(F)
    dec = (nd * (cfg["alpha"] + (cfg["beta"] * n).astype(F)).astype(F)).astype(F)
    serv = (n / (pre + dec).astype(F)).astype(F)
    lam_max = (serv * (F(1) - F(0.001))).astype(F)
    return (lam_max * F(1000)).astype(F), serv


def test_queue_analyze_fuzz_1e7(wva, oracle, ctx):
    """1e7 random (alpha, beta, gamma, delta, in, out, b, lambda) through wva_queue_analyze (certified tails on)
    against the oracle, with the rate drawn so that r = lambda/s[N-1] covers (0, 0.999] and piles up at the
    certificate's precondition edges r ~ 0.9995 and M(1-r) ~ 0.3."""
    th = _threads(oracle)
    rng = np.random.default_rng(77)
    chunk = 2_000_000
    done = 0
    n_ok = 0
    for it in range(5):
        n = chunk
        cfg = _fuzz_configs(wva, rng, n)
        rmax, serv = _max_rates(wva, cfg)
        u = rng.uniform(0, 1, n)
        frac = np.where(u < 0.55, rng.uniform(0.0005, 1.0, n),
                np.where(u < 0.75, 1.0 - np.exp(rng.uniform(np.log(2e-4), np.log(2e-3), n)),       # r around 0.9995
                np.where(u < 0.95, 1.0 - 0.3 * np.exp(rng.uniform(-0.3, 0.3, n)) / (10.0 * cfg["max_batch_size"]),  # M(1-r) ~ 0.3
                         rng.uniform(0.999, 1.002, n))))
        rates = (rmax.astype(np.float64) * frac / 0.999).astype(F)
        want_m, want_s = oracle.queue_analyze(cfg, rates, threads=th)
        got_m, got_s = ctx.queue_analyze(cfg, rates)
        assert np.array_equal(got_s, want_s), it
        assert got_m.tobytes() == want_m.tobytes(), it
        n_ok += int((want_s == 0).sum())
        done += n
    assert done == 10_000_000 and n_ok > 5_500_000


def test_queue_analyze_large_K_edges(wva, oracle, ctx):
    """K at and around the certificate's 2^20 bound (b up to 100 000, queue 10 b) and tiny M."""
    th = _threads(oracle)
    rng = np.random.default_rng(78)
    n = 600
    cfg = _fuzz_configs(wva, rng, n)
    b = np.concatenate([rng.integers(90_000, 100_000, 200), np.full(100, 95_325), rng.integers(1, 4, 300)]).astype(np.int32)
    cfg["max_batch_size"] = b
    cfg["max_queue_size"] = np.where(b > 1000, 10 * b, rng.integers(0, 3, n))
    cfg["avg_output_tokens"] = rng.integers(1, 64, n)
    rmax, _ = _max_rates(wva, cfg)
    rates = (rmax.astype(np.float64) * rng.uniform(0.05, 1.0005, n)).astype(F)
    want_m, want_s = oracle.queue_analyze(cfg, rates, threads=th)
    got_m, got_s = ctx.queue_analyze(cfg, rates)
    assert np.array_equal(got_s, want_s)
    assert got_m.tobytes() == want_m.tobytes()


def test_untamed_generator_pairs_vs_oracle(wva, oracle, ctx):
    """SURVEY 8(d)'s generator as written: out_tokens from {1..1024}, no server-level bound on
    N = MaxBatchSize*AtTokens/K (allocation.go:85).  N reaches 10^4-10^5 here."""
    img = wva.synth.make_system(96, 4, seed=61, n_types=2, max_pair_batch=0, out_tokens_min=1)
    # one server at the generator's extreme: out_tokens 2, maxBatch 512 at 512 tokens -> N = 131 072, K = 1 441 792
    img.srv_out_tokens[5] = 2; img.srv_max_batch[5] = 0; img.srv_arrival_rpm[5] = 900.0; img.srv_slo_tps[5] = 0.0
    img.perf_max_batch[5 * img.A:6 * img.A] = 512; img.perf_at_tokens[5 * img.A:6 * img.A] = 512
    img.perf_valid[5 * img.A:6 * img.A] = 1; img.srv_target_valid[5] = 1
    pa = img.perf_max_batch.reshape(img.M, img.A).astype(np.int64) * img.perf_at_tokens.reshape(img.M, img.A)
    N = pa[img.srv_model] // np.maximum(img.srv_out_tokens.astype(np.int64), 1)[:, None]
    N = np.where(img.srv_max_batch[:, None] > 0, img.srv_max_batch[:, None], N)
    assert N.max() > 100_000 and (N.max(axis=1) > 10_000).sum() >= 3, N.max()
    ctx.upload(img)
    got, gfe = ctx.analyze_pairs()
    want, wfe, _ = oracle.analyze_pairs(img, threads=_threads(oracle))
    assert np.array_equal(gfe, wfe)
    ok, field = got.equal_bits(want)
    assert ok, field
    assert int(gfe.sum()) > 100
    # and the sweep of the same un-tamed servers (b <= 512 is a property of the grid, not of N)
    best, cube, status = ctx.analyze_grid(16, 256, want_cube=True)
    o_best, o_cube, o_status, _ = oracle.analyze_grid(img, 16, 256, want_cube=True, threads=_threads(oracle))
    assert np.array_equal(status, o_status) and cube.tobytes() == o_cube.tobytes() and best.tobytes() == o_best.tobytes()
