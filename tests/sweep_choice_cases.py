"""Images of the sweep-choice tests (test_sweep_choice_cpu / test_sweep_choice_gpu): each server's winner above 64
replicas, and on candidate values synth.make_system never produces.

The sweep picks each server's winner by one 64-bit key (value, a, r, b), make_key in csrc/wva_kernels.cuh: the
order-preserving bits of the float32 value, 8 bits of accelerator, 10 bits of r - 1 and 14 of b - 1.  The value,
TransitionPenalty of the candidate's cost, is computed in scan_row_ctx, candidate_key, k_grid_rows and k_grid_wrow, each
with its own NaN guard and its own -0 -> +0 canonicalisation.  The images:

  R1   12 servers x 3 accelerators, r_max = 1024, b_max = 64: the scan kernels split each pair's rows over 16 blocks of
       64; min_replicas in {-1, 0, 1, 64, 65, 129, r_max, r_max + 1}, a negative-cost server (winner at r_max), a server
       whose lambda drops below 2^-100 from r = 101 on (winner at 129), one whose rate rounds to 0 from r = 200 on, and a
       loaded one whose first feasible r lies inside a middle chunk
  R2   600 x 1, r_max = 100, b_max = 48: a large shard, blocks of 56 + 44 rows; min_replicas on both sides of 56 | 57,
       three servers whose every row has lambda < 2^-100 (more than 4 096 deferred exact chains) and one whose rates
       are all +Inf (every candidate on the literal list)
  R3   1 x 1, r_max = 1024, b_max = 512: 128 blocks of 8 rows; the winner at the last block's first row
  R4a  1 x 1, r_max = 65: a last block of one row, the winner in it
  R4b  600 x 1, r_max = 65: blocks of 40 + 25 rows, winners on both sides of 40 | 41 and at r_max
  V    39 servers x 11 accelerators, r_max = 200, b_max = 64: one value fixture per server (VALUE_FIXTURES), accelerator
       costs +0, -0, 25, 25 (an identical pair), -12.5, the smallest subnormal, 3e38, the largest float32, +Inf, NaN and
       -Inf; a server's profile is valid on its fixture's accelerators only

Chunk counts are for the 132 SMs of an H100 SXM; row_plan restates the host's plan for any SM count.
"""
import numpy as np

F = np.float32
MAX_F32 = np.finfo(F).max
TINY_F32 = F(np.float32(1.4e-45))                     # 2^-149, the smallest subnormal
NEG_NAN = np.array([0xffc00000], dtype=np.uint32).view(F)[0]
H100_SMS = 132
_NONE, _UNK = -1, -2                                 # abi.ACC_NONE, abi.ACC_UNKNOWN

# set_certified_tails modes: 1 default (scan kernels), 33 scan kernels tuned for 3 blocks per SM, 0 no certificate,
# 3 one thread per candidate, 5 one thread per row, 9 one warp per row, 17 the automatic round-1 choice
MODES = (1, 33, 0, 3, 5, 9, 17)
SCAN_WARPS, SCAN_MAXROWS, GRID_THREADS, WX_CP = 8, 64, 256, 256


def _cdiv(a, b):
    return -(-a // b)


def row_plan(mode, pairs, r_max, b_max, num_sms):
    """(kernel, rows of each block of a pair) that grid_run (csrc/wva_b200.cu) launches for a one-slice shard of `pairs`
    (server, accelerator) pairs in set_certified_tails mode `mode`.  kernel is 'scan' (k_scan_prep / k_scan_cert /
    k_scan_lean), 'grid' (k_grid), 'rows' (k_grid_rows: one thread per row, a pair's rows in one block) or 'wrow'
    (k_grid_wrow)."""
    certified = bool(mode & 1)
    grid_rows = 0 if mode & 2 else (2 if mode & 4 else (3 if mode & 8 else 1))
    scan = certified and not (mode & (2 | 4 | 8 | 16))
    n = 1
    fill = 16 * num_sms
    if 0 < pairs < fill:
        n = min(_cdiv(fill, pairs), r_max)
    r_chunk = _cdiv(r_max, n)
    rows = not scan and certified and grid_rows not in (0, 3) and (grid_rows == 2 or pairs * r_max >= 32768)
    wrow = (not scan and certified and not rows and grid_rows == 3 and
            b_max * 20 + 16 + (GRID_THREADS // 32) * (WX_CP + 1 + 1024) * 8 <= 200 * 1024)
    if wrow:
        r_chunk = GRID_THREADS // 32
    if scan:
        chunks = 1
        if 0 < pairs < 4 * num_sms:
            chunks = _cdiv(4 * num_sms, pairs)
        chunks = max(min(chunks, _cdiv(r_max, SCAN_WARPS)), _cdiv(r_max, SCAN_MAXROWS))
        r_chunk = _cdiv(_cdiv(r_max, chunks), SCAN_WARPS) * SCAN_WARPS
    if rows:
        return "rows", [r_max]
    kernel = "scan" if scan else ("wrow" if wrow else "grid")
    return kernel, [min(r_chunk, r_max - r0) for r0 in range(0, r_max, r_chunk)]


def chunk_starts(shape):
    """first replica count of each block"""
    return list(np.cumsum([0] + shape[:-1]) + 1)


# ---- images -----------------------------------------------------------------------------------------------------------

def _base(wva, S, A, seed, n_types=None):
    """make_system with every pair usable, no TPS target, no current allocation, keepAccelerator off"""
    img = wva.synth.make_system(S, A, seed=seed, n_types=n_types, zero_load_fraction=0.0, keep_fraction=0.0,
                                tps_fraction=0.0, edge_fraction=0.0)
    rng = np.random.default_rng(seed + 1000)
    img.perf_valid[:] = 1
    img.srv_target_valid[:] = 1
    img.srv_slo_tps[:] = 0.0
    img.srv_max_batch[:] = rng.integers(8, 65, S)          # pair sizing's N (the sweep ignores it)
    return img, rng


def _light(img, servers):
    """loose SLOs, short requests and 6 requests per minute: b = 1 is feasible at every r"""
    img.srv_slo_itl[servers] = 200.0
    img.srv_slo_ttft[servers] = 2000.0
    img.srv_in_tokens[servers] = 128
    img.srv_out_tokens[servers] = 32
    img.srv_arrival_rpm[servers] = 6.0


def _no_current(img, servers):
    img.srv_cur_acc[servers] = _NONE
    img.srv_cur_replicas[servers] = 0
    img.srv_cur_cost[servers] = 0.0


def lambda_row(arrival, r):
    """float32 lambda of sweep row r: (arrival / 60) / r / 1000"""
    return F(F(F(arrival) / F(60)) / F(r)) / F(1000)


def rate_row(arrival, r):
    return F(F(arrival) / F(60)) / F(r)


R1_TINY_LAMBDA = F(2.0 ** -100 * 60000.0 * 100)       # lambda < 2^-100 from r = 101 on
R1_ZERO_RATE = F(2.0 ** -149 * 60 * 100)              # rate / r rounds to 0 from r = 200 on
R1_MIN_REP = [-1, 0, 1, 64, 65, 129, 1024, 1025]


def _r1(wva):
    from test_profile_edges_gpu import rate_max, rate_table
    S, A = 12, 3
    img, rng = _base(wva, S, A, 1101)
    _light(img, np.arange(S))
    _no_current(img, np.arange(S))
    img.perf_acc_count[:] = 1
    img.acc_cost[2] = -40.0                          # the negative accelerator: usable by server 8 only
    for s in range(S):
        img.perf_valid[int(img.srv_model[s]) * A + 2] = 1 if s == 8 else 0
    img.perf_valid[int(img.srv_model[8]) * A:int(img.srv_model[8]) * A + 2] = 0
    img.srv_min_replicas[:8] = R1_MIN_REP
    img.srv_min_replicas[8:] = [0, 129, 65, 0]
    img.srv_arrival_rpm[9] = R1_TINY_LAMBDA
    img.srv_arrival_rpm[10] = R1_ZERO_RATE
    # server 11: about 300 replicas at b = 64 before RateRange.Max admits the rate
    cap = min(float(rate_max(rate_table(img, 11, a, 64))[63]) for a in range(2))
    img.srv_arrival_rpm[11] = F(cap * 60.0 * 300)
    return img, 1024, 64


def _r2(wva):
    S = 600
    img, rng = _base(wva, S, 1, 1102)
    img.srv_min_replicas[:] = np.resize([-1, 0, 1, 56, 57, 64, 65, 100, 101], S)
    img.srv_arrival_rpm[[5, 300, 599]] = F(2.0 ** -101 * 60000.0)          # lambda < 2^-100 on every row
    img.srv_min_replicas[[5, 300, 599]] = 0
    # server 7: a zero profile (every rate +Inf, nGood = 0): all its candidates go to the literal list
    m = int(img.srv_model[7])
    img.perf_alpha[m] = img.perf_beta[m] = img.perf_gamma[m] = img.perf_delta[m] = 0.0
    img.srv_in_tokens[7] = 0
    return img, 100, 48


def _r3(wva):
    img, _ = _base(wva, 1, 1, 1103)
    _light(img, [0])
    _no_current(img, [0])
    img.srv_min_replicas[0] = 1017
    return img, 1024, 512


def _r4a(wva):
    img, _ = _base(wva, 1, 1, 1104)
    _light(img, [0])
    _no_current(img, [0])
    img.srv_min_replicas[0] = 65
    return img, 65, 64


def _r4b(wva):
    S = 600
    img, _ = _base(wva, S, 1, 1105)
    img.srv_min_replicas[:] = np.resize([-1, 0, 1, 40, 41, 64, 65, 66], S)
    return img, 65, 64


# V: accelerator costs (and the identical pair 2, 3)
V_COSTS = [F(0.0), F(-0.0), F(25.0), F(25.0), F(-12.5), TINY_F32, F(3e38), MAX_F32, F(np.inf), F(np.nan), F(-np.inf)]
V_R, V_B = 200, 64

# name: (usable accelerators, current accelerator, current replicas, current cost, min_replicas, keepAccelerator,
#        the (accelerator, r) the oracle picks or None)
VALUE_FIXTURES = [
    ("negzero_tie", (0, 1), 1, 100, 0.0, 0, 0, (0, 1)),            # -0 on a1 ties with +0 on a0: a0
    ("negzero_tie_hi", (0, 1), 1, 150, 0.0, 1, 0, (0, 1)),
    ("negzero_cur", (1,), 1, 150, 0.0, 150, 0, (1, 150)),          # r > 150 are -0: canonical, the zero row first
    ("negzero_cur_lo", (1,), 1, 70, 0.0, 70, 0, (1, 70)),
    ("neginf", (2, 3), 2, 120, np.inf, 120, 0, (2, 121)),          # cost - Inf = -Inf beside r = cur_rep; a3 NaN
    ("neginf_lo", (2,), 2, 1, np.inf, 0, 0, (2, 2)),
    ("nan_cur", (2, 4), 2, 150, np.nan, 0, 0, (2, 150)),           # NaN everywhere but the zero row
    ("nan_cur_blocked", (2,), 2, 150, np.nan, 151, 0, None),
    ("nan_cur_zero_rep", (2, 3), 3, 0, np.nan, 0, 0, None),
    ("nan_cur_above", (2,), 2, 250, np.nan, 0, 0, None),           # cur_rep above r_max
    ("nan_acc", (9,), _NONE, 0, 0.0, 0, 0, None),
    ("nan_acc_cur", (9,), 9, 130, 5.0, 0, 0, (9, 130)),            # the zero row needs no cost
    ("inf_acc", (8,), _NONE, 0, 0.0, 0, 0, (8, 1)),
    ("inf_minus_inf", (8,), 8, 140, np.inf, 0, 0, (8, 140)),       # Inf - Inf = NaN beside the zero row
    ("huge", (6, 7), _NONE, 0, 0.0, 0, 0, (6, 1)),                 # 3.3e38 finite; MaxFloat32's value overflows
    ("huge_min2", (6, 7), _NONE, 0, 0.0, 2, 0, (6, 2)),            # every cost overflows: +Inf ties
    ("max_cur", (7,), 7, 90, 0.0, 0, 0, (7, 90)),
    ("neg", (4,), _NONE, 0, 0.0, 0, 0, (4, V_R)),                  # negative: the largest feasible r
    ("neg_cur", (4,), 4, V_R, -1000.0, 0, 0, (4, V_R - 1)),
    ("neg_vs_zero", (0, 4), _NONE, 0, 0.0, 0, 0, (4, V_R)),
    ("neg_min_above", (4,), _NONE, 0, 0.0, V_R + 1, 0, None),
    ("subnormal", (5,), _NONE, 0, 0.0, 0, 0, (5, 1)),
    ("subnormal_vs_zero", (0, 5), _NONE, 0, 0.0, 0, 0, (0, 1)),
    ("identical", (2, 3), _NONE, 0, 0.0, 0, 0, (2, 1)),
    ("identical_min129", (2, 3), _NONE, 0, 0.0, 129, 0, (2, 129)),
    ("identical_cur_hi", (2, 3), 3, 100, 2500.0, 0, 0, (3, 1)),
    ("acc_count_le0", (2, 3), _NONE, 0, 0.0, 0, 0, (2, 1)),        # perf_acc_count 0 and -3 both count as 1
    ("acc_count_mix", (2, 3), _NONE, 0, 0.0, 0, 0, (3, 1)),        # 2 against 0
    ("keep_unknown", (0, 2), _UNK, 100, 0.0, 0, 1, None),          # keepAccelerator, unknown current: no candidate
    ("unknown_nokeep", (2,), _UNK, 100, 0.0, 0, 0, (2, 1)),
    ("keep_cur", (0, 2, 4), 4, 10, 0.0, 0, 1, (4, V_R)),
    ("keep_none", (0, 2), _NONE, 0, 0.0, 0, 1, (0, 1)),
    ("negzero_tie_min65", (0, 1), 1, 150, 0.0, 65, 0, (0, 65)),
    ("neginf_hi", (2,), 2, 64, np.inf, 64, 0, (2, 65)),
    ("nan_cur_lo", (2,), 2, 64, np.nan, 0, 0, (2, 64)),
    ("inf_acc_min65", (8,), _NONE, 0, 0.0, 65, 0, (8, 65)),
    ("negnan_cur", (2,), 2, 150, NEG_NAN, 0, 0, (2, 150)),
    ("nan_acc_cur1", (9,), 9, 1, 5.0, 0, 0, (9, 1)),               # a NaN cost the solver keeps: a NaN type total
    ("neginf_acc", (10,), _NONE, 0, 0.0, 0, 0, (10, 1)),           # -Inf ties on every row: a -Inf type total
]
FIXTURE = {f[0]: i for i, f in enumerate(VALUE_FIXTURES)}


def _v(wva):
    S, A = len(VALUE_FIXTURES), len(V_COSTS)
    img, _ = _base(wva, S, A, 1106, n_types=4)
    _light(img, np.arange(S))
    img.acc_cost[:] = V_COSTS
    img.acc_type[:] = [0, 0, 1, 1, 2, 2, 3, 3, 0, 3, 1]
    img.acc_multiplicity[3] = img.acc_multiplicity[2]
    img.perf_acc_count[:] = 1
    for s, (name, accs, cur, rep, cost, mn, keep, _) in enumerate(VALUE_FIXTURES):
        m = int(img.srv_model[s]) * A
        img.perf_valid[m:m + A] = 0
        img.perf_valid[[m + a for a in accs]] = 1
        for arr in (img.perf_alpha, img.perf_beta, img.perf_gamma, img.perf_delta, img.perf_max_batch,
                    img.perf_at_tokens):
            arr[m + 3] = arr[m + 2]                                 # identical accelerators, identical profiles
        img.srv_cur_acc[s], img.srv_cur_replicas[s], img.srv_cur_cost[s] = cur, rep, F(cost)
        img.srv_min_replicas[s], img.srv_keep_acc[s] = mn, keep
    s = FIXTURE["negnan_cur"]
    img.srv_cur_cost[s:s + 1].view(np.uint32)[:] = 0xffc00000
    m = int(img.srv_model[FIXTURE["acc_count_le0"]]) * A
    img.perf_acc_count[m + 2], img.perf_acc_count[m + 3] = 0, -3
    m = int(img.srv_model[FIXTURE["acc_count_mix"]]) * A
    img.perf_acc_count[m + 2], img.perf_acc_count[m + 3] = 2, 0
    return img, V_R, V_B


_BUILDERS = dict(R1=_r1, R2=_r2, R3=_r3, R4a=_r4a, R4b=_r4b, V=_v)
IMAGES = list(_BUILDERS)
_CACHE = {}


def image(wva, name):
    """(image, r_max, b_max), built once per session from fixed seeds"""
    if name not in _CACHE:
        _CACHE[name] = _BUILDERS[name](wva)
    return _CACHE[name]


_ORACLE = {}


def oracle_sweep(oracle, wva, name):
    """the oracle's whole sweep of an image: (best, cube, status)"""
    if name not in _ORACLE:
        img, R, B = image(wva, name)
        _ORACLE[name] = oracle.analyze_grid(img, R, B, want_cube=True, threads=max(1, oracle.hardware_threads()))[:3]
    return _ORACLE[name]


# ---- the key order, restated ------------------------------------------------------------------------------------------

def restated_best(img, R, B, values, cube, status):
    """each server's winner by (value, a, r, b) over the feasible candidates whose canonical value is not NaN, with the
    record the sweep writes for it: cost = acc_cost * float32(numInstances * r), itl, ttft = wait + prefill and rho from
    the cube.  values: oracle.grid_row_values [S, A, R]."""
    from wva_import import load
    abi = load().abi
    S, A = img.S, img.A
    out = np.zeros(S, dtype=abi.GRID_BEST_DTYPE)
    out["acc"] = -1
    feas = ((status & 1) == 1).reshape(S, A, R, B)
    cube = cube.reshape(S, A, R, B)
    for s in range(S):
        ok = feas[s] & ~np.isnan(values[s])[:, :, None]
        a, r, b = np.nonzero(ok)
        if len(a) == 0:
            continue
        v = values[s][a, r]
        j = np.lexsort((b, r, a, v))[0]
        a, r, b = int(a[j]), int(r[j]), int(b[j])
        m = cube[s, a, r, b]
        n = int(img.perf_acc_count[int(img.srv_model[s]) * A + a])
        with np.errstate(over="ignore"):
            out[s] = (a, r + 1, b + 1, F(img.acc_cost[a]) * F(max(n, 1) * (r + 1)), values[s][a, r],
                          m["avg_token_time"], F(m["avg_wait_time"]) + F(m["avg_prefill_time"]), m["rho"])
    return out
