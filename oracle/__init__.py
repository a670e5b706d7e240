"""ctypes binding of the CPU oracle (oracle/libwva_oracle.so).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import wva_import

_wva = wva_import.load()
abi = _wva.abi

_DIR = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_DIR, "libwva_oracle.so")
_lib = None


def build(force=False):
    src = os.path.join(_DIR, "wva_oracle.cpp")
    hdr = os.path.join(_DIR, "..", "include", "wva_b200.h")
    if (not force and os.path.exists(_LIB_PATH)
            and os.path.getmtime(_LIB_PATH) >= max(os.path.getmtime(src), os.path.getmtime(hdr))):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _DIR, "-B", "libwva_oracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = C.CDLL(_LIB_PATH)
        L.wvao_analyzer_new.restype = C.c_void_p
        L.wvao_analyzer_new.argtypes = [C.POINTER(abi.QueueConfig)]
        L.wvao_analyzer_free.argtypes = [C.c_void_p]
        L.wvao_analyzer_analyze.argtypes = [C.c_void_p, C.c_float, C.POINTER(abi.Metrics)]
        L.wvao_analyzer_rate_range.argtypes = [C.c_void_p, abi.f32p, abi.f32p]
        L.wvao_analyzer_serv_rate.argtypes = [C.c_void_p, abi.f32p, C.c_int32]
        L.wvao_analyzer_solve.argtypes = [C.c_void_p, C.c_float, C.c_float, abi.f32p]
        L.wvao_analyzer_probabilities.restype = C.c_int64
        L.wvao_analyzer_probabilities.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_int64]
        L.wvao_analyzer_binary_search.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float,
                                                  abi.f32p, C.POINTER(C.c_int)]
        L.wvao_within_tolerance.argtypes = [C.c_float, C.c_float, C.c_float]
        L.wvao_transition_penalty.restype = C.c_float
        L.wvao_transition_penalty.argtypes = [C.c_int32, C.c_int64, C.c_float, C.c_int32, C.c_int64, C.c_float]
        L.wvao_queue_analyze.argtypes = [C.c_int32, C.c_void_p, abi.f32p, C.c_void_p, abi.u8p]
        L.wvao_queue_size.argtypes = [C.c_int32, C.c_void_p, abi.f32p, abi.f32p, C.c_void_p, abi.f32p, abi.u8p]
        L.wvao_queue_size_mt.argtypes = [C.c_int32, C.c_void_p, abi.f32p, abi.f32p, C.c_void_p, abi.f32p, abi.u8p, C.c_int]
        L.wvao_analyzer_eval.argtypes = [C.c_void_p, C.c_int, C.c_float, abi.f32p]
        L.wvao_rescale_counts.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.wvao_queue_analyze_mt.argtypes = [C.c_int32, C.c_void_p, abi.f32p, C.c_void_p, abi.u8p, C.c_int]
        L.wvao_grid_candidates.argtypes = [C.POINTER(abi.SystemSoa), C.c_int64, abi.i32p, abi.i32p, abi.i32p, abi.i32p,
                                           C.c_void_p, abi.u8p, C.c_int]
        L.wvao_analyze_pairs.argtypes = [C.POINTER(abi.SystemSoa), C.POINTER(abi.AllocSoa), abi.u8p, C.c_int,
                                         C.POINTER(C.c_uint64)]
        L.wvao_analyze_grid.argtypes = [C.POINTER(abi.SystemSoa), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]
        L.wvao_grid_row_values.argtypes = [C.POINTER(abi.SystemSoa), C.c_int32, C.c_int32, C.c_int32, abi.f32p]
        L.wvao_grid_rows_feasible.argtypes = [C.POINTER(abi.SystemSoa), C.c_int64, abi.i32p, abi.i32p, abi.i32p, abi.i32p,
                                              abi.i32p, abi.i32p, C.c_int]
        L.wvao_solve.argtypes = [C.POINTER(abi.SystemSoa), C.POINTER(abi.AllocSoa), abi.u8p,
                                 C.POINTER(abi.OptimizerSpec), abi.i32p, C.POINTER(abi.AllocSoa)]
        L.wvao_allocate_by_type.argtypes = [C.POINTER(abi.SystemSoa), C.c_int32, C.c_int32, abi.i32p,
                                            C.POINTER(abi.AllocSoa), abi.i64p, abi.f32p]
        L.wvao_model_new.restype = C.c_void_p
        L.wvao_model_new.argtypes = [C.c_int64, abi.f32p, C.c_int32]
        L.wvao_model_free.argtypes = [C.c_void_p]
        L.wvao_model_solve.argtypes = [C.c_void_p, C.c_float, C.c_float, abi.f32p]
        L.wvao_model_probabilities.restype = C.c_int64
        L.wvao_model_probabilities.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_int64]
        L.wvao_mm1k_solve.argtypes = [C.c_int64, C.c_float, C.c_float, abi.f32p, C.POINTER(C.c_double)]
        L.wvao_binary_search_testfunc.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, abi.f32p,
                                                  C.POINTER(C.c_int)]
        L.wvao_prefill_time.restype = C.c_float
        L.wvao_prefill_time.argtypes = [C.c_float, C.c_float, C.c_int32, C.c_float]
        L.wvao_decode_time.restype = C.c_float
        L.wvao_decode_time.argtypes = [C.c_float, C.c_float, C.c_float]
        L.wvao_effective_concurrency.restype = C.c_float
        L.wvao_effective_concurrency.argtypes = [C.c_float] * 5 + [C.c_int32] * 3
        _lib = L
    return _lib


def rescale_events():
    lib().wvao_rescale_events.restype = C.c_uint64
    return int(lib().wvao_rescale_events())


def rescale_counts():
    """(chain, sum): rescale branches taken since load by the chain (mm1modelstatedependent.go:84-89) and by the
    normalising sum (:95-104); rescale_events() is their total"""
    chain, total = C.c_uint64(), C.c_uint64()
    lib().wvao_rescale_counts(C.byref(chain), C.byref(total))
    return int(chain.value), int(total.value)


def hardware_threads():
    return int(lib().wvao_hardware_threads())


class Analyzer:
    """analyzer.QueueAnalyzer with persistent model state (reference pkg/analyzer/queueanalyzer.go:14-21)."""

    def __init__(self, max_batch, max_queue, alpha, beta, gamma, delta, in_tokens, out_tokens):
        self.cfg = abi.QueueConfig(max_batch, max_queue, alpha, beta, gamma, delta, in_tokens, out_tokens)
        self.h = lib().wvao_analyzer_new(C.byref(self.cfg))
        self.K = max_batch + max_queue

    @property
    def ok(self):
        return bool(self.h)

    def __del__(self):
        if getattr(self, "h", None):
            lib().wvao_analyzer_free(self.h)
            self.h = None

    def analyze(self, rate):
        m = abi.Metrics()
        st = lib().wvao_analyzer_analyze(self.h, C.c_float(rate), C.byref(m))
        return st, m

    def rate_range(self):
        lo, hi = C.c_float(), C.c_float()
        lib().wvao_analyzer_rate_range(self.h, C.byref(lo), C.byref(hi))
        return np.float32(lo.value), np.float32(hi.value)

    def serv_rate(self):
        out = np.zeros(self.cfg.max_batch_size, dtype=np.float32)
        lib().wvao_analyzer_serv_rate(self.h, abi.ptr(out, C.c_float), len(out))
        return out

    def solve(self, lam, mu=1.0):
        out = np.zeros(9, dtype=np.float32)
        lib().wvao_analyzer_solve(self.h, C.c_float(lam), C.c_float(mu), abi.ptr(out, C.c_float))
        keys = ["valid", "rho", "resp", "wait", "serv", "in_system", "queue_len", "in_servers", "throughput"]
        return dict(zip(keys, out))

    def probabilities(self):
        out = np.zeros(self.K + 1, dtype=np.float64)
        lib().wvao_analyzer_probabilities(self.h, out.ctypes.data_as(C.POINTER(C.c_double)), len(out))
        return out

    def eval(self, kind, x):
        """EvalTTFT (kind 0) / EvalITL (kind 1) at lambda = x -> float32 y, or None where the model is invalid"""
        y = C.c_float()
        err = lib().wvao_analyzer_eval(self.h, kind, C.c_float(x), C.byref(y))
        return None if err else np.float32(y.value)

    def binary_search(self, kind, x_min, x_max, y_target):
        x, ind = C.c_float(), C.c_int()
        err = lib().wvao_analyzer_binary_search(self.h, kind, C.c_float(x_min), C.c_float(x_max),
                                                C.c_float(y_target), C.byref(x), C.byref(ind))
        return np.float32(x.value), ind.value, err


_SOLVE_KEYS = ["valid", "rho", "resp", "wait", "serv", "in_system", "queue_len", "in_servers", "throughput"]


class Model:
    """analyzer.MM1ModelStateDependent (reference pkg/analyzer/mm1modelstatedependent.go:8-26)."""

    def __init__(self, K, serv_rate):
        sr = np.ascontiguousarray(serv_rate, dtype=np.float32)
        self.K = int(K)
        self.h = lib().wvao_model_new(self.K, abi.ptr(sr, C.c_float), len(sr))

    def __del__(self):
        if getattr(self, "h", None):
            lib().wvao_model_free(self.h)
            self.h = None

    def solve(self, lam, mu=1.0):
        out = np.zeros(9, dtype=np.float32)
        lib().wvao_model_solve(self.h, C.c_float(lam), C.c_float(mu), abi.ptr(out, C.c_float))
        return dict(zip(_SOLVE_KEYS, out))

    def probabilities(self):
        out = np.zeros(self.K + 1, dtype=np.float64)
        lib().wvao_model_probabilities(self.h, out.ctypes.data_as(C.POINTER(C.c_double)), len(out))
        return out


def mm1k_solve(K, lam, mu):
    """analyzer.MM1KModel(K).Solve(lam, mu) (reference pkg/analyzer/mm1kmodel.go)."""
    out = np.zeros(8, dtype=np.float32)
    p = np.zeros(K + 1, dtype=np.float64)
    lib().wvao_mm1k_solve(K, C.c_float(lam), C.c_float(mu), abi.ptr(out, C.c_float), p.ctypes.data_as(C.POINTER(C.c_double)))
    keys = ["valid", "rho", "resp", "wait", "serv", "in_system", "queue_len", "throughput"]
    return dict(zip(keys, out)), p


def binary_search_testfunc(func, x_min, x_max, y_target):
    x, ind = C.c_float(), C.c_int()
    err = lib().wvao_binary_search_testfunc(func, C.c_float(x_min), C.c_float(x_max), C.c_float(y_target),
                                            C.byref(x), C.byref(ind))
    return np.float32(x.value), ind.value, err


def within_tolerance(x, v, tol):
    return bool(lib().wvao_within_tolerance(C.c_float(x), C.c_float(v), C.c_float(tol)))


def transition_penalty(a_acc, a_rep, a_cost, b_acc, b_rep, b_cost):
    return np.float32(lib().wvao_transition_penalty(a_acc, a_rep, C.c_float(a_cost), b_acc, b_rep, C.c_float(b_cost)))


def prefill_time(gamma, delta, in_tok, batch):
    return np.float32(lib().wvao_prefill_time(C.c_float(gamma), C.c_float(delta), in_tok, C.c_float(batch)))


def decode_time(alpha, beta, batch):
    return np.float32(lib().wvao_decode_time(C.c_float(alpha), C.c_float(beta), C.c_float(batch)))


def effective_concurrency(serv_time, alpha, beta, gamma, delta, in_tok, out_tok, max_batch):
    return np.float32(lib().wvao_effective_concurrency(C.c_float(serv_time), C.c_float(alpha), C.c_float(beta),
                                                       C.c_float(gamma), C.c_float(delta), in_tok, out_tok, max_batch))


def queue_analyze(cfgs, rates, threads=1):
    cfgs = np.ascontiguousarray(cfgs, dtype=abi.QUEUE_CONFIG_DTYPE)
    rates = np.ascontiguousarray(rates, dtype=np.float32)
    n = len(cfgs)
    metrics = np.zeros(n, dtype=abi.METRICS_DTYPE)
    status = np.zeros(n, dtype=np.uint8)
    lib().wvao_queue_analyze_mt(n, cfgs.ctypes.data, abi.ptr(rates, C.c_float), metrics.ctypes.data,
                                abi.ptr(status, C.c_uint8), int(threads))
    return metrics, status


def grid_candidates(img, s, a, r, b, threads=1):
    """The sweep's candidates (s, a, r, b) one by one through the reference API -> (metrics, status)."""
    sysc = img.c_struct()
    arr = [np.ascontiguousarray(x, dtype=np.int32) for x in (s, a, r, b)]
    n = len(arr[0])
    metrics = np.zeros(n, dtype=abi.METRICS_DTYPE)
    status = np.zeros(n, dtype=np.uint8)
    lib().wvao_grid_candidates(C.byref(sysc), n, *[abi.ptr(x, C.c_int32) for x in arr], metrics.ctypes.data,
                               abi.ptr(status, C.c_uint8), int(threads))
    return metrics, status


def queue_size(cfgs, targets, threads=1):
    cfgs = np.ascontiguousarray(cfgs, dtype=abi.QUEUE_CONFIG_DTYPE)
    targets = np.ascontiguousarray(targets, dtype=np.float32).reshape(-1)
    n = len(cfgs)
    rates = np.zeros(3 * n, dtype=np.float32)
    achieved = np.zeros(3 * n, dtype=np.float32)
    metrics = np.zeros(n, dtype=abi.METRICS_DTYPE)
    status = np.zeros(n, dtype=np.uint8)
    lib().wvao_queue_size_mt(n, cfgs.ctypes.data, abi.ptr(targets, C.c_float), abi.ptr(rates, C.c_float),
                             metrics.ctypes.data, abi.ptr(achieved, C.c_float), abi.ptr(status, C.c_uint8), int(threads))
    return rates.reshape(n, 3), metrics, achieved.reshape(n, 3), status


def analyze_pairs(img, threads=1):
    """Server.Calculate for all servers -> (AllocArrays[S*A], feasible[S*A], chain_steps)."""
    sysc = img.c_struct()
    out = abi.AllocArrays(img.S * img.A)
    feasible = np.zeros(img.S * img.A, dtype=np.uint8)
    steps = C.c_uint64(0)
    lib().wvao_analyze_pairs(C.byref(sysc), C.byref(out.c), abi.ptr(feasible, C.c_uint8), threads, C.byref(steps))
    return out, feasible, steps.value


def analyze_grid(img, r_max, b_max, s0=0, s1=None, want_cube=True, threads=1):
    s1 = img.S if s1 is None else s1
    ns = s1 - s0
    sysc = img.c_struct()
    best = np.zeros(ns, dtype=abi.GRID_BEST_DTYPE)
    ncand = ns * img.A * r_max * b_max
    cube = np.zeros(ncand, dtype=abi.METRICS_DTYPE) if want_cube else None
    status = np.zeros(ncand, dtype=np.uint8) if want_cube else None
    steps = C.c_uint64(0)
    lib().wvao_analyze_grid(C.byref(sysc), s0, s1, r_max, b_max, best.ctypes.data,
                            cube.ctypes.data if want_cube else None,
                            status.ctypes.data if want_cube else None, threads, C.byref(steps))
    return best, cube, status, steps.value


def grid_row_values(img, r_max, s0=0, s1=None):
    """value of every sweep row (s, a, r) -> float32 [ns, A, r_max] (NaN where the pair is unusable)."""
    s1 = img.S if s1 is None else s1
    sysc = img.c_struct()
    out = np.zeros((s1 - s0) * img.A * r_max, dtype=np.float32)
    lib().wvao_grid_row_values(C.byref(sysc), s0, s1, r_max, abi.ptr(out, C.c_float))
    return out.reshape(s1 - s0, img.A, r_max)


def grid_rows_feasible(img, s, a, r, b_lo, b_hi, threads=1):
    """feasible-candidate count of each listed row over b in [b_lo, b_hi] (reference API per candidate)."""
    sysc = img.c_struct()
    arr = [np.ascontiguousarray(x, dtype=np.int32) for x in (s, a, r, b_lo, b_hi)]
    n = len(arr[0])
    out = np.zeros(n, dtype=np.int32)
    lib().wvao_grid_rows_feasible(C.byref(sysc), n, *[abi.ptr(x, C.c_int32) for x in arr], abi.ptr(out, C.c_int32), int(threads))
    return out


def solve(img, pairs, feasible, unlimited=True, delayed_best_effort=False, policy=abi.POLICY_NONE):
    sysc = img.c_struct()
    spec = abi.OptimizerSpec(1 if unlimited else 0, 1 if delayed_best_effort else 0, int(policy))
    chosen_acc = np.zeros(img.S, dtype=np.int32)
    chosen = abi.AllocArrays(img.S)
    lib().wvao_solve(C.byref(sysc), C.byref(pairs.c), abi.ptr(feasible, C.c_uint8), C.byref(spec),
                     abi.ptr(chosen_acc, C.c_int32), C.byref(chosen.c))
    return chosen_acc, chosen


def allocate_by_type(img, chosen_acc, chosen, s0=0, s1=None):
    s1 = img.S if s1 is None else s1
    sysc = img.c_struct()
    count = np.zeros(img.T, dtype=np.int64)
    cost = np.zeros(img.T, dtype=np.float32)
    lib().wvao_allocate_by_type(C.byref(sysc), s0, s1, abi.ptr(chosen_acc, C.c_int32), C.byref(chosen.c),
                                abi.ptr(count, C.c_int64), abi.ptr(cost, C.c_float))
    return count, cost
