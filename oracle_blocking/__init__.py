"""ctypes binding of the oracle's blocking-probability sibling (oracle_blocking/libwva_oracle_blocking.so).

TEST INFRASTRUCTURE ONLY, like the oracle it extends: the product package never imports this module.
grid_candidates_blocking is oracle.grid_candidates plus p_block, the float32 of the oracle's own normalised p[K].
"""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle

abi = oracle.abi

_DIR = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_DIR, "libwva_oracle_blocking.so")
_lib = None


def build(force=False):
    """Build the library (force: even when it is newer than its sources).  The oracle's library it links against is
    only built when missing or out of date: __graft_entry__.build() forces that one itself."""
    src = os.path.join(_DIR, "wva_oracle_blocking.cpp")
    deps = [src, os.path.join(_DIR, "..", "include", "wva_b200.h"), oracle.build()]
    if (not force and os.path.exists(_LIB_PATH)
            and os.path.getmtime(_LIB_PATH) >= max(os.path.getmtime(d) for d in deps)):
        return _LIB_PATH
    subprocess.check_call(["make", "-C", _DIR, "-B", "libwva_oracle_blocking.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        oracle.lib()
        L = C.CDLL(_LIB_PATH)
        L.wvao_grid_candidates_blocking.argtypes = [C.POINTER(abi.SystemSoa), C.c_int64, abi.i32p, abi.i32p, abi.i32p,
                                                    abi.i32p, C.c_void_p, abi.u8p, abi.f32p, C.c_int]
        _lib = L
    return _lib


def grid_candidates_blocking(img, s, a, r, b, threads=1):
    """The sweep's candidates (s, a, r, b) one by one through the reference API -> (metrics, status, p_block)."""
    sysc = img.c_struct()
    arr = [np.ascontiguousarray(x, dtype=np.int32) for x in (s, a, r, b)]
    n = len(arr[0])
    metrics = np.zeros(n, dtype=abi.METRICS_DTYPE)
    status = np.zeros(n, dtype=np.uint8)
    p_block = np.zeros(n, dtype=np.float32)
    rc = lib().wvao_grid_candidates_blocking(C.byref(sysc), n, *[abi.ptr(x, C.c_int32) for x in arr], metrics.ctypes.data,
                                             abi.ptr(status, C.c_uint8), abi.ptr(p_block, C.c_float), int(threads))
    if rc != abi.OK:
        raise RuntimeError("the oracle's analyzer rejected a candidate its sweep accepted")
    return metrics, status, p_block


def grid_plane_blocking(img, r_max, b_max, s0=0, s1=None, threads=1):
    """Every candidate of servers [s0, s1) in cube order -> (metrics, status, p_block), each [ns*A*r_max*b_max]."""
    s1 = img.S if s1 is None else s1
    n = (s1 - s0) * img.A * r_max * b_max
    idx = np.arange(n, dtype=np.int64)
    b = idx % b_max + 1
    r = (idx // b_max) % r_max + 1
    pair = idx // (b_max * r_max)
    return grid_candidates_blocking(img, s0 + pair // img.A, pair % img.A, r, b, threads=threads)
