"""ctypes binding of libwva_b200.so (the C-ABI of include/wva_b200.h).

The library holds sm_90a kernels only.  There is no CPU implementation behind this module:
loading fails loudly when the shared object has not been built, and every compute call fails
with WvaError(ECUDA) when no H100 is present.
"""
import ctypes as C
import os

import numpy as np

from . import abi
from .image import SystemImage

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "libwva_b200.so")
_lib = None

# every symbol include/wva_b200.h declares (tests/test_abi_symbols.py checks the header against this)
EXPORTS = [
    "wva_abi_version", "wva_ctx_create", "wva_ctx_destroy", "wva_last_error", "wva_system_upload", "wva_set_shard",
    "wva_analyze_pairs", "wva_pairs_device", "wva_pairs_commit", "wva_pair_steps", "wva_pair_counters", "wva_pair_debug", "wva_analyze_grid",
    "wva_analyze_grid_device", "wva_grid_fetch", "wva_grid_cube_device", "wva_solve", "wva_solution_fetch", "wva_allocate_by_type", "wva_type_totals_device",
    "wva_solution_time_usec", "wva_queue_analyze", "wva_queue_size", "wva_launch_count", "wva_phase_time_usec",
    "wva_grid_counters", "wva_selftest_division", "wva_stream", "wva_grid_set_tail_cap", "wva_grid_list_sizes", "wva_grid_set_fused", "wva_grid_last_fused", "wva_pairs_set_warp_max", "wva_pairs_set_pstore", "wva_solve_set_ranked", "wva_solve_greedy_path", "wva_solve_stats", "wva_type_totals_merge", "wva_set_certified_tails", "wva_analyze", "wva_pairs_fetch", "wva_grid_deferred_fetch",
    "wva_system_upload_arrays", "wva_analyze_pairs_arrays", "wva_pairs_fetch_arrays", "wva_solve_arrays",
    "wva_system_update_servers", "wva_system_update_models", "wva_system_remove_server", "wva_system_set_capacity", "wva_upload_bytes", "wva_system_dims",
    "wva_model_solve",
    "wva_comm_unique_id", "wva_comm_init", "wva_comm_destroy", "wva_comm_info", "wva_comm_shard",
    "wva_group_create", "wva_group_destroy", "wva_group_size", "wva_group_ctx", "wva_group_last_error", "wva_group_upload",
    "wva_group_analyze", "wva_group_pairs_fetch", "wva_group_grid_fetch", "wva_group_solve", "wva_group_allocate_by_type",
    "wva_grid_blocking", "wva_grid_blocking_size", "wva_grid_blocking_device", "wva_grid_best_blocking", "wva_grid_blocking_counts", "wva_grid_blocking_exact_fetch",
    "wva_group_grid_best_blocking",
    "wva_analyze_pairs_batches", "wva_pairs_batches_counters", "wva_group_analyze_pairs_batches", "wva_shard_info",
    "wva_analyze_pairs_loads", "wva_pairs_loads_counters", "wva_group_analyze_pairs_loads",
]


class WvaError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("wva_b200 error %d: %s" % (code, msg))
        self.code = code


def lib():
    """Load libwva_b200.so (built by __graft_entry__.build()).  No fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("CUDA library %s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU implementation to fall back to)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
        L.wva_abi_version.restype = C.c_int
        L.wva_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
        L.wva_ctx_destroy.argtypes = [vp]
        L.wva_ctx_destroy.restype = None
        L.wva_last_error.argtypes = [vp]
        L.wva_last_error.restype = C.c_char_p
        L.wva_system_upload.argtypes = [vp, C.POINTER(abi.SystemSoa)]
        L.wva_set_shard.argtypes = [vp, i32, i32]
        L.wva_analyze_pairs.argtypes = [vp, C.POINTER(abi.AllocSoa), abi.u8p]
        L.wva_pairs_device.argtypes = [vp, C.POINTER(abi.AllocSoa), C.POINTER(vp)]
        L.wva_pairs_commit.argtypes = [vp]
        L.wva_pair_steps.argtypes = [vp, C.POINTER(u64)]
        L.wva_pair_counters.argtypes = [vp, C.POINTER(u64)]
        L.wva_pair_debug.argtypes = [vp, C.POINTER(u64), i32]
        L.wva_analyze_grid.argtypes = [vp, i32, i32, vp, vp, vp]
        L.wva_analyze_grid_device.argtypes = [vp, i32, i32, i32]
        L.wva_grid_fetch.argtypes = [vp, vp]
        L.wva_grid_cube_device.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_size_t)]
        L.wva_solve.argtypes = [vp, C.POINTER(abi.OptimizerSpec), abi.i32p, C.POINTER(abi.AllocSoa)]
        L.wva_solution_fetch.argtypes = [vp, abi.i32p, C.POINTER(abi.AllocSoa)]
        L.wva_allocate_by_type.argtypes = [vp, abi.i64p, abi.f32p]
        L.wva_type_totals_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
        L.wva_solution_time_usec.argtypes = [vp]
        L.wva_solution_time_usec.restype = i64
        L.wva_queue_analyze.argtypes = [vp, i32, vp, abi.f32p, vp, abi.u8p]
        L.wva_queue_size.argtypes = [vp, i32, vp, abi.f32p, abi.f32p, vp, abi.f32p, abi.u8p]
        L.wva_launch_count.argtypes = [vp]
        L.wva_launch_count.restype = i64
        L.wva_phase_time_usec.argtypes = [vp, C.c_int]
        L.wva_phase_time_usec.restype = i64
        L.wva_grid_counters.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
        L.wva_selftest_division.argtypes = [vp, u64, u64, C.c_int, C.POINTER(u64)]
        L.wva_pairs_set_warp_max.argtypes = [vp, i32]
        L.wva_pairs_set_pstore.argtypes = [vp, i32]
        L.wva_solve_set_ranked.argtypes = [vp, i32]
        L.wva_solve_greedy_path.argtypes = [vp]
        L.wva_solve_stats.argtypes = [vp, C.POINTER(C.c_uint64)]
        L.wva_type_totals_merge.argtypes = [vp, C.c_void_p, i32]
        L.wva_set_certified_tails.argtypes = [vp, i32]
        L.wva_analyze.argtypes = [vp, i32, i32, i32]
        L.wva_pairs_fetch.argtypes = [vp, C.POINTER(abi.AllocSoa), abi.u8p]
        L.wva_grid_set_tail_cap.argtypes = [vp, i32]
        L.wva_grid_list_sizes.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
        L.wva_grid_set_fused.argtypes = [vp, i32]
        L.wva_grid_last_fused.argtypes = [vp]
        L.wva_grid_deferred_fetch.argtypes = [vp, C.POINTER(u64), i32, C.POINTER(i32)]
        L.wva_stream.argtypes = [vp]
        L.wva_stream.restype = vp
        L.wva_system_update_servers.argtypes = [vp, i32, i32, C.POINTER(abi.SystemSoa)]
        L.wva_system_update_models.argtypes = [vp, i32, i32, C.POINTER(abi.SystemSoa)]
        L.wva_system_remove_server.argtypes = [vp, i32]
        L.wva_system_set_capacity.argtypes = [vp, abi.i64p]
        L.wva_upload_bytes.argtypes = [vp]
        L.wva_upload_bytes.restype = i64
        L.wva_system_dims.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
        L.wva_model_solve.argtypes = [vp, i64, abi.f32p, i32, i32, abi.f32p, abi.f32p, abi.f32p, C.POINTER(C.c_double)]
        L.wva_comm_unique_id.argtypes = [vp]
        L.wva_comm_init.argtypes = [vp, vp, i32, i32]
        L.wva_comm_destroy.argtypes = [vp]
        L.wva_comm_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
        L.wva_comm_shard.argtypes = [vp]
        L.wva_group_create.argtypes = [abi.i32p, i32, C.POINTER(vp)]
        L.wva_group_destroy.argtypes = [vp]
        L.wva_group_destroy.restype = None
        L.wva_group_size.argtypes = [vp]
        L.wva_group_ctx.argtypes = [vp, i32]
        L.wva_group_ctx.restype = vp
        L.wva_group_last_error.argtypes = [vp]
        L.wva_group_last_error.restype = C.c_char_p
        L.wva_group_upload.argtypes = [vp, C.POINTER(abi.SystemSoa)]
        L.wva_group_analyze.argtypes = [vp, i32, i32, i32]
        L.wva_group_pairs_fetch.argtypes = [vp, C.POINTER(abi.AllocSoa), abi.u8p]
        L.wva_group_grid_fetch.argtypes = [vp, vp]
        L.wva_group_solve.argtypes = [vp, C.POINTER(abi.OptimizerSpec), abi.i32p, C.POINTER(abi.AllocSoa)]
        L.wva_group_allocate_by_type.argtypes = [vp, abi.i64p, abi.f32p]
        L.wva_grid_blocking.argtypes = [vp, abi.f32p]
        L.wva_grid_blocking_size.argtypes = [vp, C.POINTER(C.c_size_t)]
        L.wva_grid_blocking_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
        L.wva_grid_best_blocking.argtypes = [vp, abi.f32p]
        L.wva_grid_blocking_counts.argtypes = [vp, abi.i64p]
        L.wva_grid_blocking_exact_fetch.argtypes = [vp, C.POINTER(u64), i32, C.POINTER(i32)]
        L.wva_group_grid_best_blocking.argtypes = [vp, abi.f32p]
        L.wva_analyze_pairs_batches.argtypes = [vp, i32, abi.i32p, vp, vp]
        L.wva_pairs_batches_counters.argtypes = [vp, C.POINTER(u64)]
        L.wva_group_analyze_pairs_batches.argtypes = [vp, i32, abi.i32p, vp, vp]
        L.wva_shard_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
        L.wva_analyze_pairs_loads.argtypes = [vp, i32, abi.f32p, vp, vp]
        L.wva_pairs_loads_counters.argtypes = [vp, C.POINTER(u64)]
        L.wva_group_analyze_pairs_loads.argtypes = [vp, i32, abi.f32p, vp, vp]
        if L.wva_abi_version() != abi.ABI_VERSION:
            raise ImportError("libwva_b200.so ABI version mismatch")
        _lib = L
    return _lib


def comm_unique_id():
    """128-byte NCCL id (rank 0 creates it, the host distributes it, every rank passes it to Context.comm_init)."""
    buf = C.create_string_buffer(abi.COMM_ID_BYTES)
    rc = lib().wva_comm_unique_id(buf)
    if rc != abi.OK:
        raise WvaError(rc, lib().wva_last_error(None).decode())
    return bytes(buf.raw)


class Context:
    """wva_ctx: one CUDA device, one stream, one call in flight."""

    def __init__(self, device=0, _borrowed=None):
        self._h = C.c_void_p()
        self._owned = _borrowed is None
        if _borrowed is not None:
            self._h = C.c_void_p(_borrowed)
        else:
            rc = lib().wva_ctx_create(int(device), C.byref(self._h))
            if rc != abi.OK:
                raise WvaError(rc, lib().wva_last_error(None).decode())
        self.device = int(device)
        self.image = None

    def close(self):
        if self._h and self._owned:
            lib().wva_ctx_destroy(self._h)
        self._h = C.c_void_p()

    # ---- multi-rank (one process per GPU) ------------------------------------------------
    def comm_init(self, unique_id, rank, n_ranks):
        assert len(unique_id) == abi.COMM_ID_BYTES
        self._ck(lib().wva_comm_init(self._h, C.c_char_p(unique_id), int(rank), int(n_ranks)))

    def comm_destroy(self):
        self._ck(lib().wva_comm_destroy(self._h))

    def comm_info(self):
        r, n = C.c_int32(0), C.c_int32(1)
        self._ck(lib().wva_comm_info(self._h, C.byref(r), C.byref(n)))
        return r.value, n.value

    def comm_shard(self):
        """this rank's contiguous server range of the uploaded image: floor(S*g/G) boundaries"""
        self._ck(lib().wva_comm_shard(self._h))
        r, n = self.comm_info()
        S = self.image.S
        self.first = S * r // n
        self.count = S * (r + 1) // n - self.first

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != abi.OK:
            raise WvaError(rc, lib().wva_last_error(self._h).decode())

    # ---- system ------------------------------------------------------------------------
    def upload(self, image: SystemImage):
        s = image.c_struct()
        self._ck(lib().wva_system_upload(self._h, C.byref(s)))
        self.image = image
        self._read_shard()

    # ---- incremental updates of the resident image (system.go:99-171) ------------------------
    def update_servers(self, first, rows: SystemImage):
        """overwrite / append server rows [first, first+rows.S) from `rows` (its server arrays); self.image follows"""
        s = rows.c_struct()
        self._ck(lib().wva_system_update_servers(self._h, int(first), rows.S, C.byref(s)))
        if rows.S == 0:
            return              # a zero-row update changes nothing, the shard included
        img = self.image
        newS = max(img.S, first + rows.S)
        for name, dt in abi.SRV_FIELDS:
            arr = getattr(img, name)
            if newS > img.S:
                arr = np.concatenate([arr, np.zeros(newS - img.S, dtype=dt)])
            arr[first:first + rows.S] = getattr(rows, name)
            setattr(img, name, arr)
        img.S = newS
        self._read_shard()

    def update_models(self, first, rows: SystemImage):
        s = rows.c_struct()
        self._ck(lib().wva_system_update_models(self._h, int(first), rows.M, C.byref(s)))
        if rows.M == 0:
            return
        img = self.image
        newM = max(img.M, first + rows.M)
        for name, dt in abi.PERF_FIELDS:
            arr = getattr(img, name)
            if newM > img.M:
                arr = np.concatenate([arr, np.zeros((newM - img.M) * img.A, dtype=dt)])
            arr[first * img.A:(first + rows.M) * img.A] = getattr(rows, name)
            setattr(img, name, arr)
        img.M = newM
        self._read_shard()

    def remove_server(self, index):
        """RemoveServer: the last server's row moves into `index`; self.image follows"""
        self._ck(lib().wva_system_remove_server(self._h, int(index)))
        img = self.image
        for name, _ in abi.SRV_FIELDS:
            arr = getattr(img, name)
            arr[index] = arr[img.S - 1]
            setattr(img, name, arr[:img.S - 1].copy())
        img.S -= 1
        self._read_shard()

    def set_capacity(self, type_capacity):
        cap = np.ascontiguousarray(type_capacity, dtype=np.int64)
        self._ck(lib().wva_system_set_capacity(self._h, abi.ptr(cap, C.c_int64)))
        self.image.type_capacity = cap.copy()

    def upload_bytes(self):
        return int(lib().wva_upload_bytes(self._h))

    def dims(self):
        v = [C.c_int32(0) for _ in range(4)]
        self._ck(lib().wva_system_dims(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def _read_shard(self):
        """the library's shard after an upload or update: everything, or the communicator range with one attached"""
        f, n = C.c_int32(0), C.c_int32(0)
        self._ck(lib().wva_shard_info(self._h, C.byref(f), C.byref(n)))
        self.first, self.count = f.value, n.value

    def set_shard(self, first, count):
        self._ck(lib().wva_set_shard(self._h, int(first), int(count)))
        self.first, self.count = int(first), int(count)

    # ---- analyze -----------------------------------------------------------------------
    def analyze_pairs(self, download=True):
        """Server.Calculate for the shard.  Returns (AllocArrays[S*A], feasible[S*A]) (rows outside the
        shard are zero) or None when download is False (results stay on the device)."""
        if not download:
            self._ck(lib().wva_analyze_pairs(self._h, None, None))
            return None
        n = self.image.S * self.image.A
        out = abi.AllocArrays(n)
        feasible = np.zeros(n, dtype=np.uint8)
        self._ck(lib().wva_analyze_pairs(self._h, C.byref(out.c), abi.ptr(feasible, C.c_uint8)))
        return out, feasible

    def analyze(self, r_max, b_max, want_cube=False):
        """Server.Calculate for every pair and the candidate sweep, overlapped; results stay on the device."""
        self._ck(lib().wva_analyze(self._h, int(r_max), int(b_max), 1 if want_cube else 0))

    def pairs_fetch(self):
        n = self.image.S * self.image.A
        out = abi.AllocArrays(n)
        feasible = np.zeros(n, dtype=np.uint8)
        self._ck(lib().wva_pairs_fetch(self._h, C.byref(out.c), abi.ptr(feasible, C.c_uint8)))
        return out, feasible

    def analyze_pairs_batches(self, batch, plane=True):
        """Pair sizing under each batch-size override of `batch` (strictly increasing, values in 1..8192): returns
        (plane, best), numpy arrays of abi.PAIR_REC_DTYPE.  plane[(s - first) * A + a, j] is the record of pair (s, a)
        with ServerSpec.MaxBatchSize = batch[j], or None when plane=False (it then stays off PCIe); best[s - first] is
        SolveUnlimited over the server's records.  Resident results are left as they were."""
        b = np.ascontiguousarray(batch, dtype=np.int32)
        best = np.zeros(self.count, dtype=abi.PAIR_REC_DTYPE)
        pl = np.zeros((self.count * self.image.A, len(b)), dtype=abi.PAIR_REC_DTYPE) if plane else None
        self._ck(lib().wva_analyze_pairs_batches(self._h, len(b), abi.ptr(b, C.c_int32),
                                                 pl.ctypes.data if plane else None, best.ctypes.data))
        return pl, best

    def pairs_batches_counters(self):
        """counters of the last analyze_pairs_batches"""
        v = (C.c_uint64 * 4)()
        self._ck(lib().wva_pairs_batches_counters(self._h, v))
        return dict(slices=v[0], materialised=v[1], steps=v[2], sized=v[3])

    def analyze_pairs_loads(self, rpm, plane=True):
        """Pair sizing under each arrival-rate scenario: rpm [count, n_l] holds the shard's servers'
        ServerLoadSpec.ArrivalRate (req/min) per scenario.  Returns (plane, best), numpy arrays of abi.PAIR_REC_DTYPE:
        plane [count, n_l, A] with plane[s - first, j, a] the record of pair (s, a) at rate rpm[s - first, j], or None
        when plane=False (it then stays off PCIe); best [count, n_l] is SolveUnlimited over each (server, scenario)'s A
        records.  The resident image and results are left as they were."""
        r = np.ascontiguousarray(rpm, dtype=np.float32)
        if r.ndim != 2 or r.shape[0] != self.count:
            raise ValueError("rpm must be shaped [count, n_l]")
        n_l = r.shape[1]
        best = np.zeros((self.count, n_l), dtype=abi.PAIR_REC_DTYPE)
        pl = np.zeros((self.count, n_l, self.image.A), dtype=abi.PAIR_REC_DTYPE) if plane else None
        self._ck(lib().wva_analyze_pairs_loads(self._h, n_l, abi.ptr(r, C.c_float), pl.ctypes.data if plane else None,
                                               best.ctypes.data))
        return pl, best

    def pairs_loads_counters(self):
        """counters of the last analyze_pairs_loads"""
        v = (C.c_uint64 * 5)()
        self._ck(lib().wva_pairs_loads_counters(self._h, v))
        return dict(slices=v[0], sized_pairs=v[1], analyzed=v[2], materialised=v[3], steps=v[4])

    def pair_counters(self):
        v = (C.c_uint64 * 4)()
        self._ck(lib().wva_pair_counters(self._h, v))
        return dict(steps=v[0], rounds_sum=v[1], rounds_max=v[2], trailing=v[3])

    def set_certified_tails(self, on):
        self._ck(lib().wva_set_certified_tails(self._h, int(on)))

    def pair_debug(self):
        n = self.count * self.image.A
        out = np.zeros(2 * n, dtype=np.uint64)
        self._ck(lib().wva_pair_debug(self._h, out.ctypes.data_as(C.POINTER(C.c_uint64)), n))
        return out.reshape(n, 2)

    def pairs_set_pstore(self, on):
        self._ck(lib().wva_pairs_set_pstore(self._h, int(on)))

    def solve_set_ranked(self, on):
        self._ck(lib().wva_solve_set_ranked(self._h, int(on)))

    def type_totals_merge(self, gathered_ptr, n_ranks):
        self._ck(lib().wva_type_totals_merge(self._h, C.c_void_p(int(gathered_ptr)), int(n_ranks)))

    def solve_stats(self):
        v = (C.c_uint64 * 4)()
        self._ck(lib().wva_solve_stats(self._h, v))
        return [int(x) for x in v]

    def solve_greedy_path(self):
        return int(lib().wva_solve_greedy_path(self._h))

    def pairs_set_warp_max(self, n):
        self._ck(lib().wva_pairs_set_warp_max(self._h, int(n)))

    def pair_steps(self):
        v = C.c_uint64(0)
        self._ck(lib().wva_pair_steps(self._h, C.byref(v)))
        return v.value

    def pairs_device(self):
        """Device pointers of the candidate records: dict field -> (address, numpy dtype), plus 'feasible'."""
        dev = abi.AllocSoa()
        fe = C.c_void_p()
        self._ck(lib().wva_pairs_device(self._h, C.byref(dev), C.byref(fe)))
        out = {}
        for name, dt in abi.ALLOC_FIELDS:
            out[name] = (C.cast(getattr(dev, name), C.c_void_p).value, np.dtype(dt))
        out["feasible"] = (fe.value, np.dtype(np.uint8))
        return out

    def pairs_commit(self):
        self._ck(lib().wva_pairs_commit(self._h))

    def analyze_grid(self, r_max, b_max, want_cube=False):
        """Candidate sweep over the shard.  Returns (best[count], cube|None, status|None)."""
        ns = self.count
        best = np.zeros(ns, dtype=abi.GRID_BEST_DTYPE)
        ncand = ns * self.image.A * r_max * b_max
        cube = np.zeros(ncand, dtype=abi.METRICS_DTYPE) if want_cube else None
        status = np.zeros(ncand, dtype=np.uint8) if want_cube else None
        self._ck(lib().wva_analyze_grid(self._h, int(r_max), int(b_max), best.ctypes.data,
                                        cube.ctypes.data if want_cube else None,
                                        status.ctypes.data if want_cube else None))
        return best, cube, status

    def analyze_grid_device(self, r_max, b_max, want_cube=False):
        self._ck(lib().wva_analyze_grid_device(self._h, int(r_max), int(b_max), 1 if want_cube else 0))

    def grid_fetch(self):
        best = np.zeros(self.count, dtype=abi.GRID_BEST_DTYPE)
        self._ck(lib().wva_grid_fetch(self._h, best.ctypes.data))
        return best

    def grid_cube_device(self):
        """(cube address, status address, candidates) of the last sweep's metric cube left on the device."""
        cube, status, n = C.c_void_p(), C.c_void_p(), C.c_size_t()
        self._ck(lib().wva_grid_cube_device(self._h, C.byref(cube), C.byref(status), C.byref(n)))
        return cube.value, status.value, n.value

    def grid_blocking(self, download=True):
        """Blocking probability p_block of every candidate of the last sweep (float32, cube order over the shard; the quiet
        NaN where Analyze does not accept the candidate).  download=False leaves the plane on the device only."""
        if not download:
            self._ck(lib().wva_grid_blocking(self._h, None))
            return None
        n = C.c_size_t()
        self._ck(lib().wva_grid_blocking_size(self._h, C.byref(n)))       # the library's extent, not the caller's
        out = np.empty(n.value, dtype=np.float32)
        self._ck(lib().wva_grid_blocking(self._h, abi.ptr(out, C.c_float)))
        return out

    def grid_blocking_device(self):
        """(address, candidates) of the blocking-probability plane on the device"""
        p, n = C.c_void_p(), C.c_size_t()
        self._ck(lib().wva_grid_blocking_device(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def grid_blocking_counts(self):
        """how the last plane was produced: candidates decided by the certified zero, the certified closed form, an exact chain"""
        out = np.zeros(3, dtype=np.int64)
        self._ck(lib().wva_grid_blocking_counts(self._h, abi.ptr(out, C.c_int64)))
        return dict(zero=int(out[0]), closed_form=int(out[1]), exact=int(out[2]))

    def grid_blocking_exact(self, cap=1 << 24):
        """cube indices (relative to the shard) the last grid_blocking ran as exact chains (sorted, unique)"""
        n = C.c_int32(0)
        ids = np.zeros(cap, dtype=np.uint64)
        self._ck(lib().wva_grid_blocking_exact_fetch(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)), cap, C.byref(n)))
        return np.unique(ids[:min(n.value, cap)]), n.value

    def grid_best_blocking(self):
        """p_block of each server's sweep winner (NaN where no candidate is feasible), [servers of the shard]"""
        out = np.empty(self.count, dtype=np.float32)
        self._ck(lib().wva_grid_best_blocking(self._h, abi.ptr(out, C.c_float)))
        return out

    def grid_set_tail_cap(self, cap):
        self._ck(lib().wva_grid_set_tail_cap(self._h, int(cap)))

    def grid_list_sizes(self):
        a, b = C.c_int32(0), C.c_int32(0)
        self._ck(lib().wva_grid_list_sizes(self._h, C.byref(a), C.byref(b)))
        return dict(deferred=a.value, literal=b.value)

    def grid_set_fused(self, on):
        self._ck(lib().wva_grid_set_fused(self._h, 1 if on else 0))

    def grid_last_fused(self):
        return int(lib().wva_grid_last_fused(self._h))

    def grid_deferred(self, cap=1 << 22):
        """cube indices (relative to the shard) of the candidates the last sweep slice ran as exact chains."""
        n = C.c_int32(0)
        ids = np.zeros(cap, dtype=np.uint64)
        self._ck(lib().wva_grid_deferred_fetch(self._h, ids.ctypes.data_as(C.POINTER(C.c_uint64)), cap, C.byref(n)))
        return ids[:min(n.value, cap)].copy(), n.value

    def grid_counters(self):
        a, b, c = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._ck(lib().wva_grid_counters(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(steps_executed=a.value, steps_algorithmic=b.value, candidates_ok=c.value)

    # ---- optimize ----------------------------------------------------------------------
    def solve(self, unlimited=True, delayed_best_effort=False, policy=abi.POLICY_NONE, download=True):
        """Solver.Solve.  Returns (chosen_acc[S], AllocArrays[S])."""
        spec = abi.OptimizerSpec(1 if unlimited else 0, 1 if delayed_best_effort else 0, int(policy))
        if not download:
            self._ck(lib().wva_solve(self._h, C.byref(spec), None, None))
            return None
        chosen_acc = np.full(self.image.S, -1, dtype=np.int32)
        chosen = abi.AllocArrays(self.image.S)
        self._ck(lib().wva_solve(self._h, C.byref(spec), abi.ptr(chosen_acc, C.c_int32), C.byref(chosen.c)))
        return chosen_acc, chosen

    def solution_fetch(self):
        """The decisions of the last solve (also one made with download=False): (chosen_acc[S], AllocArrays[S])."""
        chosen_acc = np.full(self.image.S, -1, dtype=np.int32)
        chosen = abi.AllocArrays(self.image.S)
        self._ck(lib().wva_solution_fetch(self._h, abi.ptr(chosen_acc, C.c_int32), C.byref(chosen.c)))
        return chosen_acc, chosen

    def allocate_by_type(self, download=True):
        if not download:           # totals stay on the device (type_totals_device)
            self._ck(lib().wva_allocate_by_type(self._h, None, None))
            return None
        count = np.zeros(self.image.T, dtype=np.int64)
        cost = np.zeros(self.image.T, dtype=np.float32)
        self._ck(lib().wva_allocate_by_type(self._h, abi.ptr(count, C.c_int64), abi.ptr(cost, C.c_float)))
        return count, cost

    def type_totals_device(self):
        p, n = C.c_void_p(), C.c_size_t()
        self._ck(lib().wva_type_totals_device(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def solution_time_usec(self):
        return int(lib().wva_solution_time_usec(self._h))

    # ---- pkg/analyzer batched API ----------------------------------------------------
    def queue_analyze(self, cfgs, rates):
        cfgs = np.ascontiguousarray(cfgs, dtype=abi.QUEUE_CONFIG_DTYPE)
        rates = np.ascontiguousarray(rates, dtype=np.float32)
        n = len(cfgs)
        metrics = np.zeros(n, dtype=abi.METRICS_DTYPE)
        status = np.zeros(n, dtype=np.uint8)
        self._ck(lib().wva_queue_analyze(self._h, n, cfgs.ctypes.data, abi.ptr(rates, C.c_float), metrics.ctypes.data,
                                         abi.ptr(status, C.c_uint8)))
        return metrics, status

    def queue_size(self, cfgs, targets):
        cfgs = np.ascontiguousarray(cfgs, dtype=abi.QUEUE_CONFIG_DTYPE)
        targets = np.ascontiguousarray(targets, dtype=np.float32).reshape(-1)
        n = len(cfgs)
        rates = np.zeros(3 * n, dtype=np.float32)
        achieved = np.zeros(3 * n, dtype=np.float32)
        metrics = np.zeros(n, dtype=abi.METRICS_DTYPE)
        status = np.zeros(n, dtype=np.uint8)
        self._ck(lib().wva_queue_size(self._h, n, cfgs.ctypes.data, abi.ptr(targets, C.c_float), abi.ptr(rates, C.c_float),
                                      metrics.ctypes.data, abi.ptr(achieved, C.c_float), abi.ptr(status, C.c_uint8)))
        return rates.reshape(n, 3), metrics, achieved.reshape(n, 3), status

    def model_solve(self, K, serv_rate, lambdas, mus):
        """MM1ModelStateDependent(K, serv_rate): consecutive Solve(lambda, mu) calls on one model -> (out[n, 9], p[K+1])"""
        sr = np.ascontiguousarray(serv_rate, dtype=np.float32)
        lam = np.ascontiguousarray(lambdas, dtype=np.float32); mu = np.ascontiguousarray(mus, dtype=np.float32)
        out = np.zeros((len(lam), 9), dtype=np.float32)
        p = np.zeros(int(K) + 1, dtype=np.float64)
        self._ck(lib().wva_model_solve(self._h, int(K), abi.ptr(sr, C.c_float), len(sr), len(lam), abi.ptr(lam, C.c_float),
                                       abi.ptr(mu, C.c_float), abi.ptr(out.reshape(-1), C.c_float), p.ctypes.data_as(C.POINTER(C.c_double))))
        return out, p

    # ---- instrumentation ---------------------------------------------------------------
    def launch_count(self):
        return int(lib().wva_launch_count(self._h))

    def phase_usec(self, phase):
        return int(lib().wva_phase_time_usec(self._h, int(phase)))

    def stream(self):
        """cudaStream_t (as int) all work of this ctx is enqueued on."""
        return int(lib().wva_stream(self._h) or 0)

    def selftest_division(self, seed, n, mode):
        bad = C.c_uint64(0)
        self._ck(lib().wva_selftest_division(self._h, int(seed), int(n), int(mode), C.byref(bad)))
        return bad.value


class Group:
    """wva_group: ONE process driving several GPUs (the shape of the reference's single reconcile goroutine).
    Servers shard over the devices; host outputs have the full extent; totals are global."""

    def __init__(self, devices):
        devs = np.ascontiguousarray(devices, dtype=np.int32)
        self._h = C.c_void_p()
        rc = lib().wva_group_create(abi.ptr(devs, C.c_int32), len(devs), C.byref(self._h))
        if rc != abi.OK:
            raise WvaError(rc, lib().wva_last_error(None).decode())
        self.n = len(devs)
        self.ctxs = [Context(int(devs[i]), _borrowed=lib().wva_group_ctx(self._h, i)) for i in range(self.n)]
        self.image = None

    def close(self):
        if self._h:
            lib().wva_group_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != abi.OK:
            raise WvaError(rc, lib().wva_group_last_error(self._h).decode())

    def upload(self, image: SystemImage):
        s = image.c_struct()
        self._ck(lib().wva_group_upload(self._h, C.byref(s)))
        self.image = image
        for i, c in enumerate(self.ctxs):
            c.image = image
            c.first = image.S * i // self.n
            c.count = image.S * (i + 1) // self.n - c.first

    def analyze(self, r_max=0, b_max=0, want_cube=False):
        self._ck(lib().wva_group_analyze(self._h, int(r_max), int(b_max), 1 if want_cube else 0))

    def pairs_fetch(self):
        n = self.image.S * self.image.A
        out = abi.AllocArrays(n)
        feasible = np.zeros(n, dtype=np.uint8)
        self._ck(lib().wva_group_pairs_fetch(self._h, C.byref(out.c), abi.ptr(feasible, C.c_uint8)))
        return out, feasible

    def grid_fetch(self):
        best = np.zeros(self.image.S, dtype=abi.GRID_BEST_DTYPE)
        self._ck(lib().wva_group_grid_fetch(self._h, best.ctypes.data))
        return best

    def grid_best_blocking(self):
        """p_block of every server's sweep winner, assembled from the devices' shards [S]"""
        out = np.empty(self.image.S, dtype=np.float32)
        self._ck(lib().wva_group_grid_best_blocking(self._h, abi.ptr(out, C.c_float)))
        return out

    def analyze_pairs_batches(self, batch, plane=True):
        """Context.analyze_pairs_batches over every device's servers, assembled: plane [S * A, n_b], best [S]"""
        b = np.ascontiguousarray(batch, dtype=np.int32)
        best = np.zeros(self.image.S, dtype=abi.PAIR_REC_DTYPE)
        pl = np.zeros((self.image.S * self.image.A, len(b)), dtype=abi.PAIR_REC_DTYPE) if plane else None
        self._ck(lib().wva_group_analyze_pairs_batches(self._h, len(b), abi.ptr(b, C.c_int32),
                                                       pl.ctypes.data if plane else None, best.ctypes.data))
        return pl, best

    def analyze_pairs_loads(self, rpm, plane=True):
        """Context.analyze_pairs_loads over every device's servers, assembled: rpm [S, n_l] -> plane [S, n_l, A],
        best [S, n_l]"""
        r = np.ascontiguousarray(rpm, dtype=np.float32)
        if r.ndim != 2 or r.shape[0] != self.image.S:
            raise ValueError("rpm must be shaped [S, n_l]")
        n_l = r.shape[1]
        best = np.zeros((self.image.S, n_l), dtype=abi.PAIR_REC_DTYPE)
        pl = np.zeros((self.image.S, n_l, self.image.A), dtype=abi.PAIR_REC_DTYPE) if plane else None
        self._ck(lib().wva_group_analyze_pairs_loads(self._h, n_l, abi.ptr(r, C.c_float), pl.ctypes.data if plane else None,
                                                     best.ctypes.data))
        return pl, best

    def solve(self, unlimited=True, delayed_best_effort=False, policy=abi.POLICY_NONE, download=True):
        spec = abi.OptimizerSpec(1 if unlimited else 0, 1 if delayed_best_effort else 0, int(policy))
        if not download:
            self._ck(lib().wva_group_solve(self._h, C.byref(spec), None, None))
            return None
        chosen_acc = np.full(self.image.S, -1, dtype=np.int32)
        chosen = abi.AllocArrays(self.image.S)
        self._ck(lib().wva_group_solve(self._h, C.byref(spec), abi.ptr(chosen_acc, C.c_int32), C.byref(chosen.c)))
        return chosen_acc, chosen

    def allocate_by_type(self, download=True):
        if not download:
            self._ck(lib().wva_group_allocate_by_type(self._h, None, None))
            return None
        count = np.zeros(self.image.T, dtype=np.int64)
        cost = np.zeros(self.image.T, dtype=np.float32)
        self._ck(lib().wva_group_allocate_by_type(self._h, abi.ptr(count, C.c_int64), abi.ptr(cost, C.c_float)))
        return count, cost
