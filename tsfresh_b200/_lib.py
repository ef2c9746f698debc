"""ctypes binding of libtsfx.so (include/tsfx.h).  There is no fallback: if the library is missing or
cannot create a context on a CUDA device, every entry point raises."""
import ctypes
import os
import threading
import weakref

import numpy as np

from .plan import DESC_DTYPE, Plan

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libtsfx.so")

FLAG_DEVICE_PTRS = 1
FLAG_TIMING = 2
FLAG_NO_NAN_CHECK = 4
FLAG_IMPUTE = 8
FLAG_ALL_MEDIANS = 16
PEER_AUTO, PEER_COPY, PEER_STORE, PEER_MULTICAST = 0, 1, 2, 3
IMPUTE_RANGE, IMPUTE_ZERO, IMPUTE_GIVEN, IMPUTE_STATS = 0, 1, 2, 3

_ERR = {-1: ValueError, -2: RuntimeError, -3: NotImplementedError, -4: ValueError, -5: MemoryError, -6: ValueError}

_lib = None
_lock = threading.Lock()

EXPORTS = ["tsfx_ctx_create", "tsfx_ctx_destroy", "tsfx_last_error", "tsfx_sync", "tsfx_version",
           "tsfx_plan_create", "tsfx_plan_destroy", "tsfx_extract_csr", "tsfx_extract_dense",
           "tsfx_extract_long", "tsfx_build_csr", "tsfx_roll_windows", "tsfx_get_timings",
           "tsfx_last_launch_count", "tsfx_last_kernels", "tsfx_kernel_variants", "tsfx_impute", "tsfx_extract_long_alloc", "tsfx_host_alloc", "tsfx_host_free",
           "tsfx_set_peer_outputs", "tsfx_peer_flush", "tsfx_set_max_len_hint", "tsfx_set_row_times", "tsfx_select_classification", "tsfx_extract_long_kinds", "tsfx_device_count", "tsfx_select_regression"]


def load():
    """Loads (building first when nvcc and the sources are newer) and returns the ctypes library."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        from . import build as _build
        if not os.path.exists(LIB_PATH) or os.path.exists(_build.NVCC):
            _build.build()               # no-op when the stamp matches the sources; a box without nvcc uses the shipped .so
        lib = ctypes.CDLL(LIB_PATH)
        vp, i32, i64, u32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32
        lib.tsfx_ctx_create.argtypes = [ctypes.c_int, vp, ctypes.POINTER(vp)]
        lib.tsfx_ctx_destroy.argtypes = [vp]
        lib.tsfx_ctx_destroy.restype = None
        lib.tsfx_last_error.argtypes = [vp]
        lib.tsfx_last_error.restype = ctypes.c_char_p
        lib.tsfx_sync.argtypes = [vp]
        lib.tsfx_plan_create.argtypes = [vp, vp, i32, i32, vp, vp, vp, i32, ctypes.POINTER(vp)]
        lib.tsfx_plan_destroy.argtypes = [vp]
        lib.tsfx_plan_destroy.restype = None
        lib.tsfx_extract_csr.argtypes = [vp, vp, vp, i64, vp, vp, i64, vp, u32]
        lib.tsfx_extract_dense.argtypes = [vp, vp, vp, i64, i32, vp, u32]
        lib.tsfx_extract_long.argtypes = [vp, vp, vp, vp, i32, vp, i64, vp, vp, i64, ctypes.POINTER(i64), u32]
        lib.tsfx_build_csr.argtypes = [vp, vp, vp, i32, vp, i64, vp, vp, vp, vp, i64, ctypes.POINTER(i64)]
        lib.tsfx_roll_windows.argtypes = [vp, vp, i64, i32, i32, i32, vp, vp, vp, vp, i64]
        lib.tsfx_roll_windows.restype = i64
        lib.tsfx_get_timings.argtypes = [vp, vp, vp, i32]
        lib.tsfx_last_launch_count.argtypes = [vp]
        lib.tsfx_last_kernels.argtypes = [vp, vp, i32]
        lib.tsfx_kernel_variants.argtypes = [vp, i32]
        lib.tsfx_impute.argtypes = [vp, vp, i64, i32, i32, vp, u32]
        lib.tsfx_extract_long_alloc.argtypes = [vp, vp, vp, vp, i32, vp, i64, ctypes.POINTER(vp), ctypes.POINTER(vp),
                                                ctypes.POINTER(i64), u32]
        lib.tsfx_host_alloc.argtypes = [vp, ctypes.c_size_t]
        lib.tsfx_host_alloc.restype = vp
        lib.tsfx_host_free.argtypes = [vp, vp]
        lib.tsfx_host_free.restype = None
        lib.tsfx_set_peer_outputs.argtypes = [vp, vp, i32, i32, ctypes.c_uint64, i32]
        lib.tsfx_peer_flush.argtypes = [vp]
        lib.tsfx_set_max_len_hint.argtypes = [vp, i32]
        lib.tsfx_set_row_times.argtypes = [vp, vp, i64, u32]
        lib.tsfx_select_classification.argtypes = [vp, vp, i64, i32, vp, i32, vp, u32]
        lib.tsfx_select_regression.argtypes = [vp, vp, i64, i32, vp, vp, u32]
        lib.tsfx_extract_long_kinds.argtypes = [vp, vp, vp, vp, i32, vp, i32, i64, ctypes.POINTER(vp), ctypes.POINTER(vp),
                                                ctypes.POINTER(i64), u32]
        _lib = lib
        return lib


def device_count():
    return int(load().tsfx_device_count())


def kernel_variants():
    """Every kernel variant name Context.last_kernels can report."""
    lib = load()
    n = lib.tsfx_kernel_variants(None, 0)
    names = (ctypes.c_char_p * n)()
    lib.tsfx_kernel_variants(names, n)
    return [names[i].decode() for i in range(n)]


def _ptr(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


class Context:
    """One per process and device (tsfx_ctx)."""

    def __init__(self, device=0, stream=None):
        self.lib = load()
        h = ctypes.c_void_p()
        rc = self.lib.tsfx_ctx_create(int(device), ctypes.c_void_p(stream) if stream else None, ctypes.byref(h))
        if rc != 0:
            raise _ERR.get(rc, RuntimeError)("tsfx_ctx_create: " + self.lib.tsfx_last_error(None).decode())
        self.h = h
        self.device = int(device)
        self._plans = {}
        self._alive = {"h": h}           # shared with the finalizers of pinned arrays: None once the context is destroyed
        # the context owns device scratch that every entry point reuses: calls on one context are serialised
        # (include/tsfx.h "Threading"); ctypes releases the GIL, so the lock is needed for multi-threaded callers
        self.lock = threading.RLock()

    def close(self):
        if getattr(self, "h", None):
            for p in list(self._plans.values()):
                p.close()
            self._plans.clear()
            self._alive["h"] = None      # pinned arrays still alive keep their memory (not returned to a destroyed pool)
            self.lib.tsfx_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc, what):
        if rc != 0:
            raise _ERR.get(rc, RuntimeError)("%s: %s" % (what, self.lib.tsfx_last_error(self.h).decode()))

    def sync(self):
        self.check(self.lib.tsfx_sync(self.h), "tsfx_sync")

    def timings(self):
        ms = (ctypes.c_float * 16)()
        names = (ctypes.c_char_p * 16)()
        k = self.lib.tsfx_get_timings(self.h, ms, names, 16)
        if k < 0:
            self.check(k, "tsfx_get_timings")
        return {names[i].decode(): float(ms[i]) for i in range(k)}

    def launch_count(self):
        return int(self.lib.tsfx_last_launch_count(self.h))

    def last_kernels(self):
        """The kernel variant every group of the last extract call ran (e.g. "basic/w12/shared"), in group order."""
        names = (ctypes.c_char_p * 16)()
        k = self.lib.tsfx_last_kernels(self.h, names, 16)
        if k < 0:
            self.check(k, "tsfx_last_kernels")
        return [names[i].decode() for i in range(k)]

    def impute(self, matrix, mode=IMPUTE_RANGE, col_stats=None, all_medians=False):
        """tsfx_impute on a host matrix (C-contiguous float64 [rows x cols]), in place.  Returns the
        [3 x cols] array min | max | median (None for IMPUTE_ZERO)."""
        if not (isinstance(matrix, np.ndarray) and matrix.dtype == np.float64 and matrix.flags.c_contiguous
                and matrix.ndim == 2):
            raise ValueError("impute needs a C-contiguous float64 2-d array")
        rows, cols = matrix.shape
        stats = None
        if mode != IMPUTE_ZERO:
            stats = np.full((3, cols), np.nan) if col_stats is None else np.ascontiguousarray(col_stats, dtype=np.float64)
            if stats.shape != (3, cols):
                raise ValueError("col_stats must have shape (3, n_cols)")
        with self.lock:
            rc = self.lib.tsfx_impute(self.h, _ptr(matrix), rows, cols, mode, _ptr(stats),
                                      FLAG_ALL_MEDIANS if all_medians else 0)
            self.check(rc, "tsfx_impute")
        return stats

    def impute_device(self, matrix_ptr, rows, cols, mode=IMPUTE_RANGE):
        rc = self.lib.tsfx_impute(self.h, ctypes.c_void_p(matrix_ptr), rows, cols, mode, None, FLAG_DEVICE_PTRS)
        self.check(rc, "tsfx_impute")

    # ---- pinned host memory (tsfx_host_alloc): numpy arrays the device can copy to / from at full PCIe speed
    def pinned_array(self, shape, dtype):
        """numpy array on page-locked memory from the context's pool; the block returns to the pool when the array
        (and every view / DataFrame built on it) has been garbage collected."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        p = self.lib.tsfx_host_alloc(self.h, max(n, 1))
        if not p:
            raise MemoryError("tsfx_host_alloc(%d bytes) failed" % n)
        return self._wrap_pinned(p, shape, dtype)

    def _wrap_pinned(self, p, shape, dtype):
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        buf = (ctypes.c_char * max(n, 1)).from_address(p)
        arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
        lib, alive = self.lib, self._alive

        def give_back(lib=lib, alive=alive, p=p):
            if alive["h"] is not None:
                lib.tsfx_host_free(alive["h"], ctypes.c_void_p(p))
        weakref.finalize(buf, give_back)
        return arr

    def select_classification(self, X, y_codes, n_classes):
        """tsfx_select_classification on a host matrix: returns [n_classes, n_cols, 8] sufficient statistics"""
        X = np.ascontiguousarray(X, dtype=np.float64)
        y = np.ascontiguousarray(y_codes, dtype=np.int32)
        n, f = X.shape
        out = np.zeros((int(n_classes), f, 8), dtype=np.float64)
        with self.lock:
            rc = self.lib.tsfx_select_classification(self.h, _ptr(X), n, f, _ptr(y), int(n_classes), _ptr(out), 0)
            self.check(rc, "tsfx_select_classification")
        return out

    def select_regression(self, X, y):
        """tsfx_select_regression on host arrays: returns ([n_cols, 8] statistics, (ytie, y0, y1, n))"""
        X = np.ascontiguousarray(X, dtype=np.float64)
        y = np.ascontiguousarray(y, dtype=np.float64)
        n, f = X.shape
        out = np.zeros(f * 8 + 4, dtype=np.float64)
        with self.lock:
            rc = self.lib.tsfx_select_regression(self.h, _ptr(X), n, f, _ptr(y), _ptr(out), 0)
            self.check(rc, "tsfx_select_regression")
        return out[:f * 8].reshape(f, 8), out[f * 8:]

    def set_row_times(self, times_ns):
        """timestamps (int64 ns) of the rows of the NEXT extract call's values (linear_trend_timewise)"""
        t = np.ascontiguousarray(times_ns, dtype=np.int64)
        self.check(self.lib.tsfx_set_row_times(self.h, _ptr(t), len(t), 0), "tsfx_set_row_times")

    # ---- multi-GPU result placement (tsfx_set_peer_outputs)
    def set_peer_outputs(self, peer_ptrs, self_index, multicast_ptr=0, mode=PEER_AUTO):
        arr = (ctypes.c_uint64 * max(1, len(peer_ptrs)))(*[int(x) for x in peer_ptrs])
        rc = self.lib.tsfx_set_peer_outputs(self.h, arr, len(peer_ptrs), int(self_index), int(multicast_ptr), int(mode))
        self.check(rc, "tsfx_set_peer_outputs")

    def peer_flush(self):
        self.check(self.lib.tsfx_peer_flush(self.h), "tsfx_peer_flush")


class DevicePlan:
    """tsfx_plan: the compiled settings on one context."""

    def __init__(self, ctx, plan):
        assert isinstance(plan, Plan)
        self.ctx, self.plan = ctx, plan
        self.n_cols = plan.n_cols
        tables, off, half = plan.cwt_tables()
        descs = np.ascontiguousarray(plan.descs, dtype=DESC_DTYPE)
        h = ctypes.c_void_p()
        rc = ctx.lib.tsfx_plan_create(ctx.h, _ptr(descs), len(descs), plan.n_cols, _ptr(tables), _ptr(off),
                                      _ptr(half), len(half), ctypes.byref(h))
        ctx.check(rc, "tsfx_plan_create")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.ctx.lib.tsfx_plan_destroy(self.h)
            self.h = None

    # ---- host-pointer entry points -------------------------------------------------------------
    def extract_csr(self, values, begin, length, flags=0, times=None):
        values = np.ascontiguousarray(values, dtype=np.float32)
        begin = np.ascontiguousarray(begin, dtype=np.int64)
        length = np.ascontiguousarray(length, dtype=np.int32)
        out = np.empty((len(begin), self.n_cols), dtype=np.float64)
        with self.ctx.lock:
            if times is not None:
                self.ctx.set_row_times(times)
            rc = self.ctx.lib.tsfx_extract_csr(self.ctx.h, self.h, _ptr(values), values.size, _ptr(begin), _ptr(length),
                                               len(begin), _ptr(out), flags)
            self.ctx.check(rc, "tsfx_extract_csr")
        return out

    def extract_dense(self, values2d, flags=0, out=None):
        values2d = np.ascontiguousarray(values2d, dtype=np.float32)
        n, L = values2d.shape
        if out is None:
            out = np.empty((n, self.n_cols), dtype=np.float64)
        with self.ctx.lock:
            rc = self.ctx.lib.tsfx_extract_dense(self.ctx.h, self.h, _ptr(values2d), n, L, _ptr(out), flags)
            self.ctx.check(rc, "tsfx_extract_dense")
        return out

    def extract_long(self, ids, sort_keys, values, flags=0, times=None):
        """(id, sort key, value) rows in any order -> (unique ids ascending, [n_ids x n_cols] matrix).  One C call
        (tsfx_extract_long_alloc): the library sizes the result and returns it on pinned host memory.
        times: int64 ns timestamp of every row (the frame's DatetimeIndex) when the plan has linear_trend_timewise."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        values = np.ascontiguousarray(values, dtype=np.float32)
        is_f64 = 0
        if sort_keys is not None:
            sort_keys = np.asarray(sort_keys)
            if sort_keys.dtype.kind == "f":
                sort_keys = np.ascontiguousarray(sort_keys, dtype=np.float64)
                is_f64 = 1
            else:
                sort_keys = np.ascontiguousarray(sort_keys, dtype=np.int64)
        n_series = ctypes.c_int64(0)
        p_ids, p_out = ctypes.c_void_p(), ctypes.c_void_p()
        ctx = self.ctx
        with ctx.lock:
            if times is not None:
                ctx.set_row_times(times)
            rc = ctx.lib.tsfx_extract_long_alloc(ctx.h, self.h, _ptr(ids), _ptr(sort_keys), is_f64, _ptr(values), len(ids),
                                                 ctypes.byref(p_ids), ctypes.byref(p_out), ctypes.byref(n_series), flags)
            ctx.check(rc, "tsfx_extract_long")
        k = n_series.value
        if k == 0 or not p_out.value:
            return np.empty(0, dtype=np.int64), np.empty((0, self.n_cols), dtype=np.float64)
        return ctx._wrap_pinned(p_ids.value, (k,), np.int64), ctx._wrap_pinned(p_out.value, (k, self.n_cols), np.float64)

    def extract_long_into(self, ids, sort_keys, values, out_ids, out, flags=0):
        """tsfx_extract_long into caller buffers (rows of a larger pinned matrix): returns the number of series written"""
        is_f64 = 0
        if sort_keys is not None and sort_keys.dtype.kind == "f":
            is_f64 = 1
        n_series = ctypes.c_int64(0)
        ctx = self.ctx
        with ctx.lock:
            rc = ctx.lib.tsfx_extract_long(ctx.h, self.h, _ptr(ids), _ptr(sort_keys), is_f64, _ptr(values), len(ids), _ptr(out_ids),
                                           _ptr(out), len(out), ctypes.byref(n_series), flags)
            ctx.check(rc, "tsfx_extract_long")
        return n_series.value

    # ---- device-pointer entry points (torch tensors own the memory) ----------------------------
    def extract_dense_device(self, values_ptr, n_series, length, out_ptr, timing=False):
        flags = FLAG_DEVICE_PTRS | (FLAG_TIMING if timing else 0)
        rc = self.ctx.lib.tsfx_extract_dense(self.ctx.h, self.h, ctypes.c_void_p(values_ptr), n_series, length,
                                             ctypes.c_void_p(out_ptr), flags)
        self.ctx.check(rc, "tsfx_extract_dense")

    def extract_csr_device(self, values_ptr, n_values, begin_ptr, len_ptr, n_series, out_ptr, timing=False, max_len=0):
        """max_len: upper bound of the series lengths if the caller knows one (keeps the call asynchronous)"""
        flags = FLAG_DEVICE_PTRS | (FLAG_TIMING if timing else 0)
        self.ctx.check(self.ctx.lib.tsfx_set_max_len_hint(self.ctx.h, int(max_len)), "tsfx_set_max_len_hint")
        rc = self.ctx.lib.tsfx_extract_csr(self.ctx.h, self.h, ctypes.c_void_p(values_ptr), n_values,
                                           ctypes.c_void_p(begin_ptr), ctypes.c_void_p(len_ptr), n_series,
                                           ctypes.c_void_p(out_ptr), flags)
        self.ctx.check(rc, "tsfx_extract_csr")


def extract_long_kinds(ctx, device_plans, ids, sort_keys, value_columns, flags=0, times=None):
    """Wide format: K value columns sharing ids / sort keys, one DevicePlan per kind -> (unique ids, matrix
    [n_ids x sum of the plans' columns]) from ONE stage (a) (tsfx_extract_long_kinds)."""
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    cols = [np.ascontiguousarray(v, dtype=np.float32) for v in value_columns]
    assert len(cols) == len(device_plans) and all(len(c) == len(ids) for c in cols)
    is_f64 = 0
    if sort_keys is not None:
        sort_keys = np.asarray(sort_keys)
        if sort_keys.dtype.kind == "f":
            sort_keys = np.ascontiguousarray(sort_keys, dtype=np.float64)
            is_f64 = 1
        else:
            sort_keys = np.ascontiguousarray(sort_keys, dtype=np.int64)
    K = len(cols)
    plan_arr = (ctypes.c_void_p * K)(*[dp.h for dp in device_plans])
    val_arr = (ctypes.c_void_p * K)(*[c.ctypes.data for c in cols])
    total = sum(dp.n_cols for dp in device_plans)
    n_series = ctypes.c_int64(0)
    p_ids, p_out = ctypes.c_void_p(), ctypes.c_void_p()
    with ctx.lock:
        if times is not None:
            ctx.set_row_times(times)
        rc = ctx.lib.tsfx_extract_long_kinds(ctx.h, plan_arr, _ptr(ids), _ptr(sort_keys), is_f64, val_arr, K, len(ids),
                                             ctypes.byref(p_ids), ctypes.byref(p_out), ctypes.byref(n_series), flags)
        ctx.check(rc, "tsfx_extract_long_kinds")
    k = n_series.value
    if k == 0 or not p_out.value:
        return np.empty(0, dtype=np.int64), np.empty((0, total), dtype=np.float64)
    return ctx._wrap_pinned(p_ids.value, (k,), np.int64), ctx._wrap_pinned(p_out.value, (k, total), np.float64)


def build_csr(ctx, ids, sort_keys, values):
    """Stage (a) alone: returns (unique_ids, begin, len, values_in_series_order)."""
    ids = np.ascontiguousarray(ids, dtype=np.int64)
    values = np.ascontiguousarray(values, dtype=np.float32)
    is_f64 = 0
    if sort_keys is not None:
        sort_keys = np.asarray(sort_keys)
        if sort_keys.dtype.kind == "f":
            sort_keys = np.ascontiguousarray(sort_keys, dtype=np.float64)
            is_f64 = 1
        else:
            sort_keys = np.ascontiguousarray(sort_keys, dtype=np.int64)
    n = len(ids)
    uid = np.empty(n, dtype=np.int64)
    begin = np.empty(n, dtype=np.int64)
    length = np.empty(n, dtype=np.int32)
    sv = np.empty(n, dtype=np.float32)
    k = ctypes.c_int64(0)
    with ctx.lock:
        rc = ctx.lib.tsfx_build_csr(ctx.h, _ptr(ids), _ptr(sort_keys), is_f64, _ptr(values), n, _ptr(uid), _ptr(begin),
                                    _ptr(length), _ptr(sv), n, ctypes.byref(k))
        ctx.check(rc, "tsfx_build_csr")
    k = k.value
    return uid[:k].copy(), begin[:k].copy(), length[:k].copy(), sv


def roll_windows(begin, length, rolling_direction, max_timeshift, min_timeshift):
    lib = load()
    begin = np.ascontiguousarray(begin, dtype=np.int64)
    length = np.ascontiguousarray(length, dtype=np.int32)
    k = lib.tsfx_roll_windows(_ptr(begin), _ptr(length), len(begin), rolling_direction, max_timeshift, min_timeshift,
                              None, None, None, None, 0)
    if k < 0:
        raise ValueError("tsfx_roll_windows: invalid arguments")
    wb, wl = np.empty(k, dtype=np.int64), np.empty(k, dtype=np.int32)
    wp, we = np.empty(k, dtype=np.int64), np.empty(k, dtype=np.int32)
    k2 = lib.tsfx_roll_windows(_ptr(begin), _ptr(length), len(begin), rolling_direction, max_timeshift, min_timeshift,
                               _ptr(wb), _ptr(wl), _ptr(wp), _ptr(we), k)
    assert k2 == k
    return wb, wl, wp, we
