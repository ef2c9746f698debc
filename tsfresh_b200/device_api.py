"""extract_features_device(): features of series that already live on the GPU, into a float64 matrix on the GPU.

    X, columns = extract_features_device(values)                        # [N, L] or [N, L, K] channels-last
    X, columns = extract_features_device(values, begin, length)         # CSR views: series s = values[begin[s]:+length[s]]

No host copy of the series or of the result: the call enqueues its work on torch's current stream of the tensor's
device and blocks the host once per kind, for the checked pass (include/tsfx.h, TSFX_FLAG_CHECK_DEVICE_INPUT) that
measures the longest series and rejects invalid views and NaN values before any kernel group sees the input.
Columns are named and ordered as `extract_features` names them for the equivalent wide frame (one value column per
kind, no DatetimeIndex, so linear_trend_timewise is skipped); rows follow the input order.

    X, row_ids, columns = extract_features_long_device(ids, values, sort, kind, kinds=[...])   # long format

takes one tensor per column of a long frame, rows in any order, and returns what extract_features returns for that frame
with column_kind: one row per id of any kind (ids ascending), one column block per kind.  Its row count is only known
after the rows are grouped, so the library stages the rows first (tsfx_stage_long_stacked, one host synchronisation)
and torch then allocates the result that the extraction (tsfx_extract_staged) fills.

    X, window_ids, window_keys, columns = extract_features_rolled_device(ids, values, sort, kind, kinds=[...],
                                                                         rolling_direction=32, max_timeshift=255)

is extract_features(roll_time_series(frame, ...)) for the same rows: between the two calls, tsfx_roll_staged turns the
staged series into their rolled windows (views on the staged values) and their union of names, with a second host
synchronisation to learn the number of windows.

    X, package_numbers, package_ids, columns = extract_features_sub_device(ids, values, sort, kind, kinds=[...],
                                                                           sub_length=1000)

is extract_features(add_sub_time_series_index(frame, 1000, ...), column_id="id") for the same rows: tsfx_sub_staged
cuts the staged series into consecutive packages of sub_length rows (views again), named (package number, parent id).

    X, window_keys, y, columns = extract_features_forecasting_device(x, "sensor", max_timeshift=255, rolling_direction=1)

is make_forecasting_frame(x, ...) extracted, with its target vector aligned to the rows of X: the rolled call on one
series whose windows tsfx_roll_staged (TSFX_FLAG_FORECAST) shortens by their last row, and whose targets it reports as
input row numbers that torch gathers from x.

    ex = DeviceExtractor(4096, length=256)                              # or max_length=... for CSR views
    X = ex(values, out=X)                                               # enqueues only: no host synchronisation
    ex.check()                                                          # raises what extract_features_device would have

is extract_features_device prepared once for a batch shape: each call only enqueues work on torch's current stream, so
it overlaps other work and can be captured in a CUDA graph.  Its input is checked on the device (TSFX_FLAG_DEFER_CHECK):
rejected series come out as NaN rows and check() raises the error at a sync point the caller chooses.

    ex = DeviceLongExtractor(max_rows, max_ids, max_length, kinds=[...])
    X, row_ids, n_ids = ex(ids, values, sort, kind, n_rows=None, out=X)   # enqueues only
    ex.check()

is the same for extract_features_long_device: the rows are grouped on the device into a result of max_ids rows
(tsfx_extract_long_deferred), the number of ids stays on the device, and the data errors wait for check().
"""
import numbers

import numpy as np
import pandas as pd

from . import _lib
from .dataframe_functions import impute, impute_dataframe_zero
from .extraction import _check_colname, _default_settings, _device_plan, _kind_plan, _nan_column, get_context


def _layout(values, begin, length, kinds):
    """(number of series, kinds, CSR?) from the shapes and dtypes alone (no device needed)."""
    import torch
    if not isinstance(values, torch.Tensor):
        raise TypeError("values must be a torch.Tensor, not %s" % type(values).__name__)
    if values.dtype not in (torch.float32, torch.float64, torch.float16, torch.bfloat16):
        raise TypeError("values must be float32, float64, float16 or bfloat16, not %s" % values.dtype)
    csr = begin is not None or length is not None
    if csr:
        if begin is None or length is None:
            raise ValueError("begin and length must be given together")
        for name, t in (("begin", begin), ("length", length)):
            if not isinstance(t, torch.Tensor):
                raise TypeError("%s must be a torch.Tensor, not %s" % (name, type(t).__name__))
            if t.ndim != 1:
                raise ValueError("%s must be 1-D, got shape %s" % (name, tuple(t.shape)))
        if begin.dtype != torch.int64:
            raise TypeError("begin must be int64, not %s" % begin.dtype)
        if length.dtype not in (torch.int32, torch.int64):
            raise TypeError("length must be int32 or int64, not %s" % length.dtype)
        if begin.shape[0] != length.shape[0]:
            raise ValueError("begin has %d entries, length %d" % (begin.shape[0], length.shape[0]))
        if values.ndim not in (1, 2):
            raise ValueError("CSR values must be [R] or [R, K], got shape %s" % (tuple(values.shape),))
        n, n_kinds = begin.shape[0], (1 if values.ndim == 1 else values.shape[1])
    else:
        if values.ndim not in (2, 3):
            raise ValueError("dense values must be [N, L] or [N, L, K], got shape %s" % (tuple(values.shape),))
        if values.shape[1] > 0x7fffffff:
            raise ValueError("series of %d samples" % values.shape[1])
        n, n_kinds = values.shape[0], (1 if values.ndim == 2 else values.shape[2])
    if n_kinds < 1:
        raise ValueError("values has no kind (K = 0)")
    kinds = list(range(n_kinds)) if kinds is None else list(kinds)
    if len(kinds) != n_kinds:
        raise ValueError("%d kinds named for %d in values" % (len(kinds), n_kinds))
    if len(set(map(str, kinds))) != len(kinds):
        raise ValueError("kinds must have distinct names: %r" % (kinds,))
    _check_colname(*kinds)
    return n, kinds, csr


def _plans(kinds, default_fc_parameters, kind_to_fc_parameters):
    """One Plan per kind and the result's column names, as extract_features gives them for a wide frame."""
    default_fc_parameters = _default_settings(default_fc_parameters, kind_to_fc_parameters)
    plans, columns = [], []
    for kind in kinds:
        plan, names = _kind_plan(kind, default_fc_parameters, kind_to_fc_parameters)
        plans.append(plan)
        columns += names
    return plans, columns


def _check_out(out, n, width):
    import torch
    if not isinstance(out, torch.Tensor):
        raise TypeError("out must be a torch.Tensor, not %s" % type(out).__name__)
    if out.dtype != torch.float64:
        raise TypeError("out must be float64, not %s" % out.dtype)
    if tuple(out.shape) != (n, width):
        raise ValueError("out has shape %s, the result is (%d, %d)" % (tuple(out.shape), n, width))
    if n > 0 and width > 0 and ((width > 1 and out.stride(1) != 1) or out.stride(0) < width):
        raise ValueError("out must have unit column stride and a row stride >= its width (got strides %s)" % (out.stride(),))


def extract_features_device(values, begin=None, length=None, *, default_fc_parameters=None, kind_to_fc_parameters=None,
                            kinds=None, impute_function=None, out=None):
    """Extracts features from CUDA tensors into a CUDA tensor.

    values: [N, L] or channels-last [N, L, K] (dense), or [R] / [R, K] with `begin` (int64) and `length` (int32 or
    int64) CUDA tensors of N entries (series s is values[begin[s] : begin[s] + length[s]]; views may overlap).
    float32 is read in place; float64, float16 and bfloat16 are rounded to float32 on the device.
    default_fc_parameters / kind_to_fc_parameters: as extract_features; `kinds` names the K kinds (default 0 .. K-1).
    impute_function: impute or impute_dataframe_zero impute on the device; any other callable gets a host DataFrame.
    out: a float64 CUDA tensor [N, n_features] (or a column slice of a wider one) to fill instead of a new one.

    Returns (X, columns): X float64 [N, n_features] on values' device, rows in input order.  Raises ValueError for
    NaN values, invalid views and series longer than the plan allows, before any feature kernel runs."""
    import torch
    n, kinds, csr = _layout(values, begin, length, kinds)
    plans, columns = _plans(kinds, default_fc_parameters, kind_to_fc_parameters)
    width = len(columns)
    if out is not None:
        _check_out(out, n, width)
    dev = values.device
    if dev.type != "cuda":
        raise ValueError("values must be a CUDA tensor, got one on %s" % dev)
    for name, t in (("begin", begin), ("length", length), ("out", out)):
        if t is not None and t.device != dev:
            raise ValueError("%s is on %s, values on %s" % (name, t.device, dev))
    mode = _lib.IMPUTE_RANGE if impute_function is impute else _lib.IMPUTE_ZERO if impute_function is impute_dataframe_zero else None
    with torch.cuda.device(dev):
        X = out if out is not None else torch.empty((n, width), dtype=torch.float64, device=dev)
        if n == 0 or width == 0:
            return X, columns
        v = values if values.dtype == torch.float32 else values.to(torch.float32)
        if csr:
            b = begin.contiguous()
            # int64 lengths beyond int32 become lengths the checked pass rejects, never wrapped-around valid ones
            ln = length.contiguous() if length.dtype == torch.int32 else length.clamp(0, 0x7fffffff).to(torch.int32)
        # device imputation needs the whole matrix contiguous: a strided `out` is filled through a contiguous one
        target = X if (mode is None or X.stride(0) == width) else torch.empty((n, width), dtype=torch.float64, device=dev)
        ctx = get_context(dev.index)
        stream = torch.cuda.current_stream(dev).cuda_stream
        scratch = None
        with ctx.lock:
            ctx.set_stream(stream or _lib.STREAM_LEGACY)
            try:
                ctx.set_out_ld(target.stride(0))
                c0 = 0
                for k, plan in enumerate(plans):
                    if plan.n_cols == 0:
                        continue
                    if v.ndim == (2 if csr else 3):             # channels-last: this kind's values, contiguous
                        scratch = torch.empty(v.shape[:-1], dtype=torch.float32, device=dev) if scratch is None else scratch
                        col = scratch.copy_(v[..., k])
                    else:
                        col = v.contiguous()
                    dp = _device_plan(ctx, plan)
                    o = target.data_ptr() + c0 * 8
                    with _nan_column(kinds[k]):
                        if csr:
                            dp.extract_csr_device(col.data_ptr(), col.shape[0], b.data_ptr(), ln.data_ptr(), n, o, checked=True)
                        else:
                            dp.extract_dense_device(col.data_ptr(), n, col.shape[1], o, checked=True)
                    c0 += plan.n_cols
                if mode is not None:
                    ctx.impute_device(target.data_ptr(), n, width, mode)
            finally:
                ctx.set_out_ld(0)
                ctx.set_stream(None)
        if target is not X:
            X.copy_(target)
    if impute_function is not None and mode is None:
        df = pd.DataFrame(X.cpu().numpy(), columns=columns)
        impute_function(df)
        X.copy_(torch.from_numpy(df.to_numpy(dtype=np.float64)))
    return X, columns


class DeviceExtractor:
    """extract_features_device prepared for one batch shape, for calls that only enqueue work.

        ex = DeviceExtractor(batch_size, length=L)            # dense [n, L] or channels-last [n, L, K], n <= batch_size
        ex = DeviceExtractor(batch_size, max_length=M)        # CSR views (values, begin, length), each <= M samples
        X = ex(values, out=None)  /  X = ex(values, begin, length, out=None)
        ex.check()

    kinds, default_fc_parameters and kind_to_fc_parameters are as for extract_features_device (kinds default: one kind,
    named 0); `columns` are the names it gives.  device: the CUDA device of the inputs (default: the current one).

    The plans are compiled, their length limits checked against length / max_length (ValueError), and every working
    buffer sized once, here.  The extractor owns a private library context, so calls never share scratch with the eager
    API or another extractor (and may be replayed from a CUDA graph on any stream): 256 MB of working memory (1 GB when
    length / max_length exceeds 1 024) plus the per-kind staging matrices (batch_size x staged columns x 8 bytes) and 13
    bytes per series of check buffers.  Calls on one extractor are stream-ordered: use one extractor per concurrent
    stream.

    A call checks the tensors' shapes, dtypes and devices, and `out`, at once (TypeError / ValueError, nothing enqueued).
    It then enqueues on torch's current stream, with no host synchronisation, no allocation in the library and no read
    of device memory on the host; float64, float16 and bfloat16 are rounded to float32 on the device.  The data are
    checked on the device: a series with a NaN value, an invalid view (len < 1, begin < 0, begin + len > R) or a view
    longer than max_length is rejected.  Every other row is what extract_features_device gives (bit for bit for dense
    input and for views whose longest equals max_length; a shorter longest view may select other kernel variants, which
    agree within the oracle parity); a rejected row is NaN in every column of its kind.  check() synchronises the device
    and raises the ValueError extract_features_device would have raised for the first call since the last check() that
    rejected a series, then clears that state.  impute_function is not offered (imputation synchronises): impute X
    afterwards."""

    def __init__(self, batch_size, length=None, max_length=None, *, kinds=None, default_fc_parameters=None,
                 kind_to_fc_parameters=None, device=None):
        import torch
        if (length is None) == (max_length is None):
            raise ValueError("give exactly one of length (dense input) or max_length (CSR views)")
        for name, v in (("batch_size", batch_size), ("length", length), ("max_length", max_length)):
            if v is not None and (not isinstance(v, numbers.Integral) or not 1 <= v <= 0x7fffffff):
                raise ValueError("%s must be an integer in 1 .. 2^31 - 1, got %r" % (name, v))
        self.batch_size, self.length, self.max_length = int(batch_size), length, max_length
        kinds = [0] if kinds is None else list(kinds)
        _layout(torch.empty((0, 1, len(kinds)), device="meta"), None, None, kinds)      # the kinds' names, as a call checks them
        self.kinds = kinds
        self._plans, self.columns = _plans(kinds, default_fc_parameters, kind_to_fc_parameters)
        longest = length if length is not None else max_length
        for kind, plan in zip(kinds, self._plans):
            limit = _lib.plan_max_len(plan)
            if longest > limit:
                raise ValueError("series of %d samples exceed the limit of kind %r's settings (%d samples)" % (longest, kind, limit))
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("device must be a CUDA device, got %s" % self.device)
        self._open()

    def _open(self):
        """The private context, its prepared plans and the status words (tsfx.h "Deferred input check")."""
        import torch
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._ctx = _lib.Context(self.device.index)
        self._dps = [None if p.n_cols == 0 else _device_plan(self._ctx, p) for p in self._plans]
        for dp in self._dps:
            if dp is not None:
                dp.prepare(self.batch_size, self.length or self.max_length)
        self._status = torch.zeros(_lib.STATUS_WORDS, dtype=torch.int64, device=self.device)
        self._ctx.set_status(self._status.data_ptr())

    def __call__(self, values, begin=None, length=None, out=None):
        import torch
        n, _, csr = _layout(values, begin, length, self.kinds)
        if csr != (self.max_length is not None):
            raise ValueError("this extractor takes %s" % ("CSR views (values, begin, length)" if self.max_length is not None
                                                           else "dense [n, length] or [n, length, K] values"))
        if n > self.batch_size:
            raise ValueError("%d series, the extractor was built for at most %d" % (n, self.batch_size))
        if not csr and values.shape[1] != self.length:
            raise ValueError("series of %d samples, the extractor was built for length=%d" % (values.shape[1], self.length))
        if csr and n > 0 and values.shape[0] == 0:
            raise ValueError("values is empty")
        width = len(self.columns)
        if out is not None:
            _check_out(out, n, width)
        dev = self.device
        for name, t in (("values", values), ("begin", begin), ("length", length), ("out", out)):
            if t is not None and t.device != dev:
                raise ValueError("%s is on %s, the extractor on %s" % (name, t.device, dev))
        with torch.cuda.device(dev):
            X = out if out is not None else torch.empty((n, width), dtype=torch.float64, device=dev)
            if n == 0 or width == 0:
                return X
            v = values if values.dtype == torch.float32 else values.to(torch.float32)
            if csr:
                b = begin.contiguous()
                # int64 lengths beyond int32 become lengths the check rejects, never wrapped-around valid ones
                ln = length.contiguous() if length.dtype == torch.int32 else length.clamp(0, 0x7fffffff).to(torch.int32)
            ctx = self._ctx
            scratch = None
            with ctx.lock:
                # the context stays bound to the stream it last ran on: rebinding it after a capture would order a
                # stream outside the graph after work inside it
                ctx.set_stream(torch.cuda.current_stream(dev).cuda_stream or _lib.STREAM_LEGACY)
                ctx.set_out_ld(X.stride(0))
                c0 = 0
                for k, dp in enumerate(self._dps):
                    if dp is None:
                        continue
                    if v.ndim == (2 if csr else 3):             # channels-last: this kind's values, contiguous
                        scratch = torch.empty(v.shape[:-1], dtype=torch.float32, device=dev) if scratch is None else scratch
                        col = scratch.copy_(v[..., k])
                    else:
                        col = v.contiguous()
                    o = X.data_ptr() + c0 * 8
                    if csr:
                        dp.extract_csr_device(col.data_ptr(), col.shape[0], b.data_ptr(), ln.data_ptr(), n, o,
                                              max_len=self.max_length, deferred=True)
                    else:
                        dp.extract_dense_device(col.data_ptr(), n, col.shape[1], o, deferred=True)
                    c0 += dp.n_cols
        return X

    def check(self):
        """Synchronises the device; raises the ValueError of the first call since the last check() that rejected a
        series (then forgets it)."""
        import torch
        torch.cuda.synchronize(self.device)
        st = self._status.cpu().tolist()
        bad = st[_lib.STATUS_BAD]
        if bad == 0:
            return
        self._status[_lib.STATUS_BAD] = 0
        torch.cuda.synchronize(self.device)
        active = [k for k, dp in zip(self.kinds, self._dps) if dp is not None]
        kind = active[(bad - 1) % len(active)]                # every call makes one library call per kind with columns
        if st[_lib.STATUS_VIEW] >= 0:
            raise ValueError("series %d has an invalid (begin, len): len < 1, begin < 0 or begin + len > n_values"
                             % st[_lib.STATUS_VIEW])
        if st[_lib.STATUS_LONG] >= 0:
            raise ValueError("series %d is longer than max_length=%d" % (st[_lib.STATUS_LONG], self.max_length))
        raise ValueError("Column must not contain NaN values: {} (first in series {})".format(kind, st[_lib.STATUS_NAN]))


def _long_layout(ids, values, sort, kind, kinds, times, need_ids=True):
    """(number of rows, kind names) of long-format row tensors from their shapes and dtypes alone (no device needed).
    need_ids=False: ids may be None (every row belongs to one id)."""
    import torch
    columns = (("ids", ids), ("values", values), ("sort", sort), ("kind", kind), ("times", times))
    for name, t in columns:
        if t is None and (name == "values" or (name == "ids" and need_ids)):
            raise TypeError("%s must be a torch.Tensor, not None" % name)
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor, not %s" % (name, type(t).__name__))
        if t.ndim != 1:
            raise ValueError("%s must be 1-D, got shape %s" % (name, tuple(t.shape)))
    if ids is not None and ids.dtype != torch.int64:
        raise TypeError("ids must be int64, not %s" % ids.dtype)
    if values.dtype not in (torch.float32, torch.float64, torch.float16, torch.bfloat16):
        raise TypeError("values must be float32, float64, float16 or bfloat16, not %s" % values.dtype)
    if sort is not None and sort.dtype not in (torch.int64, torch.float64):
        raise TypeError("sort must be int64 or float64, not %s" % sort.dtype)
    if kind is not None and kind.dtype not in (torch.int32, torch.int64):
        raise TypeError("kind must be int32 or int64, not %s" % kind.dtype)
    if times is not None and times.dtype != torch.int64:
        raise TypeError("times must be int64 nanoseconds, not %s" % times.dtype)
    n, by = (values.shape[0], "values") if ids is None else (ids.shape[0], "ids")
    for name, t in columns[1:]:
        if t is not None and t.shape[0] != n:
            raise ValueError("%s has %d rows, %s %d" % (name, t.shape[0], by, n))
    if n > (1 << 31) - 2 - 64 * 64:
        raise ValueError("%d rows: at most 2^31 - 4 098 in one call" % n)
    if kind is None:
        kinds = ["value"] if kinds is None else list(kinds)
        if len(kinds) != 1:
            raise ValueError("without kind codes there is one kind, %d named" % len(kinds))
    else:
        if kinds is None:
            raise ValueError("kinds must name the kinds that the codes 0 .. K-1 of kind stand for")
        kinds = list(kinds)
        if not 1 <= len(kinds) <= 64:
            raise ValueError("between 1 and 64 kinds, %d named" % len(kinds))
    if len(set(map(str, kinds))) != len(kinds):
        raise ValueError("kinds must have distinct names: %r" % (kinds,))
    _check_colname(*kinds)
    return n, kinds


def extract_features_long_device(ids, values, sort=None, kind=None, *, kinds=None, times=None, default_fc_parameters=None,
                                 kind_to_fc_parameters=None, impute_function=None):
    """Extracts features from long-format rows held in CUDA tensors into a CUDA tensor.

    ids (int64), values, sort, kind and times are 1-D CUDA tensors with one entry per row, rows in any order.
    values: float32 is read in place; float64, float16 and bfloat16 are rounded to float32 on the device.
    sort: int64 or float64 sort keys (None: rows keep their input order); equal keys keep their input order.
    kind: int32 or int64 codes 0 .. K-1 of the kinds that `kinds` names (None: one kind, named "value").
    times: int64 nanosecond timestamp of every row; given, linear_trend_timewise is computed as extract_features computes
    it for a frame with that DatetimeIndex.
    default_fc_parameters / kind_to_fc_parameters / impute_function: as extract_features_device.

    Returns (X, row_ids, columns), what extract_features returns for the equivalent frame with column_kind: row_ids
    (int64, CUDA) is the ascending union of the ids of every kind, X float64 [len(row_ids), len(columns)] on values'
    device, one column block per kind in code order, NaN where an id has no rows of a kind; a kind without rows has no
    columns.  Runs on torch's current stream and blocks the host once, to learn the number of ids.  Raises ValueError for
    NaN values or sort keys, kind codes out of range and series longer than their kind's plan allows, before any feature
    kernel runs."""
    X, row_ids, _, columns, _ = _extract_staged(ids, values, sort, kind, kinds, times, None, default_fc_parameters,
                                                kind_to_fc_parameters, impute_function)
    return X, row_ids, columns


class DeviceLongExtractor:
    """extract_features_long_device prepared for one shape, for calls that only enqueue work.

        ex = DeviceLongExtractor(max_rows, max_ids, max_length, kinds=[...])
        X, row_ids, n_ids = ex(ids, values, sort=None, kind=None, n_rows=None, out=None)
        ex.check()

    A call takes at most max_rows long-format rows (ids, values, sort, kind as extract_features_long_device takes them,
    rows in any order, times not offered) with at most max_ids distinct ids and (id, kind) series of at most max_length
    samples.  kinds names the kind codes 0 .. K-1 (at most 64; None: one kind, "value"); default_fc_parameters and
    kind_to_fc_parameters are as for extract_features_long_device, and `columns` are the names of ALL kinds' columns.
    device: the CUDA device of the inputs (default: the current one).

    The constructor compiles the plans, checks max_length against every plan's length limit (ValueError) and prepares a
    private library context once: the stage's buffers for max_rows rows (about 90 bytes per row), the slot and check
    buffers of K x max_ids series (29 bytes each), a staging block per kind (max_ids x its columns x 8 bytes) and what
    DeviceExtractor prepares per plan for max_ids series of max_length samples.

    A call checks the tensors' metadata at once (TypeError / ValueError, nothing enqueued): the layout checks of
    extract_features_long_device, at most max_rows rows, one device, `out`, and n_rows.  It then only enqueues work on
    torch's current stream: no host synchronisation, no allocation in the library, no read of device memory on the host.
    values other than float32 are rounded to float32 on the device.  n_rows, a 0-d int64 CUDA tensor, makes only rows
    [0, n_rows) count, so a captured graph can be replayed with another row count every step.

    Returns X (float64 [max_ids, len(columns)]), row_ids (int64 [max_ids]) and n_ids (0-d int64), all on the device.
    Rows [0, n_ids) of X are extract_features_long_device's rows for the same data, ids ascending in row_ids, and the
    rows past n_ids are NaN, with row_ids 2**63 - 1, so row_ids stays ascending.  Unlike extract_features_long_device,
    whose result has no columns for a kind without rows, X always has every kind's columns: a kind without rows in the
    call has NaN columns.  With the longest series of every kind equal to max_length the rows are equal bit for bit; a
    shorter longest series may select other kernel variants, which agree within the oracle parity.

    The data are checked on the device.  A kind code outside 0 .. K-1, a NaN float64 sort key or more than max_ids
    distinct ids reject the whole call (X all NaN, n_ids 0); a NaN value or more than max_length samples in the series
    of an (id, kind) pair make that series' cells NaN in its kind's columns.  check() synchronises the device and raises
    the ValueError of the first call since the last check() that met such an error, then forgets it: the message of
    extract_features_long_device for a kind code, a NaN sort key or a NaN value; a message naming max_ids or max_length
    and the id for the two limits.  impute_function and times (linear_trend_timewise) are not offered, as for
    DeviceExtractor: imputation synchronises, and times would add a column only some calls could fill."""

    def __init__(self, max_rows, max_ids, max_length, *, kinds=None, default_fc_parameters=None,
                 kind_to_fc_parameters=None, device=None):
        import torch
        for name, v, top in (("max_rows", max_rows, _MAX_ROWS), ("max_ids", max_ids, _I32_MAX),
                             ("max_length", max_length, _I32_MAX)):
            if not isinstance(v, numbers.Integral) or not 1 <= v <= top:
                raise ValueError("%s must be an integer in 1 .. %d, got %r" % (name, top, v))
        self.max_rows, self.max_ids, self.max_length = int(max_rows), int(max_ids), int(max_length)
        kinds = ["value"] if kinds is None else list(kinds)
        if not 1 <= len(kinds) <= 64:
            raise ValueError("between 1 and 64 kinds, %d named" % len(kinds))
        if len(set(map(str, kinds))) != len(kinds):
            raise ValueError("kinds must have distinct names: %r" % (kinds,))
        _check_colname(*kinds)
        self.kinds = kinds
        self._plans, self.columns = _plans(kinds, default_fc_parameters, kind_to_fc_parameters)
        for kind, plan in zip(kinds, self._plans):
            limit = _lib.plan_max_len(plan)
            if self.max_length > limit:
                raise ValueError("series of %d samples exceed the limit of kind %r's settings (%d samples)"
                                 % (self.max_length, kind, limit))
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("device must be a CUDA device, got %s" % self.device)
        self._open()

    def _open(self):
        """The private context, its prepared shape and the status words (tsfx.h "Deferred long format")."""
        import torch
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._ctx = _lib.Context(self.device.index)
        self._dps = [None if p.n_cols == 0 else _device_plan(self._ctx, p) for p in self._plans]
        self._ctx.prepare_long(self._dps, self.max_rows, self.max_ids, self.max_length)
        self._status = torch.zeros(_lib.STATUS_WORDS, dtype=torch.int64, device=self.device)
        self._ctx.set_status(self._status.data_ptr())

    def __call__(self, ids, values, sort=None, kind=None, n_rows=None, out=None):
        import torch
        n, _ = _long_layout(ids, values, sort, kind, self.kinds, None)
        if n > self.max_rows:
            raise ValueError("%d rows, the extractor was built for at most %d" % (n, self.max_rows))
        if n_rows is not None:
            if not isinstance(n_rows, torch.Tensor):
                raise TypeError("n_rows must be a torch.Tensor, not %s" % type(n_rows).__name__)
            if n_rows.dtype != torch.int64 or n_rows.ndim != 0:
                raise ValueError("n_rows must be a 0-d int64 tensor, got %s of shape %s" % (n_rows.dtype, tuple(n_rows.shape)))
        width = len(self.columns)
        if out is not None:
            _check_out(out, self.max_ids, width)
        dev = self.device
        for name, t in (("ids", ids), ("values", values), ("sort", sort), ("kind", kind), ("n_rows", n_rows), ("out", out)):
            if t is not None and t.device != dev:
                raise ValueError("%s is on %s, the extractor on %s" % (name, t.device, dev))
        with torch.cuda.device(dev):
            X = out if out is not None else torch.empty((self.max_ids, width), dtype=torch.float64, device=dev)
            row_ids = torch.empty(self.max_ids, dtype=torch.int64, device=dev)
            n_ids = torch.empty((), dtype=torch.int64, device=dev)
            v = values.contiguous() if values.dtype == torch.float32 else values.to(torch.float32).contiguous()
            i, s = ids.contiguous(), None if sort is None else sort.contiguous()
            k = None if kind is None else kind.contiguous()
            ctx = self._ctx
            with ctx.lock:
                # bound to the stream it last ran on, as DeviceExtractor: see there
                ctx.set_stream(torch.cuda.current_stream(dev).cuda_stream or _lib.STREAM_LEGACY)
                ctx.extract_long_deferred(i.data_ptr() if n else 0, 0 if s is None else s.data_ptr(),
                                          s is not None and s.dtype == torch.float64, v.data_ptr() if n else 0,
                                          0 if k is None else k.data_ptr(), k is not None and k.dtype == torch.int64, n,
                                          0 if n_rows is None else n_rows.data_ptr(), row_ids.data_ptr(), n_ids.data_ptr(),
                                          X.data_ptr() if width else 0, X.stride(0) if width else 0)
        return X, row_ids, n_ids

    def check(self):
        """Synchronises the device; raises the ValueError of the first call since the last check() that met a data
        error (then forgets it)."""
        import torch
        torch.cuda.synchronize(self.device)
        st = self._status.cpu().tolist()
        if st[_lib.STATUS_BAD] == 0:
            return
        self._status[_lib.STATUS_BAD] = 0
        torch.cuda.synchronize(self.device)
        what = "tsfx_stage_long_stacked"            # the eager call's messages name the stage that raises them
        if st[_lib.STATUS_KIND]:
            raise ValueError("%s: a kind code is outside 0 .. %d" % (what, len(self.kinds) - 1))
        if st[_lib.STATUS_KEY_NAN]:
            raise _lib.NanValuesError("%s: the float64 sort keys contain NaN" % what)
        if st[_lib.STATUS_IDS]:
            raise ValueError("%d distinct ids, more than max_ids=%d: id %d is the first past them"
                             % (st[_lib.STATUS_IDS], self.max_ids, st[_lib.STATUS_ID]))
        if st[_lib.STATUS_NAN] >= 0:
            raise _lib.NanValuesError("%s: the value column contains NaN" % what)
        raise ValueError("the series of id %d and kind %r is longer than max_length=%d"
                         % (st[_lib.STATUS_ID], self.kinds[st[_lib.STATUS_LONG] // self.max_ids], self.max_length))


_I32_MAX = (1 << 31) - 1
_MAX_ROWS = (1 << 31) - 2 - 64 * 64


def _roll_args(rolling_direction, max_timeshift, min_timeshift):
    """roll_time_series's argument errors, with its messages; then the arguments as tsfx_roll_staged takes them (int32,
    max_timeshift 0 for None; values beyond int32 act as the largest one would)"""
    if rolling_direction == 0:
        raise ValueError("Rolling direction of 0 is not possible")
    if max_timeshift is not None and max_timeshift <= 0:
        raise ValueError("max_timeshift needs to be positive!")
    if min_timeshift < 0:
        raise ValueError("min_timeshift needs to be positive or zero!")
    direction = max(-_I32_MAX, min(int(rolling_direction), _I32_MAX))
    return direction, 0 if max_timeshift is None else min(int(max_timeshift), _I32_MAX), min(int(min_timeshift), _I32_MAX)


def extract_features_rolled_device(ids, values, sort=None, kind=None, *, kinds=None, rolling_direction=1, max_timeshift=None,
                                   min_timeshift=0, default_fc_parameters=None, kind_to_fc_parameters=None,
                                   impute_function=None):
    """Extracts features from the rolled windows of long-format rows held in CUDA tensors into a CUDA tensor.

    ids, values, sort, kind, kinds, default_fc_parameters, kind_to_fc_parameters and impute_function: as
    extract_features_long_device.  rolling_direction, max_timeshift and min_timeshift: as roll_time_series.

    Returns (X, window_ids, window_keys, columns), what extract_features returns for roll_time_series(df, column_id="id",
    column_sort="time", column_kind="kind", ...) of the equivalent frame: row r of X is the window named (window_ids[r],
    window_keys[r]), names ascending.  window_ids is int64; window_keys has the sort keys' dtype, or is int64 holding the
    row number inside the series with sort=None.  A window is named by its last row for a positive direction and by its
    first row for a negative one.  Every kind rolls on its own, the shifts anchored to the longest (kind, id) series; the
    rows are the union of the window names over all kinds, NaN where a kind has no window of that name.  Like the rolled
    frame, linear_trend_timewise is skipped.  The quadratic entropies' length limit applies to each window, not to the
    series it comes from.

    Runs on torch's current stream and blocks the host twice: to group the rows and to count the windows.  Raises
    roll_time_series's errors for its arguments before the device is touched, and ValueError for two windows of one kind
    with the same name (sort keys tied at their naming rows), NaN values or sort keys, kind codes out of range and windows
    longer than their kind's plan allows, before any feature kernel runs."""
    regroup = ("roll",) + _roll_args(rolling_direction, max_timeshift, min_timeshift)
    return _extract_staged(ids, values, sort, kind, kinds, None, regroup, default_fc_parameters, kind_to_fc_parameters,
                           impute_function)[:4]


def extract_features_forecasting_device(x, kind, max_timeshift, rolling_direction, min_timeshift=0, *, index=None,
                                        default_fc_parameters=None, kind_to_fc_parameters=None, impute_function=None):
    """Extracts features from the forecasting windows of one series held in a CUDA tensor, with their targets.

    x: 1-D CUDA tensor, float32, float64, float16 or bfloat16 (rounded to float32 for the features).  index: 1-D CUDA
    tensor of int64 or float64 sort keys, the role of a pd.Series' index (None: 0 .. n-1; datetimes as int64
    nanoseconds).  kind, max_timeshift, rolling_direction and min_timeshift: as make_forecasting_frame.
    default_fc_parameters, kind_to_fc_parameters and impute_function: as extract_features_long_device.

    Returns (X, window_keys, y, columns).  X and columns are what extract_features(df_shift, column_id="id",
    column_sort="time", column_kind="kind", column_value="value") returns for (df_shift, _) = make_forecasting_frame(...)
    on the equivalent Series: the series is rolled as roll_time_series rolls it, every window loses its last row and the
    windows this empties are dropped.  Row r of X is the window named ("id", window_keys[r]), names ascending;
    window_keys has the index's dtype (int64 row numbers without an index).  y (x's dtype, bit-exact) is the target of
    every row: x at the row that names the window (its last row before the drop for a positive direction, its first row
    for a negative one), what make_forecasting_frame's y holds for that name.  One window has no target: the one named by
    x[0], which make_forecasting_frame's y (x[1:]) leaves out.  With a positive direction and an ascending index it is
    the one-row window that the drop empties; with a negative direction (or an index whose first key is not its smallest)
    it is a row of X, and its y is NaN.  Drop the rows where y is NaN before select_features_device.

    Runs on torch's current stream and blocks the host twice: to stage the rows and to count the windows.  Raises
    roll_time_series's errors for its arguments, and for a series of zero or one rows, before the device is touched, and
    ValueError for NaN values or index keys, two windows with the same name (index keys tied at their naming rows,
    counting the one-row windows that the drop of the last row empties, which the reference merges too) and windows
    longer than the plan allows, before any feature kernel runs.  The plan's length limits apply to the windows, not to
    the series."""
    import torch
    regroup = ("forecast",) + _roll_args(rolling_direction, max_timeshift, min_timeshift)
    for name, t in (("x", x), ("index", index)):
        if t is None and name == "index":
            continue
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor, not %s" % (name, type(t).__name__))
        if t.ndim != 1:
            raise ValueError("%s must be 1-D, got shape %s" % (name, tuple(t.shape)))
    if index is not None and index.shape[0] != x.shape[0]:
        raise ValueError("index has %d entries, x %d" % (index.shape[0], x.shape[0]))
    if x.dtype not in (torch.float32, torch.float64, torch.float16, torch.bfloat16):
        raise TypeError("x must be float32, float64, float16 or bfloat16, not %s" % x.dtype)
    if index is not None and index.dtype not in (torch.int64, torch.float64):
        raise TypeError("index must be int64 or float64, not %s" % index.dtype)
    if x.shape[0] <= 1:
        raise ValueError("Your time series container has zero or one rows!. Can not perform rolling.")
    _check_colname(kind)
    if x.device.type != "cuda":
        raise ValueError("x must be a CUDA tensor, got one on %s" % x.device)
    if index is not None and index.device != x.device:
        raise ValueError("index is on %s, x on %s" % (index.device, x.device))
    X, _, window_keys, columns, targets = _extract_staged(None, x, index, None, [kind], None, regroup,
                                                          default_fc_parameters, kind_to_fc_parameters, impute_function)
    with torch.cuda.device(x.device):
        nan = torch.full((), float("nan"), dtype=x.dtype, device=x.device)
        y = torch.where(targets >= 0, x[targets.clamp(min=0)], nan)
    return X, window_keys, y, columns


def _sub_length(sub_length):
    """add_sub_time_series_index's exception types for a sub_length it cannot package with (TypeError for a non-number,
    ZeroDivisionError for 0, AssertionError for a negative or fractional length); then the length as int"""
    if not isinstance(sub_length, numbers.Real):
        raise TypeError("unsupported operand type(s) for //: 'int' and '%s'" % type(sub_length).__name__)
    if sub_length == 0:
        raise ZeroDivisionError("integer division or modulo by zero")
    if not sub_length > 0 or sub_length != int(sub_length):
        raise AssertionError("sub_length must be a positive integer, got %r" % (sub_length,))
    return min(int(sub_length), (1 << 63) - 1)


def extract_features_sub_device(ids, values, sort=None, kind=None, *, kinds=None, sub_length, times=None,
                                default_fc_parameters=None, kind_to_fc_parameters=None, impute_function=None):
    """Extracts features from fixed-length packages of long-format rows held in CUDA tensors into a CUDA tensor.

    ids, values, sort, kind, kinds, times, default_fc_parameters, kind_to_fc_parameters and impute_function: as
    extract_features_long_device, except that ids may be None: every kind is then one series, as with column_id=None.
    sub_length: as add_sub_time_series_index.

    Returns (X, package_numbers, package_ids, columns), what extract_features returns for add_sub_time_series_index(df,
    sub_length, column_id="id", column_sort="time", column_kind="kind") of the equivalent frame, extracted with
    column_id="id": every (id, kind) series, in sort order, is cut into packages of sub_length rows, the last one
    shorter, and row r of X is the package named (package_numbers[r], package_ids[r]) (both int64; package_ids is None
    without ids), names ascending, package number first.  The rows are the union of the package names over all kinds,
    NaN where a kind has no package of that name.  The quadratic entropies' length limit applies to each package, not to
    the series it comes from.

    Runs on torch's current stream and blocks the host twice: to group the rows and to count the packages.  Raises
    add_sub_time_series_index's exception types for a bad sub_length before the device is touched, and ValueError for
    NaN values or sort keys, kind codes out of range and packages longer than their kind's plan allows, before any
    feature kernel runs."""
    L = _sub_length(sub_length)
    X, package_ids, package_numbers, columns, _ = _extract_staged(ids, values, sort, kind, kinds, times, ("sub", L),
                                                                  default_fc_parameters, kind_to_fc_parameters,
                                                                  impute_function)
    return X, package_numbers, package_ids if ids is not None else None, columns


def _extract_staged(ids, values, sort, kind, kinds, times, regroup, default_fc_parameters, kind_to_fc_parameters,
                    impute_function):
    """(X, row ids, row keys, columns, targets) of long-format rows, staged by kind and extracted.  regroup replaces the
    staged series first: ("roll", direction, max_timeshift, min_timeshift) by their rolled windows (row keys: the
    windows' naming keys), ("forecast", direction, max_timeshift, min_timeshift) by make_forecasting_frame's windows
    (row keys as for "roll"; targets: the target input row of every window, -1: none; ids may be None), ("sub",
    sub_length) by their packages (row keys: the package numbers; ids may be None).  regroup None: the series as
    staged.  Row keys and targets are None where the regrouping has none."""
    import torch
    how = regroup[0] if regroup else None
    windows, forecast = how in ("roll", "forecast"), how == "forecast"
    n, kinds = _long_layout(ids, values, sort, kind, kinds, times, need_ids=how in (None, "roll"))
    if windows and n <= 1:
        raise ValueError("Your time series container has zero or one rows!. Can not perform rolling.")
    default_fc_parameters = _default_settings(default_fc_parameters, kind_to_fc_parameters)
    plans = [_kind_plan(k, default_fc_parameters, kind_to_fc_parameters, has_datetime_index=times is not None)
             for k in kinds]
    dev = values.device
    if dev.type != "cuda":
        raise ValueError("values must be a CUDA tensor, got one on %s" % dev)
    for name, t in (("ids", ids), ("sort", sort), ("kind", kind), ("times", times)):
        if t is not None and t.device != dev:
            raise ValueError("%s is on %s, values on %s" % (name, t.device, dev))
    mode = _lib.IMPUTE_RANGE if impute_function is impute else _lib.IMPUTE_ZERO if impute_function is impute_dataframe_zero else None
    row_keys = targets = None
    with torch.cuda.device(dev):
        v = values.contiguous() if values.dtype == torch.float32 else values.to(torch.float32).contiguous()
        i = torch.zeros(n, dtype=torch.int64, device=dev) if ids is None else ids.contiguous()
        s = None if sort is None else sort.contiguous()
        k = None if kind is None else kind.contiguous()
        t = None if times is None else times.contiguous()
        ctx = get_context(dev.index)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with ctx.lock:
            ctx.set_stream(stream or _lib.STREAM_LEGACY)
            try:
                n_rows, rows, _ = ctx.stage_long_stacked(
                    i.data_ptr(), 0 if s is None else s.data_ptr(), s is not None and s.dtype == torch.float64,
                    v.data_ptr(), 0 if k is None else k.data_ptr(), k is not None and k.dtype == torch.int64, len(kinds),
                    0 if t is None else t.data_ptr(), n, keep_sort_keys=windows, keep_row_numbers=forecast)
                if how is not None:
                    if windows:
                        n_rows, _ = ctx.roll_staged(*regroup[1:], len(kinds), forecast=forecast)
                    else:
                        n_rows, _ = ctx.sub_staged(regroup[1], len(kinds))
                    row_keys = torch.empty(n_rows, dtype=s.dtype if windows and s is not None else torch.int64, device=dev)
                    ctx.staged_row_keys(row_keys.data_ptr())
                if forecast:
                    targets = torch.empty(n_rows, dtype=torch.int64, device=dev)
                    ctx.staged_targets(targets.data_ptr())
                present = [c for c in range(len(kinds)) if rows[c] > 0]
                columns = [name for c in present for name in plans[c][1]]
                width = len(columns)
                X = torch.empty((n_rows, width), dtype=torch.float64, device=dev)
                row_ids = torch.empty(n_rows, dtype=torch.int64, device=dev)
                dps = [_device_plan(ctx, plans[c][0]) if rows[c] > 0 else None for c in range(len(kinds))]
                ctx.extract_staged(dps, row_ids.data_ptr(), X.data_ptr(), width,
                                   _lib.FLAG_IMPUTE if mode == _lib.IMPUTE_RANGE else 0)
                if mode == _lib.IMPUTE_ZERO and n_rows and width:
                    ctx.impute_device(X.data_ptr(), n_rows, width, mode)
            finally:
                ctx.set_stream(None)
    if impute_function is not None and mode is None:
        df = pd.DataFrame(X.cpu().numpy(), columns=columns)
        impute_function(df)
        X.copy_(torch.from_numpy(df.to_numpy(dtype=np.float64)))
    return X, row_ids, row_keys, columns, targets
