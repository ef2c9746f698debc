"""extract_features(): the drop-in host side of the hot path.

Mirrors the reference driver (tsfresh/feature_extraction/extraction.py:30-305) and its input adapters
(tsfresh/feature_extraction/data.py:124-338, 447-500): same signature, same validation errors, same
column names / order / index.  Everything between "a long (id, sort, value) frame" and "the dense
[n_ids x n_features] float64 matrix" happens on the GPU behind the C ABI (include/tsfx.h):
group-by-id + sort-by-time -> CSR (tsfx_extract_long), then the fused per-series kernels.

Differences that are part of the contract (BASELINE.json north_star):
  * values are ingested as float32 (arithmetic is float64); parity with the reference is defined on
    float32-representable inputs;
  * there is no CPU fallback: a calculator or parameter without a GPU implementation raises
    NotImplementedError, a missing library or device raises RuntimeError;
  * n_jobs is the number of GPUs this process may drive (the reference: worker processes, extraction.py:262-283): a
    large frame whose rows arrive ordered by (id, sort) is cut at id boundaries and every GPU fills its rows of ONE
    pinned result matrix; `device=` or a torchrun LOCAL_RANK pins the call to one GPU (one process per GPU, see
    tsfresh_b200.distributed).  chunksize / profile* are accepted for signature compatibility.
"""
import contextlib
import threading
import warnings

import numpy as np
import pandas as pd

from . import _lib
from .plan import Plan
from .settings import ComprehensiveFCParameters

_ctx_lock = threading.Lock()
_contexts = {}

# the reference's default for n_jobs (tsfresh/defaults.py: N_PROCESSES = max(1, cpu_count // 2)); here n_jobs caps the
# number of GPUs one process drives (see extract_features)
import os as _os
N_PROCESSES = max(1, (_os.cpu_count() or 2) // 2)


def get_context(device=None):
    """The process-wide tsfx context for `device` (default: LOCAL_RANK or 0)."""
    import os
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    with _ctx_lock:
        if device not in _contexts:
            _contexts[device] = _lib.Context(device)
        return _contexts[device]


def _device_plan(ctx, plan):
    key = plan.descs.tobytes() + repr(plan.cwt_scales).encode()
    dp = ctx._plans.get(key)
    if dp is None:
        dp = _lib.DevicePlan(ctx, plan)
        ctx._plans[key] = dp
    return dp


def _default_settings(default_fc_parameters, kind_to_fc_parameters):
    """extraction.py:149-152: no settings at all is ComprehensiveFCParameters; per-kind settings alone leave the other
    kinds without features."""
    if default_fc_parameters is None:
        return ComprehensiveFCParameters() if kind_to_fc_parameters is None else {}
    return default_fc_parameters


def _kind_plan(kind, default_fc_parameters, kind_to_fc_parameters, has_datetime_index=False, show_warnings=False):
    """(Plan, column names) of one kind.  The settings are looked up with the RAW kind (extraction.py:333-336), the
    names carry str(kind) (:374-378)."""
    if kind_to_fc_parameters and kind in kind_to_fc_parameters:
        fc = kind_to_fc_parameters[kind]
    else:
        fc = default_fc_parameters
    plan = Plan(fc, has_datetime_index=has_datetime_index)
    if show_warnings:
        for name in plan.skipped:
            warnings.warn("{} requires the data to have a index of type {}. Results will "
                          "not be calculated".format(name, pd.DatetimeIndex))
    return plan, [str(kind) + "__" + sfx for sfx in plan.suffixes]


@contextlib.contextmanager
def _nan_column(label):
    """Turns TSFX_E_NAN (a NaN found by the device's scan of the values) into the reference's error for the column(s)
    `label` (data.py:148-167)."""
    try:
        yield
    except _lib.NanValuesError:
        raise ValueError("Column must not contain NaN values: {}".format(label)) from None


def _impute_on_device(ctx, result):
    """impute(result) (dataframe_functions.py:49-77) by one tsfx_impute pass, as a new frame"""
    if not (result.shape[0] and result.shape[1]):
        return result
    m = np.ascontiguousarray(result.to_numpy(dtype=np.float64))
    ctx.impute(m, _lib.IMPUTE_RANGE)
    return pd.DataFrame(m, index=result.index, columns=result.columns, copy=False)


# ------------------------------------------------------------------ validation (data.py:124-167)
def _check_colname(*columns):
    for col in columns:
        if str(col).endswith("_"):
            raise ValueError("Dict keys are not allowed to end with '_': {}".format(col))
        if "__" in str(col):
            raise ValueError("Dict keys are not allowed to contain '__': {}".format(col))


_HOST_NAN_CHECK_ROWS = 1 << 20      # larger float value columns are scanned on the device instead of by pandas


def _check_nan(df, *columns, on_device=()):
    """data.py:148-167.  Integer / bool columns cannot hold NaN (no pass over the data); float VALUE columns named in
    `on_device` are scanned by the library while they are on the GPU (TSFX_E_NAN -> the same ValueError)."""
    for col in columns:
        if col not in df.columns:
            raise ValueError("Column not found: {}".format(col))
        kind = getattr(df[col].dtype, "kind", "O")
        if kind in "iub":
            continue
        if col in on_device and kind == "f" and len(df) > _HOST_NAN_CHECK_ROWS:
            continue
        if df[col].isnull().any():
            raise ValueError("Column must not contain NaN values: {}".format(col))


def _value_columns(df, *other):
    cols = [c for c in df.columns if c not in other]
    if len(cols) == 0:
        raise ValueError("Could not guess the value column! Please hand it to the function as an argument.")
    return cols


def _sort_keys(col):
    """Sort column -> int64 or float64 keys whose order equals the column's order."""
    if col is None:
        return None
    a = col.to_numpy()
    if a.dtype.kind in "iub":
        return a.astype(np.int64, copy=False)
    if a.dtype.kind == "f":
        return a.astype(np.float64, copy=False)
    if a.dtype.kind in "mM":
        return a.view(np.int64)
    _, inv = np.unique(a, return_inverse=True)      # strings / objects: order-preserving ranks
    return inv.astype(np.int64)


def _frames(container, column_id, column_kind, column_value, column_sort):
    """Normalises the supported input formats (data.py:447-500) to a list of
    (kind, id column, sort keys or None, float32 values, has_datetime_index).  `kind` is the RAW column label / dict
    key / kind value: the reference looks it up in kind_to_fc_parameters as is (extraction.py:333-336) and only
    stringifies it for the feature names (:374-378)."""
    out = []
    if isinstance(container, pd.DataFrame):
        df = container
        if column_id is None:
            raise ValueError("A value for column_id needs to be supplied")
        if column_kind is not None:                                  # long format (data.py:233-291)
            if column_value is None:
                poss = _value_columns(df, column_id, column_sort, column_kind)
                if len(poss) != 1:
                    raise ValueError(
                        "Could not guess the value column, as the number of unused columns os not equal to 1."
                        f"These columns where currently unused: {','.join(poss)}"
                        "Please hand it to the function as an argument.")
                column_value = poss[0]
            _check_nan(df, column_id, column_kind, column_value, on_device=(column_value,))
            if column_sort is not None:
                _check_nan(df, column_sort)
            for kind, sub in df.groupby(column_kind, sort=True):
                out.append((kind, sub[column_id], sub[column_sort] if column_sort is not None else None,
                            sub[column_value], isinstance(sub.index, pd.DatetimeIndex)))
            id_dtype = df[column_id].dtype
        else:                                                        # wide format (data.py:181-230)
            _check_nan(df, column_id)
            value_columns = [column_value] if column_value is not None else _value_columns(df, column_id, column_sort)
            _check_nan(df, *value_columns, on_device=tuple(value_columns))
            _check_colname(*value_columns)
            if column_sort is not None:
                _check_nan(df, column_sort)
            id_col = df[column_id]
            sort_col = df[column_sort] if column_sort is not None else None
            for kind in value_columns:         # the SAME id / sort objects for every kind: extract_features detects the wide format by it
                out.append((kind, id_col, sort_col, df[kind], isinstance(df.index, pd.DatetimeIndex)))
            id_dtype = df[column_id].dtype
    elif isinstance(container, dict):                                # dict of frames (data.py:294-338)
        _check_colname(*list(container.keys()))
        id_dtype = None
        for df in container.values():
            _check_nan(df, column_id, column_value, on_device=(column_value,))
        for kind, df in container.items():
            if column_sort is not None:
                _check_nan(df, column_sort)
            out.append((kind, df[column_id], df[column_sort] if column_sort is not None else None,
                        df[column_value], isinstance(df.index, pd.DatetimeIndex)))
            id_dtype = df[column_id].dtype
    else:
        raise ValueError("df must be a DataFrame or a dict of DataFrames. "
                         "See https://tsfresh.readthedocs.io/en/latest/text/data_formats.html")
    return out, id_dtype


def _encode_ids(id_series_list):
    """ids of all kinds -> int64 codes that sort like the ids, plus the decoder array (or None)."""
    first = id_series_list[0].to_numpy()
    if all(s.to_numpy().dtype.kind in "iu" for s in id_series_list):
        return [s.to_numpy().astype(np.int64, copy=False) for s in id_series_list], None
    allv = np.concatenate([s.to_numpy() for s in id_series_list]) if len(id_series_list) > 1 else first
    uniq, inv = np.unique(allv, return_inverse=True)
    codes, pos = [], 0
    for s in id_series_list:
        codes.append(inv[pos:pos + len(s)].astype(np.int64))
        pos += len(s)
    return codes, uniq


def _gpus_for(n_jobs, device):
    """n_jobs -> devices one process drives (SURVEY 8b): an explicit `device` or a torchrun-style LOCAL_RANK pins the
    call to that GPU (one process per GPU); otherwise min(n_jobs, visible GPUs), at least one (n_jobs = 0, the
    reference's "no parallelisation", is one GPU)."""
    import os
    if device is not None:
        return [int(device)]
    if "LOCAL_RANK" in os.environ:
        return [int(os.environ["LOCAL_RANK"])]
    have = max(1, _lib.device_count())
    return list(range(max(1, min(int(n_jobs) if n_jobs else 1, have))))


def _extract_long_multi(devices, plan, id_codes, sort_keys, v32):
    """One frame over several GPUs of this process (n_jobs > 1): rows ordered by (id, sort key) are cut at id boundaries
    into one contiguous shard per device; every device runs the pipelined long path on its shard from its own thread and
    writes its rows straight into ONE pinned result matrix (no gather, no concatenation: the frame leaves the call as the
    DataFrame's block).  Returns None when the rows are not in that order (the caller falls back to one GPU, which
    sorts on the device)."""
    n = len(id_codes)
    G = len(devices)
    cuts = [0]
    for g in range(1, G):
        r = max(cuts[-1], (n * g) // G)
        while 0 < r < n and id_codes[r] == id_codes[r - 1]:
            r += 1
        cuts.append(r)
    cuts.append(n)
    shards = [(a, b) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]
    if len(shards) < 2:
        return None
    for (a, b), (c, d) in zip(shards[:-1], shards[1:]):            # shard boundaries must separate ascending ids
        if not id_codes[b - 1] < id_codes[c]:
            return None

    def count(ab):
        a, b = ab
        return 1 + int(np.count_nonzero(id_codes[a + 1:b] != id_codes[a:b - 1]))
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(len(shards)) as pool:
        counts = list(pool.map(count, shards))                      # series per shard IF the ids inside it ascend
        total = int(sum(counts))
        ctx0 = get_context(devices[0])
        out = ctx0.pinned_array((total, plan.n_cols), np.float64)
        uid = ctx0.pinned_array((total,), np.int64)
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)

        def run(k):
            a, b = shards[k]
            dp = _device_plan(get_context(devices[k]), plan)
            sk = None if sort_keys is None else sort_keys[a:b]
            got = dp.extract_long_into(id_codes[a:b], sk, v32[a:b], uid[offs[k]:offs[k + 1]], out[offs[k]:offs[k + 1]])
            return got == counts[k]
        ok = list(pool.map(run, range(len(shards))))
    if not all(ok) or not bool(np.all(uid[1:] > uid[:-1])):          # some shard was not in (id, sort) order after all
        return None
    return uid, out


def do_extraction_on_chunks(chunks, default_fc_parameters, kind_to_fc_parameters=None, show_warnings=True, device=None):
    """Batched form of the reference's per-series function (extraction.py:308-386): `chunks` is an iterable of
    (sample_id, kind, data) with `data` a pandas.Series or 1-d array already ordered in time; every chunk of one kind
    goes to the device in ONE launch set.  Returns the flat list of (sample_id, "kind__feature", value) triples in the
    reference's order (chunk by chunk, settings order inside a chunk)."""
    ctx = get_context(device)
    by_kind, order = {}, []
    for pos, (sid, kind, data) in enumerate(chunks):
        idx = getattr(data, "index", None)
        is_dt = isinstance(idx, pd.DatetimeIndex)
        by_kind.setdefault((kind, is_dt), []).append((pos, sid, data))
        order.append(None)
    results = [None] * len(order)
    for (kind, is_dt), items in by_kind.items():
        plan, names = _kind_plan(kind, default_fc_parameters, kind_to_fc_parameters, is_dt, show_warnings)
        if plan.n_cols == 0:
            for pos, sid, _ in items:
                results[pos] = []
            continue
        vals = [np.asarray(d, dtype=np.float32).reshape(-1) for _, _, d in items]
        lens = np.array([len(v) for v in vals], dtype=np.int32)
        if (lens < 1).any():
            raise ValueError("empty time series in chunk")
        begin = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        times = None
        if plan.needs_times:
            times = np.concatenate([d.index.as_unit("ns").asi8 for _, _, d in items])
        with _nan_column(kind):
            mat = _device_plan(ctx, plan).extract_csr(np.concatenate(vals), begin, lens, times=times)
        for r, (pos, sid, _) in enumerate(items):
            results[pos] = [(sid, n, mat[r, c]) for c, n in enumerate(names)]
    return [t for chunk in results for t in chunk]


def _do_extraction_on_chunk(chunk, default_fc_parameters, kind_to_fc_parameters, show_warnings=True):
    """Drop-in for tsfresh.feature_extraction.extraction._do_extraction_on_chunk (extraction.py:308-386), the function
    the dask / spark bindings call per (id, kind) group (convenience/bindings.py:50-54): same arguments, same list of
    (sample_id, "kind__feature", value) triples -- evaluated by the GPU kernels.  One chunk per call wastes the device;
    the bindings' map functions can collect groups and call do_extraction_on_chunks instead."""
    return do_extraction_on_chunks([chunk], default_fc_parameters, kind_to_fc_parameters, show_warnings=show_warnings)


def _extract_rolled(rolled, default_fc_parameters, kind_to_fc_parameters, impute_function, show_warnings, device):
    """extract_features(roll_time_series(...)): every window is a (begin, len) view on the kind's value buffer
    (tsfresh_b200.rolling); same result frame as the reference gives on its materialised rolled frame."""
    from . import dataframe_functions as _dff
    ctx = get_context(device)
    device_impute = impute_function is _dff.impute

    def run(kind, values, begin, length, flags):
        plan, names = _kind_plan(kind, default_fc_parameters, kind_to_fc_parameters)
        if plan.n_cols == 0 or len(begin) == 0:
            return names, np.empty((len(begin), plan.n_cols))
        with _nan_column(kind):           # the reference raises this while adapting the rolled frame
            return names, _device_plan(ctx, plan).extract_csr(values, begin, length, flags=flags)

    if rolled.parts is None:                 # wide frame: every kind shares the windows
        flags = _lib.FLAG_IMPUTE if device_impute else 0          # columns are independent: per-kind impute is exact
        blocks, columns = [], []
        for kind in rolled.kinds:
            names, mat = run(kind, rolled.values[kind], rolled.begin, rolled.length, flags)
            columns += names
            blocks.append(mat)
        data = blocks[0] if len(blocks) == 1 else np.concatenate(blocks, axis=1)
        ids = rolled.ids
        imputed = device_impute
    else:                                    # kind column: every kind has its own windows; rows = union of the window ids
        per = []
        for kind, part in rolled.parts.items():
            if len(part.values) != 1:
                raise ValueError("Could not guess the value column! Please hand it to the function as an argument.")
            names, mat = run(kind, next(iter(part.values.values())), part.begin, part.length, 0)
            per.append((names, part.ids, mat))
        ids = sorted(set().union(*[set(p[1]) for p in per]))
        row = {w: r for r, w in enumerate(ids)}
        columns = [n for p in per for n in p[0]]
        data = np.full((len(ids), len(columns)), np.nan)
        c0 = 0
        for names, wids, mat in per:
            data[[row[w] for w in wids], c0:c0 + len(names)] = mat
            c0 += len(names)
        imputed = False
    index = pd.Index(ids, tupleize_cols=False)
    result = pd.DataFrame(data, index=index, columns=columns, copy=False)
    if impute_function is not None and not imputed:
        if device_impute:
            result = _impute_on_device(ctx, result)
        else:
            impute_function(result)
    return result


def extract_features(timeseries_container, default_fc_parameters=None, kind_to_fc_parameters=None, column_id=None,
                     column_sort=None, column_kind=None, column_value=None, chunksize=None, n_jobs=N_PROCESSES,
                     show_warnings=False, disable_progressbar=False, impute_function=None, profile=False,
                     profiling_filename="profile.txt", profiling_sorting="cumulative", distributor=None, pivot=True,
                     device=None):
    """GPU implementation of tsfresh.extract_features (extraction.py:30-190).  Returns the same
    pandas.DataFrame (float64, index = sorted ids, columns `{kind}__{calculator}[__{params}]`), or the
    list of (id, name, value) triples when pivot=False."""
    default_fc_parameters = _default_settings(default_fc_parameters, kind_to_fc_parameters)
    from .rolling import RolledTimeSeries
    if isinstance(timeseries_container, RolledTimeSeries):
        return _extract_rolled(timeseries_container._for_columns(column_kind, column_value), default_fc_parameters, kind_to_fc_parameters, impute_function,
                               show_warnings, device)
    if distributor is not None:
        from .distributor import is_distributor
        if not is_distributor(distributor):
            raise ValueError("the passed distributor is not an DistributorBaseClass object")

    frames, id_dtype = _frames(timeseries_container, column_id, column_kind, column_value, column_sort)
    gpus = _gpus_for(n_jobs, device)
    ctx = get_context(gpus[0])
    # impute_function=tsfresh_b200.impute: the feature matrix is imputed on the device before it is copied back
    from . import dataframe_functions as _dff
    device_impute = impute_function is _dff.impute
    extract_flags = _lib.FLAG_IMPUTE if (device_impute and len(frames) == 1 and pivot) else 0
    codes, decoder = _encode_ids([f[1] for f in frames])

    blocks = []           # (column names, ids (codes), matrix)
    # wide format (several value columns of ONE frame share the id / sort columns): the kind dimension lives in the device
    # pass -- one stage (a), one result matrix with a column block per kind (tsfx_extract_long_kinds)
    shared = len(frames) > 1 and pivot and all(f[1] is frames[0][1] and f[2] is frames[0][2] for f in frames[1:])
    if shared:
        plans, names = [], []
        for kind, _ids, sort_col, values, has_dt in frames:
            plan, kind_names = _kind_plan(kind, default_fc_parameters, kind_to_fc_parameters, has_dt, show_warnings)
            plans.append(plan)
            names += kind_names
        if len(codes[0]) and all(p.n_cols > 0 for p in plans):
            dps = [_device_plan(ctx, p) for p in plans]
            times = frames[0][3].index.as_unit("ns").asi8 if any(p.needs_times for p in plans) else None
            flags_k = _lib.FLAG_IMPUTE if device_impute else 0
            with _nan_column(", ".join(str(f[3].name) for f in frames)):
                uid, mat = _lib.extract_long_kinds(ctx, dps, codes[0], _sort_keys(frames[0][2]),
                                                   [f[3].to_numpy().astype(np.float32, copy=False) for f in frames], flags=flags_k,
                                                   times=times)
            blocks.append((names, uid, mat))
            frames, codes = [], []
            extract_flags = flags_k
    for (kind, _ids, sort_col, values, has_dt), id_codes in zip(frames, codes):
        plan, names = _kind_plan(kind, default_fc_parameters, kind_to_fc_parameters, has_dt, show_warnings)
        if plan.n_cols == 0 or len(id_codes) == 0:
            uid = np.unique(id_codes)
            blocks.append((names, uid, np.empty((len(uid), 0))))
            continue
        dp = _device_plan(ctx, plan)
        v32 = values.to_numpy().astype(np.float32, copy=False)
        # linear_trend_timewise regresses on the rows' DatetimeIndex (feature_calculators.py:2296-2299)
        times = values.index.as_unit("ns").asi8 if plan.needs_times else None
        with _nan_column(values.name):
            multi = None
            if len(gpus) > 1 and times is None and not extract_flags and len(id_codes) >= (1 << 20):
                multi = _extract_long_multi(gpus, plan, id_codes, _sort_keys(sort_col), v32)
            if multi is not None:
                uid, mat = multi
            else:
                uid, mat = dp.extract_long(id_codes, _sort_keys(sort_col), v32, flags=extract_flags, times=times)
        blocks.append((names, uid, mat))

    # ---- assemble (PartitionedTsData.pivot, data.py:86-121): union of ids, sorted, id dtype restored
    all_ids = blocks[0][1] if len(blocks) == 1 else np.unique(np.concatenate([b[1] for b in blocks]))
    index = all_ids if decoder is None else decoder[all_ids]
    if not pivot:
        triples = []
        for names, uid, mat in blocks:
            ids_out = uid if decoder is None else decoder[uid]
            for r, i in enumerate(ids_out):
                triples.extend((i, n, mat[r, c]) for c, n in enumerate(names))
        return triples
    if len(blocks) == 1:
        data = blocks[0][2]
        columns = blocks[0][0]
    else:
        columns = [n for b in blocks for n in b[0]]
        data = np.full((len(all_ids), len(columns)), np.nan)
        c0 = 0
        for names, uid, mat in blocks:
            rows = np.searchsorted(all_ids, uid)
            data[rows, c0:c0 + len(names)] = mat
            c0 += len(names)
    # the float64 matrix the device wrote becomes the frame's block as is (no copy)
    result = pd.DataFrame(np.asarray(data, dtype=np.float64), index=pd.Index(index), columns=columns, copy=False)
    if id_dtype is not None:
        try:
            result.index = result.index.astype(id_dtype)
        except (TypeError, ValueError):
            pass
    if not result.index.is_monotonic_increasing:
        result = result.sort_index()
    if impute_function is not None:
        if device_impute:
            if not extract_flags:                     # several kinds: one pass over the union
                result = _impute_on_device(ctx, result)
        else:
            impute_function(result)
    return result
