"""Device-side counterparts of the reference's imputation helpers
(tsfresh/utilities/dataframe_functions.py:49-212): same names, arguments, in-place behaviour and errors.

    impute(df)                         +inf -> column max, -inf -> column min, NaN -> column median (finite values);
                                       a column without any finite value is filled with 0
    impute_dataframe_zero(df)          every non-finite value -> 0
    impute_dataframe_range(df, ...)    the same replacement with caller-supplied values
    get_range_values_per_column(df)    (col_to_max, col_to_min, col_to_median)

The matrix goes to the GPU as one row-major float64 block; `extract_features(impute_function=impute)` skips that
round trip and imputes the feature matrix while it is still on the device (TSFX_FLAG_IMPUTE).

    add_sub_time_series_index(df, sub_length, ...)   cuts every series into packages of sub_length rows (:683-784);
                                                     pandas only (extract_features_sub_device does it on the device)
"""
import warnings

import numpy as np
import pandas as pd

from . import _lib


def _matrix(df):
    m = df.to_numpy(dtype=np.float64, copy=True)
    return np.ascontiguousarray(m)


def _write_back(df, m):
    # in place, like the reference (DataFrame.where(..., inplace=True)); all columns end up float64
    for j, c in enumerate(df.columns):
        df[c] = m[:, j]
    return df


def _ctx(device=None):
    from .extraction import get_context
    return get_context(device)


def impute(df_impute, device=None):
    """dataframe_functions.py:49-78."""
    if len(df_impute) == 0:
        return df_impute
    m = _matrix(df_impute)
    stats = _ctx(device).impute(m, _lib.IMPUTE_RANGE)
    _warn_non_finite(df_impute, m, stats)
    return _write_back(df_impute, m)


def impute_dataframe_zero(df_impute, device=None):
    """dataframe_functions.py:81-101."""
    if len(df_impute) == 0:
        return df_impute
    m = _matrix(df_impute)
    _ctx(device).impute(m, _lib.IMPUTE_ZERO)
    return _write_back(df_impute, m)


def impute_dataframe_range(df_impute, col_to_max, col_to_min, col_to_median, device=None):
    """dataframe_functions.py:104-167 (same ValueErrors)."""
    if len(df_impute) == 0:
        return df_impute
    columns = df_impute.columns
    if (not set(columns) <= set(col_to_median.keys()) or not set(columns) <= set(col_to_max.keys())
            or not set(columns) <= set(col_to_min.keys())):
        raise ValueError("Some of the dictionaries col_to_median, col_to_max, col_to_min contains more or less keys "
                         "than the column names in df")
    if (np.any(~np.isfinite(list(col_to_median.values()))) or np.any(~np.isfinite(list(col_to_min.values())))
            or np.any(~np.isfinite(list(col_to_max.values())))):
        raise ValueError("Some of the dictionaries col_to_median, col_to_max, col_to_min contains non finite values "
                         "to replace")
    stats = np.array([[col_to_min[c] for c in columns], [col_to_max[c] for c in columns],
                      [col_to_median[c] for c in columns]], dtype=np.float64)
    m = _matrix(df_impute)
    _ctx(device).impute(m, _lib.IMPUTE_GIVEN, col_stats=stats)
    return _write_back(df_impute, m)


def get_range_values_per_column(df, device=None):
    """dataframe_functions.py:170-212: three dicts column -> finite max / min / median (0 without finite values)."""
    m = _matrix(df)
    stats = _ctx(device).impute(m, _lib.IMPUTE_STATS)
    _warn_non_finite(df, m, stats, check_input=True)
    cols = df.columns
    return dict(zip(cols, stats[1])), dict(zip(cols, stats[0])), dict(zip(cols, stats[2]))


def _warn_non_finite(df, m, stats, check_input=False):
    # the reference warns about columns without any finite value (:194-201); after RANGE they are all-zero and had
    # min = max = median = 0, so look at the statistics (cheap: 3 x cols)
    zero = (stats[0] == 0.0) & (stats[1] == 0.0) & (stats[2] == 0.0)
    if zero.any():
        src = df.to_numpy(dtype=np.float64)[:, zero]
        bad = ~np.isfinite(src).any(axis=0)
        if bad.any():
            warnings.warn("The columns {} did not have any finite values. Filling with zeros.".format(
                df.columns[np.where(zero)[0][bad]].values), RuntimeWarning)


def _check_sub_length(sizes, sub_length):
    """The exceptions add_sub_time_series_index (dataframe_functions.py:683-784) raises for a sub_length that cannot cut
    series of these sizes (in group order): TypeError for a non-number, ZeroDivisionError for 0, ValueError when a
    package count would be negative, AssertionError when the packages would not cover a series exactly."""
    for n in sizes:
        n = int(n)
        q, r = divmod(n, sub_length)
        if r < 0:
            raise ValueError("negative dimensions are not allowed")
        if n and (q < 0 or q * sub_length + r != n or sub_length != int(sub_length)):
            raise AssertionError("packages of %r rows do not cover a series of %d rows" % (sub_length, n))
        if sub_length > 0 and sub_length == int(sub_length):
            return                          # a positive whole length cuts every series


def add_sub_time_series_index(df_or_dict, sub_length, column_id=None, column_sort=None, column_kind=None):
    """dataframe_functions.py:683-784: adds a column "id" that cuts every series into consecutive packages of sub_length
    rows, the last one shorter.

    A series is every (column_id, column_kind) group (groups without a key are dropped), or every column_kind group, or
    the whole frame; its rows are taken in column_sort order, or in frame order without column_sort.  The package number
    of row i of a series is i // sub_length.  "id" holds the package number, or the tuple (package number, column_id
    value) with column_id; an existing "id" column is replaced.  The rows come grouped (groups ascending) with the key
    columns moved behind the others, then sorted by column_sort when it is given; the frame's index labels are kept.
    Unlike the reference, the input frame is never modified.  Rows with equal sort keys keep their frame order.

    A dict of frames (already split by kind) is handled frame by frame; with column_kind it raises ValueError."""
    if isinstance(df_or_dict, dict):
        if column_kind is not None:
            raise ValueError("You passed in a dictionary and gave a column name for the kind. Both are not possible.")
        return {key: add_sub_time_series_index(frame, sub_length, column_id=column_id, column_sort=column_sort)
                for key, frame in df_or_dict.items()}
    df = df_or_dict
    grouper = [c for c in (column_id, column_kind) if c is not None]
    sort = None if column_sort is None else df[column_sort].to_numpy()
    if grouper:
        group = df.groupby(grouper, sort=True).ngroup().to_numpy()
        columns = [c for c in df.columns if c not in grouper] + grouper
    else:
        group = np.zeros(len(df), dtype=np.int64)
        columns = list(df.columns)
    keep = np.flatnonzero(group >= 0)
    if grouper and len(keep) == 0:
        return df[columns[:len(columns) - len(grouper)]].iloc[:0]
    # rows group by group (input order inside a group), then by sort key inside each group
    order = pd.DataFrame({"g": group[keep]} if sort is None else {"g": group[keep], "s": sort[keep]})
    order = keep[order.sort_values(list(order.columns), kind="stable").index.to_numpy()]
    g = group[order]
    starts = np.flatnonzero(np.r_[True, g[1:] != g[:-1]]) if len(g) else np.zeros(0, np.int64)
    _check_sub_length(np.diff(np.r_[starts, len(g)]), sub_length)
    rank = np.arange(len(g)) - np.repeat(starts, np.diff(np.r_[starts, len(g)]))
    package = rank // sub_length
    out = df.iloc[order][columns]
    out["id"] = list(zip(package, out[column_id])) if column_id is not None else package
    if column_sort is not None:
        out = out.sort_values(column_sort)
    return out
