"""roll_time_series as window VIEWS (SURVEY section 8f row 1; BASELINE.json configs[4]).

The reference (tsfresh/utilities/dataframe_functions.py:376-603) materialises every window as copied rows
(`groupby.apply` per shift, :340-373) -- an 8x data blow-up at window 256 / stride 32.  Here the frame is brought into
series order once and every window becomes a `(begin, len)` view on that one value buffer (`tsfx_roll_windows`,
include/tsfx.h); the result is a `RolledTimeSeries` that `tsfresh_b200.extract_features` consumes directly:

    rolled = roll_time_series(df, column_id="id", column_sort="time", rolling_direction=32, max_timeshift=255,
                              min_timeshift=255)
    X = extract_features(rolled, default_fc_parameters=...)        # index: (id, time of the window's id row)

Same arguments, validation errors and window ids as the reference; `chunksize / n_jobs / distributor / progress bar`
are accepted for signature compatibility only.  `rolled.to_frame()` materialises the reference's DataFrame
(testing / interchange; not used by the extraction path).

make_forecasting_frame (dataframe_functions.py:606-680) rolls one series the same way and shortens every window by its
last row; its df_shift is a ForecastingFrame of such views, and extract_features reads it as the reference reads its
frame with column_id="id", column_sort="time" and column_value="value" (and column_kind="kind").
"""
import warnings

import numpy as np
import pandas as pd

from . import _lib


class RolledTimeSeries:
    """Windows of one frame: `values[kind]` float32 in (id, sort) order, `begin/length` per window, `ids` = list of
    `(original id, sort value of the row that names the window)` in the order the reference's result is sorted."""

    def __init__(self, values, begin, length, ids, parent, id_row, sort_values, column_sort, parts=None,
                 column_kind=None):
        self.parts = parts                # long format with a kind column: kind -> RolledTimeSeries of that kind's rows
        self.column_kind = column_kind
        self.values = values              # dict kind -> float32 array
        self.begin = begin
        self.length = length
        self.ids = ids
        self.parent = parent              # index of the original series of every window
        self.id_row = id_row              # row (inside the original series) whose sort value names the window
        self.sort_values = sort_values    # sort column in series order (None: row numbers)
        self.column_sort = column_sort

    def __len__(self):
        return len(self.begin) if self.parts is None else sum(len(p) for p in self.parts.values())

    @property
    def kinds(self):
        return list(self.values.keys()) if self.parts is None else list(self.parts.keys())

    def to_frame(self):
        """The reference's rolled DataFrame (rows copied once per window): columns id, sort column, one per kind."""
        if self.parts is not None:
            frames = []
            for kind, part in self.parts.items():
                f = part.to_frame()
                f[self.column_kind] = kind
                frames.append(f)
            out = pd.concat(frames, ignore_index=True)
            # the reference concatenates its per-shift chunks and sorts by (id, sort) with a stable multi-key sort
            return out.sort_values(by=["id", self.column_sort or "sort"], kind="stable").reset_index(drop=True)
        rows = np.concatenate([np.arange(b, b + n) for b, n in zip(self.begin, self.length)]) if len(self) else np.zeros(0, np.int64)
        out = {"id": np.repeat(np.arange(len(self)), self.length)}
        ids = np.empty(len(self), dtype=object)
        ids[:] = self.ids
        out["id"] = ids[out["id"]]
        sort_name = self.column_sort or "sort"
        out[sort_name] = self.sort_values[rows] if self.sort_values is not None else rows
        for k, v in self.values.items():
            out[k] = v[rows]
        return pd.DataFrame(out)

    def _for_columns(self, column_kind, column_value):
        """the windows as extract_features(self, column_kind=..., column_value=...) reads them: a rolled frame names its
        kinds itself"""
        return self


class ForecastingFrame(RolledTimeSeries):
    """make_forecasting_frame's df_shift: windows of one series without their last rows, as views on its values (x's
    dtype, time order); to_frame() gives the reference's columns time, value, kind and id, in its order."""

    def __init__(self, values, begin, length, ids, parent, id_row, sort_values, kind):
        super().__init__({"value": values}, begin, length, ids, parent, id_row, sort_values, "time")
        self.kind = kind

    def to_frame(self):
        out = super().to_frame()
        out["kind"] = [self.kind] * len(out)
        return out[["time", "value", "kind", "id"]]

    def _for_columns(self, column_kind, column_value):
        # the frame's value column is "value"; with column_kind its one kind is named by the kind column
        name = str(self.kind) if column_kind is not None else "value"
        return RolledTimeSeries({name: self.values["value"]}, self.begin, self.length, self.ids, self.parent, self.id_row,
                                self.sort_values, self.column_sort)


def make_forecasting_frame(x, kind, max_timeshift, rolling_direction, min_timeshift=0):
    """dataframe_functions.py:606-680: (df_shift, y) for one series x (list, numpy array or pd.Series, whose index is
    then the time).  df_shift holds roll_time_series's windows of x, each without its last row and the windows this
    empties left out, as a ForecastingFrame; y (named "value", x's dtype) is x[1:] indexed by ("id", time), restricted
    to the names of the windows, in x's order.  Raises ValueError when two windows have the same name (the index ties at
    the rows that name them), which the reference merges into one series."""
    n = len(x)
    t = x.index if isinstance(x, pd.Series) else range(n)
    df = pd.DataFrame({"id": ["id"] * n, "time": t, "value": x, "kind": kind})
    if rolling_direction == 0:
        raise ValueError("Rolling direction of 0 is not possible")
    if max_timeshift is not None and max_timeshift <= 0:
        raise ValueError("max_timeshift needs to be positive!")
    if min_timeshift < 0:
        raise ValueError("min_timeshift needs to be positive or zero!")
    if n <= 1:
        raise ValueError("Your time series container has zero or one rows!. Can not perform rolling.")
    if df["time"].isnull().any():
        raise ValueError("You have NaN values in your sort column.")
    order = np.argsort(df["time"].to_numpy(), kind="stable")       # the series order _roll_frame would choose
    rolled = _roll_frame(df[["id", "time", "value"]].iloc[order], "id", "time", rolling_direction, max_timeshift,
                         min_timeshift, False, None)
    if len(set(rolled.ids)) != len(rolled.ids):
        # the reference merges windows of one name into one series before it drops a row of it: not a view
        raise ValueError("two windows have the same name (id, time): the index ties at the rows that name them")
    keep = np.flatnonzero(rolled.length >= 2)                       # a window of one row is empty without its last row
    ids = [rolled.ids[i] for i in keep]
    df_shift = ForecastingFrame(df["value"].to_numpy()[order], rolled.begin[keep], rolled.length[keep] - 1, ids,
                                rolled.parent[keep], rolled.id_row[keep], rolled.sort_values, kind)
    y = df["value"][1:]
    y.index = map(lambda v: ("id", v), y.index)
    return df_shift, y[y.index.isin(set(ids))]


def roll_time_series(df_or_dict, column_id, column_sort=None, column_kind=None, rolling_direction=1, max_timeshift=None,
                     min_timeshift=0, chunksize=None, n_jobs=0, show_warnings=False, disable_progressbar=True,
                     distributor=None):
    """dataframe_functions.py:376-603 with window views instead of copied rows."""
    if rolling_direction == 0:
        raise ValueError("Rolling direction of 0 is not possible")
    if max_timeshift is not None and max_timeshift <= 0:
        raise ValueError("max_timeshift needs to be positive!")
    if min_timeshift < 0:
        raise ValueError("min_timeshift needs to be positive or zero!")
    if isinstance(df_or_dict, dict):
        if column_kind is not None:
            raise ValueError("You passed in a dictionary and gave a column name for the kind. Both are not possible.")
        return {key: roll_time_series(df_or_dict[key], column_id, column_sort, column_kind, rolling_direction,
                                      max_timeshift, min_timeshift) for key in df_or_dict}
    df = df_or_dict
    if len(df) <= 1:
        raise ValueError("Your time series container has zero or one rows!. Can not perform rolling.")
    if column_id is None:
        raise ValueError("You have to set the column_id which contains the ids of the different time series")
    if column_id not in df:
        raise AttributeError("The given column for the id is not present in the data.")
    if column_sort is not None and df[column_sort].isnull().any():
        raise ValueError("You have NaN values in your sort column.")
    if column_kind is not None:
        # long format with a kind column (:518-523): every (kind, id) group is rolled on its own, the shifts are
        # anchored to the longest group of the whole frame
        longest = int(df.groupby([column_kind, column_id]).size().max())
        parts = {}
        for kind, sub in df.groupby(column_kind, sort=True):
            parts[str(kind)] = _roll_frame(sub.drop(columns=[column_kind]), column_id, column_sort, rolling_direction,
                                           max_timeshift, min_timeshift, show_warnings, longest)
        return RolledTimeSeries(None, None, None, None, None, None, None, column_sort, parts=parts, column_kind=column_kind)
    return _roll_frame(df, column_id, column_sort, rolling_direction, max_timeshift, min_timeshift, show_warnings, None)


def _roll_frame(df, column_id, column_sort, rolling_direction, max_timeshift, min_timeshift, show_warnings, longest):

    # series order: stable sort by (id, sort) -- skipped when the frame already is in that order
    ids_col = df[column_id].to_numpy()
    keys = [column_id] if column_sort is None else [column_id, column_sort]
    order = None
    id_codes, uniq_first = pd.factorize(ids_col, sort=True)
    sort_col = df[column_sort].to_numpy() if column_sort is not None else None
    in_order = bool(np.all(id_codes[1:] >= id_codes[:-1]))
    if in_order and sort_col is not None:
        same = id_codes[1:] == id_codes[:-1]
        in_order = bool(np.all(~same | (sort_col[1:] >= sort_col[:-1])))
    if not in_order:
        order = np.lexsort((sort_col, id_codes)) if sort_col is not None else np.argsort(id_codes, kind="stable")
        id_codes = id_codes[order]
        if sort_col is not None:
            sort_col = sort_col[order]
    uid = np.asarray(uniq_first)
    lens = np.bincount(id_codes, minlength=len(uid)).astype(np.int32)
    begin = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    if show_warnings and sort_col is not None and sort_col.dtype != object and len(sort_col) > 1:
        d = np.diff(sort_col)[id_codes[1:] == id_codes[:-1]]
        if len(d) and d.min() != d.max():
            warnings.warn("Your time stamps are not uniformly sampled, which makes rolling nonsensical in some domains.")
    own_longest = int(lens.max())
    longest = own_longest if longest is None else int(longest)
    mx = int(max_timeshift) if max_timeshift else longest                 # `max_timeshift or prediction_steps` (:552)
    if longest > own_longest:
        # the shifts are anchored to the longest group of the WHOLE frame: a phantom series of that length (its
        # windows are dropped again) makes tsfx_roll_windows use it
        wb, wl, wp, we = _lib.roll_windows(np.append(begin, 0), np.append(lens, np.int32(longest)), int(rolling_direction),
                                           mx, int(min_timeshift))
        keep = wp < len(lens)
        wb, wl, wp, we = wb[keep], wl[keep], wp[keep], we[keep]
    else:
        wb, wl, wp, we = _lib.roll_windows(begin, lens, int(rolling_direction), mx, int(min_timeshift))

    value_cols = [c for c in df.columns if c not in keys]
    values = {}
    for c in value_cols:
        v = df[c].to_numpy()
        values[str(c)] = np.ascontiguousarray(v if order is None else v[order], dtype=np.float32)
    row_of_id = begin[wp] + we
    # window names keep their pandas scalar types (Timestamp / Timedelta for datetime-like sort columns, as the
    # reference's (id, timestamp) tuples do, dataframe_functions.py:365-366); plain numbers go through tolist()
    if sort_col is None:
        names = np.asarray(we).tolist()
    elif sort_col.dtype.kind in "mM":
        names = list(pd.Index(sort_col[row_of_id]))
    else:
        names = np.asarray(sort_col[row_of_id]).tolist()
    ids = list(zip(uid[wp].tolist(), names))
    return RolledTimeSeries(values, wb, wl, ids, wp, we, sort_col, column_sort)
