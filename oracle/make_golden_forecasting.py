"""TEST INFRASTRUCTURE (build container only): tests/golden/forecasting.npz from the UNMODIFIED reference.

    python -m oracle.make_golden_forecasting

tsfresh.utilities.dataframe_functions.make_forecasting_frame (dataframe_functions.py:606-680) on the grid of grid():
n in {2, 3, 5, 17, 64}, rolling_direction in {1, 2, 3, -1, -2, -5}, max_timeshift in {None, 1, 3, 10, 100},
min_timeshift in {0, 1, 4}, x as a range, a numpy array and a pd.Series with an int, float, unsorted and hourly
DatetimeIndex (inputs() rebuilds them).  Every window of the reference's df_shift is a run of consecutive rows of x in
time order, which is checked here, so a case is stored as its windows (input row that names the window, first position
in time order, number of rows, in df_shift's row order) and its y (input row of every entry, in y's order; the values
are x's at those rows).  A case for which the reference keeps no window (it raises KeyError then) has no windows
and is flagged in the doc.
Also stored: the reference's own test_make_forecasting_frame_* answers (tests/units/utilities/test_dataframe_functions.py:
1366-1507) and extract_features on a few forecasting frames, with and without column_kind.
"""
import json
import os
import warnings

import numpy as np
import pandas as pd

from . import ref_shim

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden")

NS = (2, 3, 5, 17, 64)
DIRECTIONS = (1, 2, 3, -1, -2, -5)
MAX_TIMESHIFTS = (None, 1, 3, 10, 100)
MIN_TIMESHIFTS = (0, 1, 4)
FORMS = ("range", "array", "int_index", "float_index", "unsorted_index", "hourly_index")


def inputs(n, form):
    """x of the given form: a range, or n standard-normal float64 values as an array or a Series"""
    if form == "range":
        return range(n)
    rng = np.random.default_rng(1000 * n + FORMS.index(form))
    v = rng.standard_normal(n)
    if form == "array":
        return v
    index = {"int_index": lambda: np.arange(n, dtype=np.int64) * 3 - 7,
             "float_index": lambda: np.arange(n) * 0.75 - 2.5,
             "unsorted_index": lambda: rng.permutation(n).astype(np.int64) * 2 + 1,
             "hourly_index": lambda: pd.date_range("2011-01-01", periods=n, freq="h")}[form]()
    return pd.Series(v, index=index)


def values_and_times(x):
    """(values as float64, time of every input row as in the reference's frame: the Series' index or 0 .. n-1)"""
    if isinstance(x, pd.Series):
        return x.to_numpy(dtype=np.float64), x.index
    return np.asarray(list(x), dtype=np.float64), pd.RangeIndex(len(x))


def float32_values(x):
    """the Series x with its values rounded to float32 (kept as float64): the features' input on the device"""
    return pd.Series(x.to_numpy().astype(np.float32).astype(np.float64), index=x.index)


def grid():
    return [(n, d, mx, mn, form) for n in NS for d in DIRECTIONS for mx in MAX_TIMESHIFTS for mn in MIN_TIMESHIFTS
            for form in FORMS]


REFERENCE_TESTS = {
    # name -> (x, kind, max_timeshift, rolling_direction, min_timeshift)
    "test_make_forecasting_frame_list": (lambda: range(4), "test", 1, 1, 0),
    "test_make_forecasting_frame_range": (lambda: np.arange(4), "test", 1, 1, 0),
    "test_make_forecasting_frame_pdSeries": (
        lambda: pd.Series(data=range(4), index=pd.date_range("1/1/2011", periods=4, freq="h")), "test", 1, 1, 0),
    "test_make_forecasting_frame_min_timeshift_default": (lambda: pd.Series([1, 2, 3, 4, 5]), "test", 3, 1, 0),
    "test_make_forecasting_frame_min_timeshift": (lambda: pd.Series([1, 2, 3, 4, 5]), "test", 3, 1, 2),
}

# extract_features(df_shift, ...) of these forecasting frames, values rounded to float32: (n, form, direction,
# max_timeshift, min_timeshift)
EXTRACT_CASES = {
    "hourly_pos": (64, "hourly_index", 2, 10, 0),
    "unsorted_neg": (64, "unsorted_index", -1, 5, 1),
    "float_none": (17, "float_index", 1, None, 0),
}


def reference(x, kind, max_timeshift, rolling_direction, min_timeshift):
    ref_shim.load()
    from tsfresh.utilities.dataframe_functions import make_forecasting_frame
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return make_forecasting_frame(x, kind, max_timeshift, rolling_direction, min_timeshift)
        except KeyError:                         # no window is kept: roll_time_series sorts an empty concatenation
            return None


def windows_of(df_shift, y, x):
    """(name row, first time position, rows) of every window in df_shift's order, and the input row of every y entry"""
    values, times = values_and_times(x)
    order = np.argsort(np.asarray(times), kind="stable")
    pos_of_row = np.empty(len(order), np.int64)
    pos_of_row[order] = np.arange(len(order))
    row_of_time = {t: r for r, t in enumerate(times)}
    assert len(row_of_time) == len(times)
    df = df_shift.reset_index(drop=True)
    names = [row_of_time[i[1]] for i in df["id"]]
    rows = [row_of_time[t] for t in df["time"]]
    assert np.array_equal(df["value"].to_numpy(dtype=np.float64), values[rows])
    wins = []
    for k, (name, row) in enumerate(zip(names, rows)):
        if k > 0 and names[k - 1] == name:
            assert pos_of_row[row] == wins[-1][1] + wins[-1][2]
            wins[-1][2] += 1
        else:
            assert all(w[0] != name for w in wins)
            wins.append([name, pos_of_row[row], 1])
    y_rows = [row_of_time[i[1]] for i in y.index]
    assert np.array_equal(y.to_numpy(dtype=np.float64), values[y_rows]) and y.name == "value"
    return np.asarray(wins, np.int32).reshape(-1, 3), np.asarray(y_rows, np.int32)


def main():
    out, doc = {}, {"grid": [], "reference_tests": {}, "extract": {}}
    wins, ys, woff, yoff = [], [], [0], [0]
    for n, d, mx, mn, form in grid():
        x = inputs(n, form)
        r = reference(x, "kk", mx, d, mn)
        if r is None:
            w, yr = np.zeros((0, 3), np.int32), np.zeros(0, np.int32)
        else:
            w, yr = windows_of(*r, x)
        doc["grid"].append([n, d, mx, mn, form, r is not None])
        wins.append(w)
        ys.append(yr)
        woff.append(woff[-1] + len(w))
        yoff.append(yoff[-1] + len(yr))
    out["windows"] = np.concatenate(wins)
    out["window_off"] = np.asarray(woff, np.int64)
    out["y_rows"] = np.concatenate(ys)
    out["y_off"] = np.asarray(yoff, np.int64)
    for name, (make, kind, mx, d, mn) in REFERENCE_TESTS.items():
        x = make()
        w, yr = windows_of(*reference(x, kind, mx, d, mn), x)
        out["ref/%s/windows" % name] = w
        out["ref/%s/y_rows" % name] = yr
        doc["reference_tests"][name] = [kind, mx, d, mn]
    from tsfresh import extract_features
    from tsfresh.feature_extraction import EfficientFCParameters
    for name, (n, form, d, mx, mn) in EXTRACT_CASES.items():
        df_shift, _ = reference(float32_values(inputs(n, form)), "kk", mx, d, mn)
        for with_kind in (False, True):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                X = extract_features(df_shift, column_id="id", column_sort="time", column_value="value",
                                     column_kind="kind" if with_kind else None,
                                     default_fc_parameters=EfficientFCParameters(), n_jobs=0, disable_progressbar=True)
            _, times = values_and_times(inputs(n, form))
            row_of_time = {t: r for r, t in enumerate(times)}
            key = "extract/%s/%s" % (name, "kind" if with_kind else "value")
            out[key + "/X"] = X.to_numpy(dtype=np.float64)
            out[key + "/rows"] = np.asarray([row_of_time[i[1]] for i in X.index], np.int32)
            doc["extract"][key] = list(X.columns)
    out["doc"] = np.asarray(json.dumps(doc))
    np.savez_compressed(os.path.join(OUT, "forecasting.npz"), **out)
    print(len(doc["grid"]), "cases,", len(out["windows"]), "windows,", len(out["y_rows"]), "targets")


if __name__ == "__main__":
    main()
