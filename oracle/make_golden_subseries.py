"""TEST INFRASTRUCTURE (build container only): tests/golden/subseries.npz from the UNMODIFIED reference.

    python -m oracle.make_golden_subseries

tsfresh.utilities.dataframe_functions.add_sub_time_series_index (dataframe_functions.py:683-784) followed by
tsfresh.extract_features(..., column_id="id") on the frames of cases(): the reference's AddSubIdTestCase frames and ragged
multi-kind frames (ids with gaps and negative ids, shuffled rows, int64 and float64 sort keys, no column_id, packages of
1, 7, 256 rows and longer than every series).  Stored per case: the kind names, the result's index (package number,
parent id), its columns and its matrix.  cases() rebuilds the input rows (id, sort key, kind code, float32 value, as the
device API takes them); the GPU tests import it and compare extract_features_sub_device with these answers without
importing the reference.
"""
import json
import os
import warnings

import numpy as np
import pandas as pd

from . import ref_shim

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "tests", "golden")

SMALL = {"value": [1, 2, 3, 4, 5, 6, 7, 8, 9], "id": [1, 1, 1, 1, 2, 2, 2, 2, 2], "kind": [0, 1, 0, 1, 0, 1, 0, 1, 0],
         "sort": [9, 8, 7, 6, 5, 4, 3, 2, 1]}


def ragged(seed, float_keys, shuffle, with_id=True):
    """three kinds of unequal lengths, ids with gaps and negative ids, some (id, kind) series missing.  Sort keys are
    distinct inside a series: inside every (id, kind) one, or, without ids, inside every kind (the reference orders
    equal keys of a series with an unstable sort)"""
    rng = np.random.default_rng(seed)
    spec = {0: {-9: 600, -2: 41, 5: 257, 40: 3}, 1: {-9: 13, 0: 300, 40: 256}, 2: {-2: 1, 5: 99, 40: 777, 1 << 40: 20}}
    cols = {"id": [], "sort": [], "kind": [], "value": []}
    for code, series in spec.items():
        for j, (i, n) in enumerate(series.items()):
            cols["id"].append(np.full(n, i, np.int64))
            keys = np.arange(n, dtype=np.int64) * 3 - 50 + (0 if with_id else 10_000 * j)
            cols["sort"].append(keys * 0.5 - 0.25 if float_keys else keys)
            cols["kind"].append(np.full(n, code, np.int64))
            cols["value"].append(rng.standard_normal(n).astype(np.float32))
    rows = {c: np.concatenate(v) for c, v in cols.items()}
    if shuffle:
        p = rng.permutation(len(rows["id"]))
        rows = {c: v[p] for c, v in rows.items()}
    return rows


def small(with_kind, with_sort):
    rows = {"id": np.asarray(SMALL["id"], np.int64), "value": np.asarray(SMALL["value"], np.float32),
            "kind": np.asarray(SMALL["kind"] if with_kind else [0] * 9, np.int64)}
    rows["sort"] = np.asarray(SMALL["sort"], np.int64) if with_sort else None
    return rows


def _efficient():
    from tsfresh.feature_extraction import EfficientFCParameters
    return EfficientFCParameters()


def _comprehensive():
    from tsfresh.feature_extraction import ComprehensiveFCParameters
    return ComprehensiveFCParameters()


def _minimal():
    from tsfresh.feature_extraction import MinimalFCParameters
    return MinimalFCParameters()


# name -> (rows, kind names, sub_length, column_id given, settings, dict input)
def cases():
    return {
        # AddSubIdTestCase (tests/units/utilities/test_dataframe_functions.py:1531-1614)
        "no_parameters": (small(False, False), ["value"], 2, False, _comprehensive, False),
        "id_parameters": (small(False, False), ["value"], 2, True, _comprehensive, False),
        "kind_parameters": (small(True, False), ["0", "1"], 2, True, _comprehensive, False),
        "sort_parameters": (small(True, True), ["0", "1"], 2, True, _comprehensive, False),
        "dict_input": (small(False, False), ["1"], 2, True, _comprehensive, True),
        # ragged multi-kind frames
        "ragged_7": (ragged(1, False, False), ["a", "b", "c"], 7, True, _minimal, False),
        "ragged_256_shuffled": (ragged(2, False, True), ["a", "b", "c"], 256, True, _comprehensive, False),
        "ragged_256_float_keys": (ragged(3, True, True), ["a", "b", "c"], 256, True, _comprehensive, False),
        "ragged_1": (ragged(4, False, True), ["a", "b", "c"], 1, True, _minimal, False),
        "ragged_longer": (ragged(5, True, True), ["a", "b", "c"], 1000, True, _efficient, False),
        "ragged_no_id_7": (ragged(6, False, True, with_id=False), ["a", "b", "c"], 7, False, _minimal, False),
        "ragged_no_id_256": (ragged(7, True, True, with_id=False), ["a", "b", "c"], 256, False, _comprehensive, False),
    }


def frame(rows, kinds, with_id):
    """the frame the reference sees: column "id" only with column_id (so that add_sub_time_series_index adds it)"""
    df = pd.DataFrame({"value": rows["value"].astype(np.float64)})
    if with_id:
        df["ID"] = rows["id"]
    if len(kinds) > 1:
        df["kind"] = np.asarray(kinds, dtype=object)[rows["kind"]]
    if rows["sort"] is not None:
        df["sort"] = rows["sort"]
    return df


def reference(rows, kinds, sub_length, with_id, settings, as_dict):
    ref_shim.load()
    from tsfresh import extract_features
    from tsfresh.utilities.dataframe_functions import add_sub_time_series_index
    df = frame(rows, kinds, with_id)
    sort = "sort" if rows["sort"] is not None else None
    kind = "kind" if len(kinds) > 1 else None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if as_dict:
            data = add_sub_time_series_index({kinds[0]: df}, sub_length, column_id="ID" if with_id else None,
                                             column_sort=sort)
            if with_id:
                data = {k: v.drop(columns="ID") for k, v in data.items()}
            X = extract_features(data, column_id="id", column_sort=sort, column_value="value",
                                 default_fc_parameters=settings(), n_jobs=0, disable_progressbar=True)
        else:
            data = add_sub_time_series_index(df, sub_length, column_id="ID" if with_id else None, column_sort=sort,
                                             column_kind=kind)
            if with_id:
                data = data.drop(columns="ID")
            X = extract_features(data, column_id="id", column_sort=sort, column_kind=kind,
                                 default_fc_parameters=settings(), n_jobs=0, disable_progressbar=True)
    index = X.index.tolist()
    package = np.asarray([i[0] if with_id else i for i in index], np.int64)
    parent = np.asarray([i[1] for i in index], np.int64) if with_id else np.zeros(0, np.int64)
    return package, parent, list(X.columns), X.to_numpy(dtype=np.float64)


def main():
    out, doc = {}, {}
    for name, (rows, kinds, sub_length, with_id, settings, as_dict) in cases().items():
        package, parent, columns, X = reference(rows, kinds, sub_length, with_id, settings, as_dict)
        out["%s/package" % name] = package
        out["%s/parent" % name] = parent
        out["%s/X" % name] = X
        doc[name] = {"kinds": kinds, "sub_length": sub_length, "with_id": with_id, "settings": settings.__name__[1:],
                     "columns": columns}
        print(name, X.shape)
    out["doc"] = np.asarray(json.dumps(doc))
    np.savez_compressed(os.path.join(OUT, "subseries.npz"), **out)


if __name__ == "__main__":
    main()
