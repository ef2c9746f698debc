"""calculate_relevance_table_device / select_features_device on CUDA matrices: the same table, bit for bit, as the
DataFrame path on the same matrix (both run tsfx_select_*, the device path with TSFX_FLAG_DEVICE_PTRS on the tensor
itself), the reference's golden tables, the whole extract -> impute -> select chain on the device, the input layouts,
torch's stream, and the errors."""
import os
import warnings

import numpy as np
import pandas as pd
import pytest

from tsfresh_b200 import (EfficientFCParameters, calculate_relevance_table, calculate_relevance_table_device,
                          extract_features, extract_features_device, impute, select_features, select_features_device)

from tests.test_gpu_selection import CASES, Z

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)
COLUMNS = list(Z["columns"])


def bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64)
    return np.where(np.isnan(a), np.nan, a).view(np.int64)


def assert_same_table(got, want):
    """same columns, index, order, dtypes and values; p-values as float64 bits"""
    pd.testing.assert_frame_equal(got, want)
    for c in got.columns:
        if c.startswith("p_value"):
            assert (bits(got[c].to_numpy(dtype=float)) == bits(want[c].to_numpy(dtype=float))).all(), c


def with_warnings(fn, *args, **kw):
    """fn's result and the warnings of the relevance table (not those of a first library load or scipy import)"""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = fn(*args, **kw)
    return out, [(x.category, str(x.message)) for x in w if os.path.basename(x.filename) == "feature_selection.py"]


def assert_golden(t, key):
    """the reference's table at the tolerances of test_gpu_selection.py"""
    assert list(t.columns) == list(Z[key + "_columns"])
    assert sorted(t.index) == sorted(Z[key + "_index"])
    for c in t.columns:
        got, want = t[c], pd.Series(Z[key + "_col_" + c], index=Z[key + "_index"]).reindex(t.index)
        if c.startswith("p_value"):
            np.testing.assert_allclose(got.to_numpy(dtype=float), want.to_numpy(dtype=float), rtol=1e-9, atol=1e-300,
                                       equal_nan=True)
        elif c.startswith("relevant") or c == "n_significant":
            assert list(got.astype(float)) == list(want.astype(float)), c
        else:
            assert list(got.astype(str)) == list(want.astype(str)), c


@pytest.mark.parametrize("size", ["small", "medium", "large"])
@pytest.mark.parametrize("case", list(CASES))
def test_golden_cases_equal_the_dataframe_path(size, case):
    ycol, kw = CASES[case]
    kw = dict(kw, ml_task="regression" if case in ("yr", "yt") else "classification", show_warnings=True)
    Xh = Z[size + "_X"]
    yh = Z["%s_%s" % (size, ycol)]
    want, want_w = with_warnings(calculate_relevance_table, pd.DataFrame(Xh, columns=COLUMNS), pd.Series(yh), **kw)
    X = torch.from_numpy(Xh).to(DEV)
    for y in (torch.from_numpy(yh).to(DEV), yh, list(yh)):
        got, got_w = with_warnings(calculate_relevance_table_device, X, y, COLUMNS, **kw)
        assert_same_table(got, want)
        assert got_w == want_w
    assert_golden(got, "%s_%s" % (size, case))


@pytest.mark.parametrize("ycol, kw", [("y2", {}), ("y3", {"multiclass": True, "n_significant": 2}), ("yr", {}),
                                      ("yt", {"hypotheses_independent": True})])
def test_selected_matrix(ycol, kw):
    Xh, yh = Z["large_X"], Z["large_" + ycol]
    want = select_features(pd.DataFrame(Xh, columns=COLUMNS), yh, **kw)
    X = torch.from_numpy(Xh).to(DEV)
    X_sel, kept = select_features_device(X, torch.from_numpy(yh).to(DEV), COLUMNS, **kw)
    assert kept == list(want.columns) and len(kept) > 0
    assert X_sel.device == DEV and X_sel.dtype == torch.float64 and X_sel.is_contiguous()
    assert (bits(X_sel) == bits(want.to_numpy())).all()


def test_extract_impute_select_on_the_device():
    N, L = 2048, 256
    rng = np.random.default_rng(21)
    x = rng.standard_normal((N, L)).astype(np.float32)
    x[:, :64] *= rng.uniform(0.5, 2.0, (N, 1)).astype(np.float32)       # a scale the features can see
    x[5, 7] = np.inf                                                     # features to impute
    scale = np.abs(x[:, :64]).mean(axis=1)
    y_class = (scale > np.median(scale)).astype(np.int64)
    y_reg = scale + 0.1 * rng.standard_normal(N)
    s = EfficientFCParameters()
    X, cols = extract_features_device(torch.from_numpy(x).to(DEV), kinds=["value"], default_fc_parameters=s,
                                      impute_function=impute)
    frame = pd.DataFrame({"id": np.repeat(np.arange(N), L), "time": np.tile(np.arange(L), N), "value": x.reshape(-1)})
    Xf = extract_features(frame, column_id="id", column_sort="time", default_fc_parameters=s, impute_function=impute)
    assert cols == list(Xf.columns) and (bits(X) == bits(Xf.to_numpy())).all()
    for y in (y_class, y_reg):
        assert_same_table(calculate_relevance_table_device(X, y, cols), calculate_relevance_table(Xf, pd.Series(y)))
        X_sel, kept = select_features_device(X, torch.from_numpy(y).to(DEV), cols)
        want = select_features(Xf, y)
        assert kept == list(want.columns) and len(kept) > 0
        assert (bits(X_sel) == bits(want.to_numpy())).all()


def test_input_layouts_and_streams():
    rng = np.random.default_rng(22)
    scale = rng.uniform(0.5, 2.0, 600)
    x = torch.from_numpy((rng.standard_normal((600, 128)) * scale[:, None]).astype(np.float32)).to(DEV)
    s = EfficientFCParameters()
    X, cols = extract_features_device(x, default_fc_parameters=s, impute_function=impute)
    y = torch.from_numpy((scale > 1.2).astype(np.int64)).to(DEV)
    want = calculate_relevance_table_device(X, y, cols)
    W = len(cols)
    big = torch.full((600, W + 11), 3.0, dtype=torch.float64, device=DEV)
    sl, _ = extract_features_device(x, default_fc_parameters=s, impute_function=impute, out=big[:, 6:6 + W])
    assert not sl.is_contiguous()
    assert_same_table(calculate_relevance_table_device(sl, y, cols), want)
    assert_same_table(calculate_relevance_table_device(X.t().contiguous().t(), y, cols), want)     # column-major
    # Torch's current stream: on a side stream held busy by a sleep, a torch op is the matrix's last writer and the
    # target is a host array, so nothing synchronises the side stream before the library call.  A selection enqueued
    # on any other stream would read the NaN the matrix holds before the copy and raise, or build another table.
    hy = y.cpu().numpy()
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):
        Xs = torch.full_like(X, float("nan"))
        sel_want = X[:, [cols.index(c) for c in want[want.relevant].feature]]
    torch.cuda.synchronize()
    for call in ("table", "select"):
        with torch.cuda.stream(side):
            Xs.fill_(float("nan"))
            torch.cuda._sleep(200_000_000)
            Xs.copy_(X)
            if call == "table":
                got = calculate_relevance_table_device(Xs, hy, cols)
            else:
                X_sel, kept = select_features_device(Xs, hy, cols)
                host_sel = X_sel.cpu()
        torch.cuda.synchronize()
    assert_same_table(got, want)
    assert kept == list(want[want.relevant].feature) and len(kept) > 0
    assert (bits(host_sel) == bits(sel_want)).all()


def test_errors():
    Xh, yh = Z["medium_X"], Z["medium_y2"]
    X = torch.from_numpy(Xh).to(DEV)
    bad = X.clone()
    bad[17, 5] = float("nan")
    for y in (yh, yh.astype(float)):
        with pytest.raises(ValueError, match="NaN"):
            calculate_relevance_table_device(bad, y, COLUMNS)
    yn = yh.astype(float)
    yn[3] = np.nan
    with pytest.raises(ValueError, match="NaN"):
        calculate_relevance_table_device(X, torch.from_numpy(yn).to(DEV), COLUMNS)
    with pytest.raises(AssertionError, match="more than 1 label/class"):
        select_features_device(X, torch.ones(len(yh), dtype=torch.int64, device=DEV), COLUMNS)
    for fn in (calculate_relevance_table_device, select_features_device):
        with pytest.raises(AssertionError, match="same number of samples"):
            fn(X, yh[:-1], COLUMNS)
        with pytest.raises(ValueError, match="X must be a CUDA tensor"):
            fn(X.cpu(), yh, COLUMNS)
        with pytest.raises(ValueError, match="y is on cuda:0, X on cpu"):
            fn(X.cpu(), torch.from_numpy(yh).to(DEV), COLUMNS)
    # the context is left bound to its own stream and usable
    t = calculate_relevance_table_device(X, yh, COLUMNS)
    assert_same_table(t, calculate_relevance_table(pd.DataFrame(Xh, columns=COLUMNS), pd.Series(yh)))
