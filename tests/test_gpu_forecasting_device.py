"""extract_features_forecasting_device on one CUDA series: its windows and targets against the reference's answers in
tests/golden/forecasting.npz, its features against the oracle on every window and bit for bit against
extract_features(make_forecasting_frame(...)[0]) on the host path, selection on its (X, y), the length limit per window,
its stream contract and the errors it raises before any kernel group runs."""
import json
import os

import numpy as np
import pandas as pd
import pytest

from oracle import make_golden_forecasting as mk
from oracle.extract import compare, oracle_rows
from tsfresh_b200 import (ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters, extract_features,
                          extract_features_forecasting_device, impute, impute_dataframe_zero, make_forecasting_frame,
                          select_features, select_features_device)
from tsfresh_b200.extraction import get_context
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)
Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "forecasting.npz"))
DOC = json.loads(str(Z["doc"]))


def bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64)
    return np.where(np.isnan(a), np.nan, a).view(np.int64)


def assert_same(got, want):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape
    bad = np.argwhere(g != w)
    assert len(bad) == 0, "%d cells differ, first %s" % (len(bad), bad[:5].tolist())


def device_index(x):
    """(index tensor or None, the index's keys as the device names windows by) for an input of mk.inputs()"""
    if not isinstance(x, pd.Series):
        return None, np.arange(len(x), dtype=np.int64)
    idx = x.index
    keys = idx.as_unit("ns").asi8 if isinstance(idx, pd.DatetimeIndex) else idx.to_numpy()
    return torch.from_numpy(np.array(keys)).to(DEV), keys


def on_device(x, dtype=torch.float64):
    values, _ = mk.values_and_times(x)
    return torch.from_numpy(np.array(values)).to(DEV, dtype)


def test_golden_keys_targets_and_lengths():
    """every grid case: window keys, window lengths (the length column) and y against the reference's"""
    settings = {"length": None}
    for i, (n, d, mx, mn, form, kept) in enumerate(DOC["grid"]):
        x = mk.inputs(n, form)
        values, _ = mk.values_and_times(x)
        index, keys = device_index(x)
        X, wkeys, y, cols = extract_features_forecasting_device(on_device(x), "kk", mx, d, mn, index=index,
                                                                default_fc_parameters=settings)
        assert cols == ["kk__length"]
        w = Z["windows"][Z["window_off"][i]:Z["window_off"][i + 1]]
        y_rows = Z["y_rows"][Z["y_off"][i]:Z["y_off"][i + 1]]
        assert kept or len(w) == 0
        order = np.argsort(keys[w[:, 0]], kind="stable")          # the device's rows ascend by key
        assert wkeys.dtype == (torch.int64 if index is None else index.dtype)
        assert np.array_equal(wkeys.cpu().numpy(), keys[w[order, 0]]), (i, n, d, mx, mn, form)
        assert np.array_equal(X[:, 0].cpu().numpy(), w[order, 2].astype(np.float64)), (i, n, d, mx, mn, form)
        want_y = np.full(len(w), np.nan)
        target = {r: values[r] for r in y_rows}
        want_y[:] = [target.get(r, np.nan) for r in w[order, 0]]
        assert y.dtype == torch.float64
        assert_same(y, want_y)
        assert sorted(set(w[:, 0]) - set(y_rows)) in ([], [0])      # only the window named by x[0] has no target


@pytest.mark.parametrize("direction", [1, 2, 32, -1, -2, -32])
def test_features_against_the_oracle_and_the_host_path(direction):
    rng = np.random.default_rng(100 + direction)
    n = 70
    x = pd.Series(rng.standard_normal(n).astype(np.float32), index=np.arange(n, dtype=np.int64) * 7 - 50)
    settings = EfficientFCParameters()
    for mx, mn in ((None, 0), (12, 0), (500, 0), (12, 8)):
        X, wkeys, y, cols = extract_features_forecasting_device(torch.from_numpy(x.to_numpy()).to(DEV), "s", mx,
                                                                direction, mn, index=torch.from_numpy(x.index.to_numpy()).to(DEV),
                                                                default_fc_parameters=settings)
        df_shift, y_host = make_forecasting_frame(x, "s", mx, direction, mn)
        want = extract_features(df_shift, column_id="id", column_sort="time", column_kind="kind", column_value="value",
                                default_fc_parameters=settings)
        assert cols == list(want.columns)
        assert [("id", k) for k in wkeys.cpu().tolist()] == want.index.tolist()
        assert_same(X, want.to_numpy())
        windows = [x.to_numpy()[b:b + ln] for b, ln in zip(df_shift.begin, df_shift.length)]
        bad = compare(X.cpu().numpy(), oracle_rows([w.astype(np.float64) for w in windows], settings),
                      Plan(settings).suffixes)
        assert not bad, bad[:5]
        got_y = dict(zip(want.index.tolist(), y.cpu().numpy().tolist()))
        assert all(got_y[k] == v for k, v in y_host.items())
        assert y.dtype == torch.float32


@pytest.mark.parametrize("form", ["range", "array", "int_index", "float_index", "unsorted_index", "hourly_index"])
def test_index_forms_and_dtypes(form):
    """index None, int64, float64, unsorted and datetime; float64 x gives y bit-identical to x, float32 x its own
    values; the matrix is the host path's for both call forms of extract_features"""
    x = mk.inputs(64, form)
    index, keys = device_index(x)
    settings = MinimalFCParameters()
    df_shift, y_host = make_forecasting_frame(x, "kk", 10, -2, 1)
    for dtype in (torch.float64, torch.float32):
        X, wkeys, y, cols = extract_features_forecasting_device(on_device(x, dtype), "kk", 10, -2, 1, index=index,
                                                                default_fc_parameters=settings)
        assert y.dtype == dtype
        rows = {k: r for r, k in enumerate(keys.tolist())}
        xv = on_device(x, dtype).cpu()
        src = [rows[k] for k in wkeys.cpu().tolist()]
        assert torch.equal(y[[r != 0 for r in src]].cpu(), xv[[r for r in src if r != 0]])
        assert bool(torch.isnan(y[[r == 0 for r in src]]).all())
    # float64 y against the host function's y, bit for bit
    X, wkeys, y, cols = extract_features_forecasting_device(on_device(x), "kk", 10, -2, 1, index=index,
                                                            default_fc_parameters=settings)
    by_key = dict(zip(wkeys.cpu().tolist(), bits(y).tolist()))
    host_keys = [k[1].value if isinstance(k[1], pd.Timestamp) else k[1] for k in y_host.index]
    assert [by_key[k] for k in host_keys] == bits(y_host.to_numpy()).tolist()
    for column_kind, prefix in (("kind", "kk__"), (None, "value__")):
        want = extract_features(df_shift, column_id="id", column_sort="time", column_kind=column_kind,
                                column_value="value", default_fc_parameters=settings)
        assert [c.replace("kk__", prefix) for c in cols] == list(want.columns)
        assert_same(X, want.to_numpy())


def test_reference_extract_features_answers():
    """extract_features(df_shift, ...) of the reference on its own forecasting frames, both call forms"""
    for key, columns in DOC["extract"].items():
        name, form_of_call = key.split("/")[1:]
        n, form, d, mx, mn = mk.EXTRACT_CASES[name]
        x = mk.float32_values(mk.inputs(n, form))
        df_shift, _ = make_forecasting_frame(x, "kk", mx, d, mn)
        got = extract_features(df_shift, column_id="id", column_sort="time", column_value="value",
                               column_kind="kind" if form_of_call == "kind" else None,
                               default_fc_parameters=EfficientFCParameters())
        assert list(got.columns) == columns
        want = Z[key + "/X"]
        bad = compare(got.to_numpy(), want, [c.split("__", 1)[1] for c in columns])
        assert not bad, bad[:5]
        index, keys = device_index(x)
        X, wkeys, _, cols = extract_features_forecasting_device(on_device(x, torch.float32), "kk", mx, d, mn, index=index,
                                                                default_fc_parameters=EfficientFCParameters())
        assert np.array_equal(wkeys.cpu().numpy(), keys[Z[key + "/rows"]])
        assert_same(X, got.to_numpy())


def test_one_window_and_no_window():
    """n = 2 has one window (of one row) for a positive direction; min_timeshift beyond the series keeps none"""
    x = torch.tensor([3.0, 5.0], dtype=torch.float64, device=DEV)
    X, wkeys, y, cols = extract_features_forecasting_device(x, "v", None, 1, default_fc_parameters={"sum_values": None})
    assert wkeys.tolist() == [1] and X.tolist() == [[3.0]] and y.tolist() == [5.0]
    X, wkeys, y, cols = extract_features_forecasting_device(x, "v", None, -1, default_fc_parameters={"sum_values": None})
    assert wkeys.tolist() == [0] and X.tolist() == [[3.0]] and bool(torch.isnan(y).all())
    X, wkeys, y, cols = extract_features_forecasting_device(x, "v", 3, 1, 5, default_fc_parameters={"sum_values": None})
    assert tuple(X.shape) == (0, 1) and len(wkeys) == 0 and len(y) == 0


def test_selection_matches_the_host():
    rng = np.random.default_rng(7)
    n = 600
    x = np.cumsum(rng.standard_normal(n)) + np.sin(np.arange(n) / 5.0) * 3
    settings = EfficientFCParameters()
    X, wkeys, y, cols = extract_features_forecasting_device(torch.from_numpy(x).to(DEV), "s", 20, 1,
                                                            default_fc_parameters=settings, impute_function=impute)
    keep = ~torch.isnan(y)
    Xs, ys = X[keep], y[keep]
    _, kept = select_features_device(Xs, ys, cols)
    df_shift, y_host = make_forecasting_frame(x, "s", 20, 1)
    F = extract_features(df_shift, column_id="id", column_sort="time", column_kind="kind", column_value="value",
                         default_fc_parameters=settings, impute_function=impute)
    pos = {k: r for r, k in enumerate(F.index.tolist())}
    Fy = F.iloc[[pos[k] for k in y_host.index]]
    assert_same(Fy.to_numpy(), Xs)
    want = select_features(Fy, pd.Series(y_host.to_numpy(), index=Fy.index))
    assert len(want.columns) > 0 and list(kept) == list(want.columns)


def test_length_limit_is_per_window():
    """25 000 samples: past sample_entropy's 21 000-sample limit as one window, not in windows of 256"""
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal(25_000)).to(DEV)
    settings = {"sample_entropy": None, "mean": None}
    ctx = get_context(0)
    with pytest.raises(ValueError, match="exceeds"):
        extract_features_forecasting_device(x, "s", None, 1, default_fc_parameters=settings)
    assert ctx.launch_count() == 0
    X, wkeys, y, _ = extract_features_forecasting_device(x, "s", 255, 1, 24_000, default_fc_parameters=settings)
    assert X.shape[0] == 0
    X, wkeys, y, _ = extract_features_forecasting_device(x, "s", 255, 97, default_fc_parameters=settings)
    ends = wkeys.cpu().numpy()
    xs = x.cpu().numpy()
    want = oracle_rows([xs[max(e - 255, 0):e] for e in ends], settings)
    bad = compare(X.cpu().numpy(), want, Plan(settings).suffixes)
    assert not bad, bad[:5]
    assert torch.equal(y.cpu(), x.cpu()[torch.from_numpy(ends)])


def test_errors_before_any_kernel_group():
    ctx = get_context(0)
    rng = np.random.default_rng(9)
    n = 500
    x = torch.from_numpy(rng.standard_normal(n)).to(DEV)
    index = torch.from_numpy(rng.permutation(n).astype(np.int64) * 3).to(DEV)
    kw = dict(default_fc_parameters=EfficientFCParameters())
    want = extract_features_forecasting_device(x, "s", 30, 3, index=index, **kw)

    def raises(match, xx=x, ii=index, d=3):
        with pytest.raises(ValueError, match=match):
            extract_features_forecasting_device(xx, "s", 30, d, index=ii, **kw)
        assert ctx.launch_count() == 0 and ctx.last_kernels() == []
        got = extract_features_forecasting_device(x, "s", 30, 3, index=index, **kw)
        assert_same(got[0], want[0])
        assert torch.equal(got[1], want[1]) and torch.equal(got[2].isnan(), want[2].isnan())
        assert ctx.launch_count() > 0

    bad = x.clone()
    bad[123] = float("nan")
    raises("value column contains NaN", xx=bad)
    fidx = index.to(torch.float64)
    fidx[17] = float("nan")
    raises("sort keys contain NaN", ii=fidx)
    tied = index.clone()
    tied[index == 9] = 6                         # the windows named by the 3rd and 4th rows in key order: one name
    raises("same name", ii=tied, d=1)
    long_x = torch.from_numpy(rng.standard_normal(21_500)).to(DEV)
    with pytest.raises(ValueError, match="exceeds"):
        extract_features_forecasting_device(long_x, "s", None, 1, default_fc_parameters={"sample_entropy": None})
    assert ctx.launch_count() == 0
    got = extract_features_forecasting_device(x, "s", 30, 3, index=index, **kw)
    assert_same(got[0], want[0])



@pytest.mark.parametrize("keys, direction", [
    ([0, 0, 1, 2, 3, 4], 1),                     # the one-row window of row 0 and the window of row 1: one name
    ([0, 1, 2, 3, 4, 4], -1),                    # the one-row window of the last row and the window before it
    ([0, 1, 2, 2, 3, 4], 1),
    ([0, 1, 2, 2, 3, 4], -1),
    ([0.0, -0.0, 1.0, 2.0, 3.0, 4.0], 1),        # -0.0 and 0.0 are one name, as pandas holds them equal
])
def test_tied_names_with_dropped_windows_are_refused(keys, direction):
    """ties that name two windows of the reference's roll, including the one-row windows that the drop of the last row
    empties: the reference merges them into one series, so both functions refuse them, before any kernel group"""
    ctx = get_context(0)
    x = pd.Series(np.arange(1.0, 7.0), index=keys)
    with pytest.raises(ValueError, match="same name"):
        make_forecasting_frame(x, "k", None, direction)
    index = torch.from_numpy(np.asarray(keys)).to(DEV)              # int64 or float64
    xd = torch.from_numpy(x.to_numpy()).to(DEV)
    with pytest.raises(ValueError, match="same name"):
        extract_features_forecasting_device(xd, "k", None, direction, index=index, default_fc_parameters={"mean": None})
    assert ctx.launch_count() == 0
    X, wkeys, y, _ = extract_features_forecasting_device(xd, "k", None, direction,
                                                         index=torch.arange(6, device=DEV) * 10,
                                                         default_fc_parameters={"mean": None})
    assert X.shape == (5, 1) and ctx.launch_count() > 0
    # with min_timeshift 1 the reference has no one-row windows, so a tie of the first (or last) two rows names one
    # window only
    if keys[0] == keys[1] and direction == 1:
        X, wkeys, y, _ = extract_features_forecasting_device(xd, "k", None, 1, 1, index=index,
                                                             default_fc_parameters={"mean": None})
        df_shift, _ = make_forecasting_frame(x, "k", None, 1, 1)
        assert [("id", k) for k in wkeys.cpu().tolist()] == df_shift.ids


def test_index_on_another_device():
    x = torch.zeros(8, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="^index is on cpu, x on cuda:0$"):
        extract_features_forecasting_device(x, "k", None, 1, index=torch.arange(8))

def test_stream_impute_and_determinism():
    rng = np.random.default_rng(11)
    n = 2_000
    xs = rng.standard_normal(n)
    xs[rng.choice(n, 30, replace=False)] = np.inf
    x = torch.from_numpy(xs).to(DEV)
    settings = EfficientFCParameters()
    for fn in (impute, impute_dataframe_zero):
        X, wkeys, y, cols = extract_features_forecasting_device(x, "s", 64, -4, default_fc_parameters=settings,
                                                                impute_function=fn)
        assert bool(torch.isfinite(X).all())
        df_shift, _ = make_forecasting_frame(xs, "s", 64, -4)
        want = extract_features(df_shift, column_id="id", column_sort="time", column_kind="kind", column_value="value",
                                default_fc_parameters=settings, impute_function=fn)
        assert_same(X, want.to_numpy())
        for _ in range(2):
            again = extract_features_forecasting_device(x, "s", 64, -4, default_fc_parameters=settings, impute_function=fn)
            assert_same(again[0], X)
            assert torch.equal(again[1], wkeys) and torch.equal(again[2].isnan(), y.isnan())
    want = extract_features_forecasting_device(x, "s", 64, -4, default_fc_parameters=settings)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        xx = x * 1.0                             # written by a torch kernel on the side stream right before the call
        X, wkeys, y, _ = extract_features_forecasting_device(xx, "s", 64, -4, default_fc_parameters=settings)
        host = X.cpu(), wkeys.cpu(), y.cpu()
    side.synchronize()
    assert_same(host[0], want[0])
    assert torch.equal(host[1], want[1].cpu()) and np.array_equal(bits(host[2]), bits(want[2]))


def test_comprehensive_matches_the_host_path():
    rng = np.random.default_rng(12)
    x = rng.standard_normal(1_000).astype(np.float32)
    settings = ComprehensiveFCParameters()
    X, _, _, cols = extract_features_forecasting_device(torch.from_numpy(x).to(DEV), "s", 255, 32,
                                                        default_fc_parameters=settings)
    df_shift, _ = make_forecasting_frame(x, "s", 255, 32)
    want = extract_features(df_shift, column_id="id", column_sort="time", column_kind="kind", column_value="value",
                            default_fc_parameters=settings)
    assert cols == list(want.columns)
    assert_same(X, want.to_numpy())
