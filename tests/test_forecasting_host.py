"""make_forecasting_frame against the reference's answers in tests/golden/forecasting.npz (oracle/make_golden_forecasting.py),
its argument errors, and the argument checks of extract_features_forecasting_device that need no device."""
import json
import os

import numpy as np
import pandas as pd
import pytest

from oracle import make_golden_forecasting as mk
from tsfresh_b200 import ForecastingFrame, extract_features_forecasting_device, make_forecasting_frame

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "forecasting.npz"))
DOC = json.loads(str(Z["doc"]))


def golden_case(i):
    w = Z["windows"][Z["window_off"][i]:Z["window_off"][i + 1]]
    return w, Z["y_rows"][Z["y_off"][i]:Z["y_off"][i + 1]]


def check_against(x, kind, mx, d, mn, windows, y_rows):
    df_shift, y = make_forecasting_frame(x, kind, mx, d, mn)
    assert isinstance(df_shift, ForecastingFrame)
    frame = df_shift.to_frame()
    assert list(frame.columns) == ["time", "value", "kind", "id"]
    assert (frame["kind"] == kind).all()
    values, _ = mk.values_and_times(x)
    # the value column and y keep x's dtype
    assert frame["value"].dtype == y.dtype == pd.DataFrame({"value": x})["value"].dtype
    got_w, got_y = mk.windows_of(frame, y, x)
    assert np.array_equal(got_w, windows)
    assert np.array_equal(got_y, y_rows)
    return frame, y


@pytest.mark.parametrize("n", mk.NS)
def test_grid_against_the_reference(n):
    cases = [(i, c) for i, c in enumerate(DOC["grid"]) if c[0] == n]
    assert len(cases) == len(mk.DIRECTIONS) * len(mk.MAX_TIMESHIFTS) * len(mk.MIN_TIMESHIFTS) * len(mk.FORMS)
    for i, (_, d, mx, mn, form, kept) in cases:
        windows, y_rows = golden_case(i)
        x = mk.inputs(n, form)
        if not kept:
            # the reference raises KeyError when no window is kept; here the frame and y are empty, as
            # roll_time_series's result is then
            df_shift, y = make_forecasting_frame(x, "kk", mx, d, mn)
            assert len(df_shift) == 0 and len(df_shift.to_frame()) == 0 and len(y) == 0
            continue
        check_against(x, "kk", mx, d, mn, windows, y_rows)


def test_reference_test_cases():
    """the answers of the reference's MakeForecastingFrameTestCase, and its stated frames and targets"""
    for name, (kind, mx, d, mn) in DOC["reference_tests"].items():
        x = mk.REFERENCE_TESTS[name][0]()
        check_against(x, kind, mx, d, mn, Z["ref/%s/windows" % name], Z["ref/%s/y_rows" % name])
    df, y = make_forecasting_frame(x=range(4), kind="test", max_timeshift=1, rolling_direction=1)
    expected_df = pd.DataFrame({"id": [("id", 1), ("id", 2), ("id", 3)], "kind": ["test"] * 3, "value": [0, 1, 2],
                                "time": [0, 1, 2]})
    pd.testing.assert_frame_equal(df.to_frame().sort_index(axis=1), expected_df.sort_index(axis=1))
    pd.testing.assert_series_equal(y, pd.Series(data=[1, 2, 3], index=[("id", 1), ("id", 2), ("id", 3)], name="value"))
    t_index = pd.date_range("1/1/2011", periods=4, freq="h")
    _, y = make_forecasting_frame(x=pd.Series(data=range(4), index=t_index), kind="test", max_timeshift=1,
                                  rolling_direction=1)
    pd.testing.assert_series_equal(y, pd.Series(data=[1, 2, 3], index=zip(["id"] * 3, t_index[1:]), name="value"))


def test_windows_are_views_on_one_buffer():
    """x = 0 .. 5, max_timeshift 2, rolling backwards: windows ("id", 0) .. ("id", 4) of 2, 2, 2, 2 and 1 rows; window 5
    is empty after the drop of its last row and gone, and y has entries for 1 .. 4"""
    df_shift, y = make_forecasting_frame(np.arange(6.0), "k", 2, -1)
    assert df_shift.ids == [("id", t) for t in range(5)]
    assert df_shift.length.tolist() == [2, 2, 2, 2, 1] and df_shift.begin.tolist() == [0, 1, 2, 3, 4]
    assert len(df_shift.values) == 1 and df_shift.values["value"].shape == (6,)
    assert y.index.tolist() == [("id", t) for t in range(1, 5)] and y.tolist() == [1.0, 2.0, 3.0, 4.0]


@pytest.mark.parametrize("kw, message", [
    (dict(rolling_direction=0), "Rolling direction of 0 is not possible"),
    (dict(max_timeshift=0), "max_timeshift needs to be positive!"),
    (dict(max_timeshift=-3), "max_timeshift needs to be positive!"),
    (dict(min_timeshift=-1), "min_timeshift needs to be positive or zero!"),
])
def test_argument_errors(kw, message):
    args = dict(x=np.arange(5.0), kind="k", max_timeshift=None, rolling_direction=1)
    with pytest.raises(ValueError, match="^" + message + "$"):
        make_forecasting_frame(**dict(args, **kw))


@pytest.mark.parametrize("x", [[], [1.0], np.zeros(1), pd.Series([2.0], index=[5])])
def test_zero_or_one_rows(x):
    with pytest.raises(ValueError, match="zero or one rows"):
        make_forecasting_frame(x, "k", None, 1)


def test_nan_in_the_index():
    with pytest.raises(ValueError, match="NaN values in your sort column"):
        make_forecasting_frame(pd.Series([1.0, 2.0, 3.0], index=[0.0, np.nan, 2.0]), "k", None, 1)


TIED = [pd.Series([1.0, 2.0, 3.0, 4.0], index=[0, 0, 1, 2]),
        pd.Series([1.0, 2.0, 3.0, 4.0], index=[0, 1, 2, 2]),
        pd.Series([1.0, 2.0, 3.0, 4.0, 5.0], index=[0, 1, 1, 2, 3])]


@pytest.mark.parametrize("x", TIED)
@pytest.mark.parametrize("direction", [1, -1])
def test_tied_window_names_are_refused(x, direction):
    """windows of one name, which the reference merges into one series before it drops a row of it"""
    with pytest.raises(ValueError, match="same name"):
        make_forecasting_frame(x, "k", None, direction)


def test_ties_that_name_no_two_windows_are_kept():
    """with stride 2 the tied keys 1, 1 name one window only: nothing is merged, as in the reference"""
    x = pd.Series([1.0, 2.0, 3.0, 4.0, 5.0], index=[0, 1, 1, 2, 3])
    df_shift, y = make_forecasting_frame(x, "k", None, 2)
    assert [i[1] for i in df_shift.ids] == [1, 3]


torch = pytest.importorskip("torch")


def call(x=None, **kw):
    x = torch.zeros(8, dtype=torch.float32) if x is None else x
    return extract_features_forecasting_device(x, kw.pop("kind", "k"), kw.pop("max_timeshift", None),
                                               kw.pop("rolling_direction", 1), **kw)


@pytest.mark.parametrize("kw, message", [
    (dict(rolling_direction=0), "Rolling direction of 0 is not possible"),
    (dict(max_timeshift=0), "max_timeshift needs to be positive!"),
    (dict(min_timeshift=-1), "min_timeshift needs to be positive or zero!"),
    (dict(x=torch.zeros(1)), "zero or one rows"),
    (dict(x=torch.zeros(0)), "zero or one rows"),
])
def test_device_argument_errors_come_before_the_device(kw, message):
    with pytest.raises(ValueError, match=message):
        call(**kw)


def test_device_argument_errors_come_before_the_tensor_checks():
    with pytest.raises(ValueError, match="Rolling direction of 0"):
        call(x=np.zeros(5), rolling_direction=0)


@pytest.mark.parametrize("kw, error, message", [
    (dict(x=np.zeros(5)), TypeError, "x must be a torch.Tensor"),
    (dict(x=torch.zeros(5, 2)), ValueError, "x must be 1-D"),
    (dict(x=torch.zeros(5, dtype=torch.int64)), TypeError, "x must be float32, float64, float16 or bfloat16"),
    (dict(index=np.arange(8)), TypeError, "index must be a torch.Tensor"),
    (dict(index=torch.arange(7)), ValueError, "index has 7 entries, x 8"),
    (dict(index=torch.arange(8, dtype=torch.int32)), TypeError, "index must be int64 or float64"),
    (dict(kind="a__b"), ValueError, "__"),
])
def test_device_tensor_checks(kw, error, message):
    with pytest.raises(error, match=message):
        call(**kw)


def test_cpu_tensors_are_refused_after_the_argument_checks():
    with pytest.raises(ValueError, match="^x must be a CUDA tensor, got one on cpu$"):
        call(x=torch.zeros(8, dtype=torch.float64), index=torch.arange(8))
