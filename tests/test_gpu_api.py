"""extract_features() drop-in behaviour on the GPU path: input formats, row-order invariance (device sort),
id dtypes, kind handling, column names -- mirrors tests/units/feature_extraction/test_extraction.py and
test_data.py of the reference."""
import numpy as np
import pandas as pd
import pytest

from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from tests.helpers import synthetic_series
from tsfresh_b200 import EfficientFCParameters, MinimalFCParameters, extract_features
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu


def long_frame(series, ids=None, shuffle_seed=None):
    ids = list(range(len(series))) if ids is None else ids
    df = pd.DataFrame({
        "id": np.concatenate([np.full(len(s), i) for i, s in zip(ids, series)]),
        "time": np.concatenate([np.arange(len(s)) for s in series]),
        "value": np.concatenate(series).astype(np.float32),
    })
    if shuffle_seed is not None:
        df = df.sample(frac=1.0, random_state=shuffle_seed).reset_index(drop=True)
    return df


def check(X, series, settings, prefix="value__"):
    plan = Plan(settings)
    assert list(X.columns) == [prefix + s for s in plan.suffixes]
    want = oracle_rows([np.asarray(s, np.float32).astype(np.float64) for s in series], settings)
    bad = compare(X.to_numpy(), want, plan.suffixes, atol=NOISE_FLOOR)     # these frames hold 1- and 2-sample series
    assert not bad, bad[:20]


def test_long_frame_sorted_and_shuffled():
    rng = np.random.default_rng(0)
    series = [rng.standard_normal(n).astype(np.float32) for n in (50, 256, 17, 300, 64, 1, 2)]
    s = EfficientFCParameters()
    X = extract_features(long_frame(series), column_id="id", column_sort="time", default_fc_parameters=s)
    assert X.index.tolist() == list(range(len(series))) and X.dtypes.eq(np.float64).all()
    check(X, series, s)
    Xs = extract_features(long_frame(series, shuffle_seed=3), column_id="id", column_sort="time", default_fc_parameters=s)
    np.testing.assert_array_equal(X.to_numpy(), Xs.to_numpy())       # test_extraction.py:207-237
    assert list(X.columns) == list(Xs.columns)


def test_ids_unsorted_negative_and_strings():
    series = list(synthetic_series(1, 5, 40))
    s = MinimalFCParameters()
    X = extract_features(long_frame(series, ids=[30, -2, 7, 100, 0], shuffle_seed=1), column_id="id", column_sort="time",
                         default_fc_parameters=s)
    assert X.index.tolist() == [-2, 0, 7, 30, 100]
    order = [1, 4, 2, 0, 3]
    check(X, [series[i] for i in order], s)
    df = long_frame(series, ids=["b", "a", "e", "d", "c"])
    X2 = extract_features(df, column_id="id", column_sort="time", default_fc_parameters=s)
    assert X2.index.tolist() == ["a", "b", "c", "d", "e"]
    check(X2, [series[i] for i in [1, 0, 4, 3, 2]], s)


def test_wide_dict_and_kind_formats():
    a = list(synthetic_series(2, 4, 30))
    b = list(synthetic_series(3, 4, 30))
    s = MinimalFCParameters()
    wide = pd.DataFrame({"id": np.repeat(np.arange(4), 30), "t": np.tile(np.arange(30), 4),
                         "a": np.concatenate(a), "b": np.concatenate(b)})
    X = extract_features(wide, column_id="id", column_sort="t", default_fc_parameters=s)
    assert X.shape == (4, 20)
    check(X[[c for c in X.columns if c.startswith("a__")]], a, s, "a__")
    check(X[[c for c in X.columns if c.startswith("b__")]], b, s, "b__")
    long = wide.melt(id_vars=["id", "t"], var_name="kind", value_name="val")
    Xl = extract_features(long, column_id="id", column_sort="t", column_kind="kind", column_value="val", default_fc_parameters=s)
    pd.testing.assert_frame_equal(X, Xl[X.columns])
    d = {"a": wide[["id", "t", "a"]].rename(columns={"a": "v"}), "b": wide[["id", "t", "b"]].rename(columns={"b": "v"})}
    Xd = extract_features(d, column_id="id", column_sort="t", column_value="v", default_fc_parameters=s)
    pd.testing.assert_frame_equal(X, Xd[X.columns])
    # per-kind settings (extraction.py:333-336, test_extraction.py:78-89)
    Xk = extract_features(wide, column_id="id", column_sort="t", default_fc_parameters=s,
                          kind_to_fc_parameters={"b": {"maximum": None, "quantile": [{"q": 0.5}]}})
    assert [c for c in Xk.columns if c.startswith("b__")] == ["b__maximum", "b__quantile__q_0.5"]


def test_errors_like_the_reference():
    df = long_frame(list(synthetic_series(1, 3, 10)))
    with pytest.raises(ValueError):
        extract_features(df, column_id=None, column_sort="time")
    bad = df.copy()
    bad.loc[3, "value"] = np.nan
    with pytest.raises(ValueError, match="must not contain NaN"):
        extract_features(bad, column_id="id", column_sort="time", default_fc_parameters=MinimalFCParameters())
    with pytest.raises(ValueError, match="not allowed to contain '__'"):
        extract_features(df.rename(columns={"value": "va__lue"}), column_id="id", column_sort="time",
                         default_fc_parameters=MinimalFCParameters())
    with pytest.raises(NotImplementedError):          # no CPU fallback for user callables
        extract_features(df, column_id="id", column_sort="time", default_fc_parameters={(lambda x: 1.0): None})
    with pytest.raises(ValueError):
        extract_features([1, 2, 3], column_id="id")

    # a NaN found on the device is the reference's error, naming the kind, with no library error chained to it
    def nan_error(label, f, *args, **kw):
        with pytest.raises(ValueError) as e:
            f(*args, default_fc_parameters=MinimalFCParameters(), **kw)
        assert str(e.value) == "Column must not contain NaN values: %s" % label and e.value.__suppress_context__
    from tsfresh_b200 import do_extraction_on_chunks, roll_time_series
    x = pd.Series(np.arange(20, dtype=np.float32))
    nan_error("b", do_extraction_on_chunks, [(1, "a", x), (1, "b", x.where(x != 5))])
    wide = df.assign(other=bad["value"])
    nan_error("other", extract_features, roll_time_series(wide, column_id="id", column_sort="time", max_timeshift=3))
    stacked = pd.concat([df.assign(kind="a"), bad.assign(kind="b")], ignore_index=True)
    nan_error("b", extract_features, roll_time_series(stacked, column_id="id", column_sort="time", column_kind="kind",
                                                      max_timeshift=3))


def test_pivot_false_triples():
    series = list(synthetic_series(5, 3, 20))
    tr = extract_features(long_frame(series), column_id="id", column_sort="time",
                          default_fc_parameters={"maximum": None, "length": None}, pivot=False)
    assert len(tr) == 6 and tr[0][1] == "value__maximum" and tr[1] == (0, "value__length", 20.0)


def test_duplicate_timestamps_are_stable():
    # equal sort keys keep their row order (documented tie rule; the reference's quicksort leaves it unspecified)
    df = pd.DataFrame({"id": [1, 1, 1, 0, 0], "time": [5, 5, 1, 2, 2], "value": np.float32([3, 4, 9, 7, 8])})
    X = extract_features(df, column_id="id", column_sort="time", default_fc_parameters={"mean_change": None})
    assert X.loc[1, "value__mean_change"] == (4 - 9) / 2 and X.loc[0, "value__mean_change"] == 1.0


def test_rolled_windows_as_views_match_oracle_on_materialised_windows():
    """BASELINE.json configs[4] path: roll_time_series(win, stride) windows are (begin, len) views over the one
    value buffer (tsfx_roll_windows, checked against the reference's window ids in tests/test_host_side.py);
    extracting the views must equal the oracle on the copied-out windows."""
    from tests.helpers import to_csr
    from tsfresh_b200 import _lib
    from tsfresh_b200.extraction import _device_plan, get_context
    series = list(synthetic_series(9, 3, 200)) + [synthetic_series(10, 1, 77)[0]]
    values, begin, lens = to_csr(series)
    wb, wl, wp, we = _lib.roll_windows(begin, lens, 32, 63, 63)         # windows of 64 rows, stride 32
    assert len(wb) == 3 * 5 + 1 and set(wl.tolist()) == {64}
    settings = EfficientFCParameters()
    plan = Plan(settings)
    dp = _device_plan(get_context(0), plan)
    got = dp.extract_csr(values, wb, wl)
    windows = [values[b:b + n].astype(np.float64) for b, n in zip(wb, wl)]
    bad = compare(got, oracle_rows(windows, settings), plan.suffixes)
    assert not bad, bad[:20]


def test_extract_features_on_rolled_views():
    """extract_features(roll_time_series(df, ...)): the two reference calls, with windows as views; equals the oracle on
    the materialised windows, index = (id, time of the id row), both rolling directions, two value columns."""
    from tsfresh_b200 import impute, roll_time_series
    from oracle import impute as oi
    series = list(synthetic_series(31, 3, 90)) + [synthetic_series(32, 1, 40)[0]]
    df = long_frame(series, ids=[7, 3, 11, 5], shuffle_seed=4)
    df["other"] = (df["value"] * 2 + 1).astype(np.float32)
    settings = EfficientFCParameters()
    plan = Plan(settings)
    for rd, mx, mn in ((16, 31, 31), (-16, 31, 31), (25, 40, 9)):
        rolled = roll_time_series(df, column_id="id", column_sort="time", rolling_direction=rd, max_timeshift=mx, min_timeshift=mn)
        X = extract_features(rolled, default_fc_parameters=settings)
        assert list(X.index) == rolled.ids and len(X) == len(rolled) > 0
        assert list(X.columns) == ["value__" + s for s in plan.suffixes] + ["other__" + s for s in plan.suffixes]
        for kind, lo in (("value", 0), ("other", plan.n_cols)):
            windows = [rolled.values[kind][b:b + n].astype(np.float64) for b, n in zip(rolled.begin, rolled.length)]
            bad = compare(X.to_numpy()[:, lo:lo + plan.n_cols], oracle_rows(windows, settings), plan.suffixes)
            assert not bad, (rd, kind, bad[:10])
    Xi = extract_features(rolled, default_fc_parameters=settings, impute_function=impute)
    assert np.array_equal(Xi.to_numpy(), oi.impute(X.to_numpy()))
    # long format with a kind column: kinds of different length, rows = union of the window ids
    stacked = pd.concat([df[["id", "time", "value"]].assign(kind="a"),
                         df[df["time"] < 50][["id", "time", "other"]].rename(columns={"other": "value"}).assign(kind="b")],
                        ignore_index=True)
    rk = roll_time_series(stacked, column_id="id", column_sort="time", column_kind="kind", rolling_direction=16,
                          max_timeshift=31, min_timeshift=31)
    Xk = extract_features(rk, default_fc_parameters=settings)
    assert list(Xk.columns) == ["a__" + s for s in plan.suffixes] + ["b__" + s for s in plan.suffixes]
    assert list(Xk.index) == sorted(set(rk.parts["a"].ids) | set(rk.parts["b"].ids))
    for kind, lo in (("a", 0), ("b", plan.n_cols)):
        part = rk.parts[kind]
        windows = [part.values["value"][b:b + n].astype(np.float64) for b, n in zip(part.begin, part.length)]
        got = Xk.loc[pd.Index(part.ids, tupleize_cols=False)].to_numpy()[:, lo:lo + plan.n_cols]
        bad = compare(got, oracle_rows(windows, settings), plan.suffixes)
        assert not bad, (kind, bad[:10])
    missing = [w for w in Xk.index if w not in set(rk.parts["b"].ids)]
    assert missing and np.isnan(Xk.loc[pd.Index(missing, tupleize_cols=False)].to_numpy()[:, plan.n_cols:]).all()


def test_distributor_plugin_map_reduce():
    """The reference's plugin seam (utilities/distribution.py:74-104): extract_features hands the distributor
    `data` (an iterable of (id, kind, pd.Series)) and `function_kwargs`; B200Distributor must return the triples
    that `data.pivot` expects without ever calling the Python map function."""
    from tsfresh_b200.distributor import B200Distributor, is_distributor
    series = list(synthetic_series(21, 4, 50))
    data = [(i, "a", pd.Series(s)) for i, s in enumerate(series)] + [(i, "b", pd.Series(s[::-1].copy())) for i, s in enumerate(series)]
    settings = {"maximum": None, "quantile": [{"q": 0.25}], "linear_trend": [{"attr": "slope"}]}
    dist = B200Distributor()
    assert is_distributor(dist)

    def must_not_be_called(*a, **k):
        raise AssertionError("the Python per-series function must not run")

    triples = dist.map_reduce(must_not_be_called, data=data, chunk_size=None,
                              function_kwargs=dict(default_fc_parameters=settings, kind_to_fc_parameters={"b": {"minimum": None}},
                                                   show_warnings=False))
    dist.close()
    got = {(i, n): v for i, n, v in triples}
    assert len(got) == 4 * 3 + 4 * 1
    for i, s in enumerate(series):
        assert got[(i, "a__maximum")] == float(s.max())
        assert got[(i, "a__quantile__q_0.25")] == pytest.approx(np.quantile(s.astype(np.float64), 0.25), rel=1e-12)
        assert got[(i, "b__minimum")] == float(s.min())
        assert (i, "b__maximum") not in got


def test_csr_tsdata_seam():
    """plugin seam #2: what the reference's ApplyDistributor does with a non-iterable TsData (apply, then pivot)"""
    from tests.helpers import to_csr
    from tsfresh_b200.distributor import CsrTsData
    series = list(synthetic_series(31, 5, 64))
    values, begin, lens = to_csr(series)
    data = CsrTsData(values, begin, lens, ids=[3, 5, 8, 13, 21])
    res = data.apply(None, meta=[("id", "int64"), ("variable", "object"), ("value", "float64")],
                     default_fc_parameters={"maximum": None, "median": None}, kind_to_fc_parameters=None, show_warnings=False)
    X = data.pivot(res)
    assert list(X.columns) == ["value__maximum", "value__median"] and list(X.index) == [3, 5, 8, 13, 21]
    np.testing.assert_array_equal(X["value__maximum"].to_numpy(), [float(s.max()) for s in series])
    np.testing.assert_array_equal(X["value__median"].to_numpy(), [float(np.median(s.astype(np.float64))) for s in series])


def test_linear_trend_timewise_on_a_datetime_index():
    """feature_calculators.py:2274-2306 through extract_features: golden values of the unmodified reference
    (tests/golden/timewise.npz, oracle/make_golden_timewise.py), rows in order and shuffled (the timestamps follow
    the device sort), and the no-DatetimeIndex case (skipped with a warning, extraction.py:349-358)."""
    import os
    import warnings
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "timewise.npz"), allow_pickle=True)
    fc = {"linear_trend_timewise": [{"attr": a} for a in ("pvalue", "rvalue", "intercept", "slope", "stderr")],
          "mean": None, "linear_trend": [{"attr": "slope"}]}
    df = pd.DataFrame({"id": z["id"], "value": z["value"]}, index=pd.DatetimeIndex(z["t_ns"].astype("datetime64[ns]")))
    for frame in (df, df.sample(frac=1.0, random_state=3)):
        # without a sort column the reference keeps the row order inside each id: shuffle whole frames only by id blocks
        if frame is not df:
            frame = pd.concat([g for _, g in sorted(df.groupby("id"), key=lambda kv: -kv[0])])
        X = extract_features(frame, column_id="id", default_fc_parameters=fc)
        assert list(X.columns) == list(z["columns"]) and list(X.index) == list(z["index"])
        suffixes = [c.split("__", 1)[1] for c in X.columns]
        bad = compare(X.to_numpy(), z["reference"], suffixes, atol=NOISE_FLOOR)     # 2- and 3-sample series
        assert not bad, bad[:20]
    plain = df.reset_index(drop=True)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        X = extract_features(plain, column_id="id", default_fc_parameters=fc, show_warnings=True)
    assert [c for c in X.columns if "timewise" in c] == [] and any("DatetimeIndex" in str(m.message) for m in w)


def test_do_extraction_on_chunk_signature():
    """the per-(id, kind) function of the dask / spark bindings (extraction.py:308-386, bindings.py:50-54)"""
    from tsfresh_b200 import _do_extraction_on_chunk, do_extraction_on_chunks
    rng = np.random.default_rng(21)
    x = pd.Series(rng.standard_normal(100).astype(np.float32))
    s = MinimalFCParameters()
    triples = _do_extraction_on_chunk((7, "a", x), default_fc_parameters=s, kind_to_fc_parameters={})
    plan = Plan(s)
    assert [t[0] for t in triples] == [7] * plan.n_cols and [t[1] for t in triples] == ["a__" + c for c in plan.suffixes]
    want = oracle_rows([x.to_numpy(np.float64)], s)
    assert not compare(np.array([[t[2] for t in triples]]), want, plan.suffixes)
    # batched: two kinds with their own settings, order of the triples = order of the chunks
    y = pd.Series(rng.standard_normal(40).astype(np.float32))
    out = do_extraction_on_chunks([(1, "a", x), (1, "b", y), (2, "a", y)], s, {"b": {"maximum": None, "minimum": None}})
    assert [t[:2] for t in out[:plan.n_cols]] == [(1, "a__" + c) for c in plan.suffixes]
    assert out[plan.n_cols:plan.n_cols + 2] == [(1, "b__maximum", float(y.max())), (1, "b__minimum", float(y.min()))]
    assert len(out) == 2 * plan.n_cols + 2


def test_wide_format_kind_dimension_on_the_device(monkeypatch):
    """several value columns of one frame: ONE stage (a), per-kind settings, one result matrix (tsfx_extract_long_kinds);
    rows in order, shuffled, and with keys shuffled inside the ids -- same frame as the per-kind path"""
    rng = np.random.default_rng(31)
    lens = rng.integers(5, 60, 300)
    ids = np.repeat(np.arange(300) * 2 + 1, lens)
    t = np.concatenate([np.arange(l) for l in lens])
    df = pd.DataFrame({"id": ids, "time": t, "a": rng.standard_normal(len(ids)).astype(np.float32),
                       "b": rng.standard_normal(len(ids)).astype(np.float32).cumsum(), 7: rng.random(len(ids)).astype(np.float32)})
    s = EfficientFCParameters()
    per_kind = {"b": MinimalFCParameters(), 7: {"maximum": None, "quantile": [{"q": 0.25}]}}
    X = extract_features(df, column_id="id", column_sort="time", default_fc_parameters=s, kind_to_fc_parameters=per_kind)
    plan_a = Plan(s)
    assert list(X.columns) == ["a__" + c for c in plan_a.suffixes] + ["b__" + c for c in Plan(MinimalFCParameters()).suffixes] + \
        ["7__maximum", "7__quantile__q_0.25"]
    assert list(X.index) == sorted(set(ids))
    series_a = [df["a"].to_numpy()[ids == i] for i in X.index]
    assert not compare(X.to_numpy()[:, :plan_a.n_cols], oracle_rows([v.astype(np.float64) for v in series_a], s), plan_a.suffixes)
    np.testing.assert_allclose(X["7__maximum"].to_numpy(), [df[7].to_numpy()[ids == i].max() for i in X.index])
    # single-kind calls give the same blocks
    Xb = extract_features(df[["id", "time", "b"]], column_id="id", column_sort="time", default_fc_parameters=MinimalFCParameters())
    assert np.array_equal(X[[c for c in X.columns if c.startswith("b__")]].to_numpy(), Xb.to_numpy(), equal_nan=True)
    for frame in (df.sample(frac=1.0, random_state=1), df.iloc[np.lexsort((rng.random(len(df)), ids))]):
        Y = extract_features(frame, column_id="id", column_sort="time", default_fc_parameters=s, kind_to_fc_parameters=per_kind)
        assert list(Y.columns) == list(X.columns) and np.array_equal(Y.to_numpy(), X.to_numpy(), equal_nan=True)
    # a NaN in any kind is the reference's ValueError: pandas' scan names the column, the device scan every value column
    from tsfresh_b200 import extraction
    bad = df.copy()
    bad.loc[17, "b"] = np.nan
    for limit, label in ((1 << 20, "b"), (0, "a, b, 7")):
        monkeypatch.setattr(extraction, "_HOST_NAN_CHECK_ROWS", limit)
        with pytest.raises(ValueError, match="^Column must not contain NaN values: %s$" % label):
            extract_features(bad, column_id="id", column_sort="time", default_fc_parameters=MinimalFCParameters())
