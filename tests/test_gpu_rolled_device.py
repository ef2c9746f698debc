"""extract_features_rolled_device on long-format CUDA tensors, bit for bit against extract_features(roll_time_series(...))
on the equivalent frame with a kind column (both run the same kernels on the same float32 windows, aligned alike), plus
the reference's RollingTestCase answers, the length limit per window, its stream contract and the errors it raises
before any kernel group runs."""
import numpy as np
import pandas as pd
import pytest

from tsfresh_b200 import (ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters, extract_features,
                          extract_features_rolled_device, impute, impute_dataframe_zero, roll_time_series)
from tsfresh_b200.extraction import get_context

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)

MOMENTS = {"mean": None, "maximum": None, "minimum": None, "standard_deviation": None, "length": None,
           "skewness": None}                     # every calculator in k_moments: the plan writes its rows directly
KINDS = ["a", "b", "c"]                          # sorted order = code order, as the rolled frame orders its kinds
K2FC = {"a": ComprehensiveFCParameters(), "b": MinimalFCParameters(), "c": MOMENTS}


def bits(a):
    """float64 bit patterns, every NaN made the same NaN"""
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64)
    a = np.where(np.isnan(a), np.nan, a)
    return a.view(np.int64)


def assert_same(got, want):
    g, w = bits(got), bits(want)
    assert g.shape == w.shape
    bad = np.argwhere(g != w)
    assert len(bad) == 0, "%d cells differ, first %s" % (len(bad), bad[:5].tolist())


def rows_of(rng, spec):
    """spec {kind code: {id: length}} -> dict of row arrays in (kind, id, time) order; `time` int64, `ftime` float64
    (distinct inside a series)"""
    cols = {"id": [], "time": [], "kind": [], "value": []}
    for code, series in spec.items():
        for i, n in series.items():
            cols["id"].append(np.full(n, i, dtype=np.int64))
            cols["time"].append(np.arange(n, dtype=np.int64) * 5 - 40)
            cols["kind"].append(np.full(n, code, dtype=np.int64))
            cols["value"].append(rng.standard_normal(n).astype(np.float32))
    rows = {c: np.concatenate(v) for c, v in cols.items()}
    rows["ftime"] = rows["time"] * 0.25 + 0.125
    return rows


def shuffled(rows, rng):
    p = rng.permutation(len(rows["id"]))
    return {c: v[p] for c, v in rows.items()}


def frame(rows, kinds=KINDS, sort="time"):
    df = pd.DataFrame({"id": rows["id"], "kind": np.array(kinds, dtype=object)[rows["kind"]], "value": rows["value"]})
    if sort is not None:
        df[sort] = rows[sort]
    return df


def on_device(rows, sort="time"):
    t = {c: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for c, v in rows.items()}
    return dict(ids=t["id"], values=t["value"], sort=t[sort] if sort is not None else None, kind=t["kind"])


ROLL = ("rolling_direction", "max_timeshift", "min_timeshift")


def host(rows, kinds=KINDS, sort="time", **kw):
    roll = {k: kw.pop(k) for k in ROLL if k in kw}
    rolled = roll_time_series(frame(rows, kinds, sort), column_id="id", column_sort=sort, column_kind="kind", **roll)
    return extract_features(rolled, **kw)


def check(rows, kinds=KINDS, sort="time", **kw):
    """extract_features_rolled_device on the rows equals extract_features(roll_time_series(...)) on their frame"""
    a = on_device(rows, sort)
    X, wid, wkey, cols = extract_features_rolled_device(a["ids"], a["values"], a["sort"], a["kind"], kinds=kinds, **kw)
    want = host(rows, kinds, sort, **kw)
    assert cols == list(want.columns)
    assert X.dtype == torch.float64 and X.device == DEV and tuple(X.shape) == want.shape
    assert wid.dtype == torch.int64 and wid.device == DEV and wkey.device == DEV
    assert wkey.dtype == (torch.int64 if sort is None else a["sort"].dtype)
    assert list(zip(wid.cpu().tolist(), wkey.cpu().tolist())) == want.index.tolist()
    assert_same(X, want.to_numpy())
    return X, wid, wkey, cols


def ragged_spec():
    """three kinds, lengths 1 .. 1 300, some ids missing from some kinds, negative and large ids"""
    ids = [-(1 << 62), -5, 0, 3, 7, 1 << 40, 123456789012]
    lens = [1, 2, 3, 255, 257, 1300]
    spec = {0: {}, 1: {}, 2: {}}
    for j, i in enumerate(ids):
        if j % 3 != 1:
            spec[0][i] = lens[j % len(lens)]
        if j % 2 == 0:
            spec[1][i] = lens[(j + 2) % len(lens)]
        spec[2][i] = lens[(j + 4) % len(lens)]
    spec[2][99] = 1300                           # an id only one kind has
    return spec


@pytest.mark.parametrize("direction", [1, 2, 32, -1, -2, -32])
def test_directions_and_strides(direction):
    rng = np.random.default_rng(abs(direction) * 2 + (direction > 0))
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    mx = 40 if abs(direction) < 32 else None
    X, wid, wkey, _ = check(rows, kind_to_fc_parameters=K2FC, rolling_direction=direction, max_timeshift=mx)
    assert bool(torch.isnan(X).any())            # window names that only some kinds have
    assert get_context(0).launch_count() > 0


@pytest.mark.parametrize("max_timeshift, min_timeshift", [(None, 0), (None, 300), (100, 0), (100, 60), (5000, 0),
                                                          (5000, 1299), (10, 20)])
def test_max_and_min_timeshift(max_timeshift, min_timeshift):
    rng = np.random.default_rng(11)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    for direction in (7, -7):
        check(rows, default_fc_parameters=EfficientFCParameters(), rolling_direction=direction,
              max_timeshift=max_timeshift, min_timeshift=min_timeshift)


def test_ordered_and_shuffled_rows_agree():
    rng = np.random.default_rng(12)
    spec = {k: {i: 200 + 17 * i + 5 * k for i in range(20)} for k in range(3)}     # every kind has every id
    ordered = rows_of(rng, spec)
    kw = dict(kind_to_fc_parameters=K2FC, rolling_direction=16, max_timeshift=63)
    X1, ids1, keys1, _ = check(ordered, **kw)
    X2, ids2, keys2, _ = check(shuffled(ordered, rng), **kw)
    assert_same(X2, X1)
    assert torch.equal(ids1, ids2) and torch.equal(keys1, keys2)


def test_sort_none_int_and_float_keys():
    rng = np.random.default_rng(13)
    rows = rows_of(rng, ragged_spec())
    kw = dict(default_fc_parameters=EfficientFCParameters(), rolling_direction=5, max_timeshift=30, min_timeshift=2)
    check(rows, sort=None, **kw)                 # input order inside a series; names are row numbers
    X1, _, k1, _ = check(shuffled(rows, rng), sort="time", **kw)
    X2, _, k2, _ = check(shuffled(rows, rng), sort="ftime", **kw)
    assert_same(X2, X1)
    assert k2.dtype == torch.float64 and torch.equal(k2, k1.to(torch.float64) * 0.25 + 0.125)


def test_device_impute():
    rng = np.random.default_rng(14)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    rows["value"][rng.choice(len(rows["value"]), 20, replace=False)] = np.inf
    rows["value"][rng.choice(len(rows["value"]), 5, replace=False)] = -np.inf
    for fn in (impute, impute_dataframe_zero):
        X, _, _, _ = check(rows, default_fc_parameters=EfficientFCParameters(), impute_function=fn, rolling_direction=9,
                           max_timeshift=50)
        assert bool(torch.isfinite(X).all())


def test_non_default_stream():
    rng = np.random.default_rng(15)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    a = on_device(rows)
    kw = dict(kinds=KINDS, kind_to_fc_parameters=K2FC, rolling_direction=-4, max_timeshift=80)
    want, want_ids, want_keys, _ = extract_features_rolled_device(a["ids"], a["values"], a["sort"], a["kind"], **kw)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        values = a["values"] * 1.0               # written by a torch kernel on the side stream right before the call
        X, ids, keys, _ = extract_features_rolled_device(a["ids"], values, a["sort"], a["kind"], **kw)
        host_x, host_ids, host_keys = X.cpu(), ids.cpu(), keys.cpu()
    side.synchronize()
    assert_same(host_x, want)
    assert torch.equal(host_ids, want_ids.cpu()) and torch.equal(host_keys, want_keys.cpu())


def reference_windows(ids, values):
    """{window name: (rows, sum)} from a rolled frame's id and value columns, as the reference's tests state them"""
    out = {}
    for i, v in zip(ids, values):
        n, s = out.get(i, (0, 0))
        out[i] = (n + 1, s + v)
    return out


def test_reference_rolling_test_case():
    """Constants of the reference's RollingTestCase (tests/units/utilities/test_dataframe_functions.py:148-740): two
    kinds a and b of ids 1 (4 rows) and 2 (2 rows)"""
    t = torch.tensor([0, 1, 2, 3, 20, 21], dtype=torch.int64, device=DEV)
    i = torch.tensor([1, 1, 1, 1, 2, 2], dtype=torch.int64, device=DEV)
    a = torch.tensor([1, 2, 3, 4, 10, 11], dtype=torch.float32, device=DEV)
    b = torch.tensor([5, 6, 7, 8, 12, 13], dtype=torch.float32, device=DEV)
    ids, sort, values = torch.cat([i, i]), torch.cat([t, t]), torch.cat([a, b])
    kind = torch.tensor([0] * 6 + [1] * 6, dtype=torch.int32, device=DEV)
    settings = {"length": None, "sum_values": None}
    cases = {
        1: ([(1, 0)] + [(1, 1)] * 2 + [(1, 2)] * 3 + [(1, 3)] * 4 + [(2, 20)] + [(2, 21)] * 2,
            [1, 1, 2, 1, 2, 3, 1, 2, 3, 4, 10, 10, 11], [5, 5, 6, 5, 6, 7, 5, 6, 7, 8, 12, 12, 13]),
        2: ([(1, 1)] * 2 + [(1, 3)] * 4 + [(2, 21)] * 2, [1, 2, 1, 2, 3, 4, 10, 11], [5, 6, 5, 6, 7, 8, 12, 13]),
        -2: ([(1, 0)] * 4 + [(1, 2)] * 2 + [(2, 20)] * 2, [1, 2, 3, 4, 3, 4, 10, 11], [5, 6, 7, 8, 7, 8, 12, 13]),
        -1: ([(1, 0)] * 4 + [(1, 1)] * 3 + [(1, 2)] * 2 + [(1, 3)] + [(2, 20)] * 2 + [(2, 21)],
             [1, 2, 3, 4, 2, 3, 4, 3, 4, 4, 10, 11, 11], [5, 6, 7, 8, 6, 7, 8, 7, 8, 8, 12, 13, 13]),
    }
    for direction, (names, va, vb) in cases.items():
        X, wid, wkey, cols = extract_features_rolled_device(ids, values, sort, kind, kinds=["a", "b"],
                                                            default_fc_parameters=settings, rolling_direction=direction)
        assert cols == ["a__length", "a__sum_values", "b__length", "b__sum_values"]
        wa, wb = reference_windows(names, va), reference_windows(names, vb)
        got = list(zip(wid.cpu().tolist(), wkey.cpu().tolist()))
        assert got == sorted(wa), direction
        X = X.cpu().numpy()
        assert [tuple(r) for r in X[:, :2].tolist()] == [wa[n] for n in got], direction
        assert [tuple(r) for r in X[:, 2:].tolist()] == [wb[n] for n in got], direction


def test_long_series_in_short_windows_against_the_oracle():
    """a 40 000-sample series is past the quadratic entropies' 21 000-sample cap, its 256-sample windows are not"""
    from oracle.extract import compare, oracle_rows
    from tsfresh_b200.plan import Plan
    rng = np.random.default_rng(16)
    n = 40_000
    x = rng.standard_normal(n).astype(np.float32)
    ids = torch.zeros(n, dtype=torch.int64, device=DEV)
    settings = ComprehensiveFCParameters()
    X, wid, wkey, cols = extract_features_rolled_device(ids, torch.from_numpy(x).to(DEV), default_fc_parameters=settings,
                                                        rolling_direction=2_011, max_timeshift=255, min_timeshift=255)
    ends = wkey.cpu().numpy()
    assert len(ends) == 20 and bool((wid == 0).all())
    assert np.array_equal(np.diff(ends), np.full(19, 2_011)) and ends[-1] == n - 1
    want = oracle_rows([x[e - 255:e + 1].astype(np.float64) for e in ends], settings)
    bad = compare(X.cpu().numpy(), want, Plan(settings).suffixes)
    assert not bad, bad[:5]


def test_window_length_limit_is_per_window():
    """max_timeshift beyond the series: the windows are only as long as the series, and the exact longest window, not
    max_timeshift + 1, is checked against sample_entropy's 21 000-sample limit"""
    rng = np.random.default_rng(17)
    n = 20_000
    rows = {"id": np.zeros(n, dtype=np.int64), "time": np.arange(n, dtype=np.int64), "kind": np.zeros(n, dtype=np.int64),
            "value": rng.standard_normal(n).astype(np.float32)}
    settings = {"sample_entropy": None, "mean": None}
    check(rows, kinds=["a"], default_fc_parameters=settings, rolling_direction=4_999, max_timeshift=30_000)
    ctx = get_context(0)
    long_rows = dict(rows, id=np.zeros(n + 1_001, dtype=np.int64), time=np.arange(n + 1_001, dtype=np.int64),
                     kind=np.zeros(n + 1_001, dtype=np.int64), value=rng.standard_normal(n + 1_001).astype(np.float32))
    a = on_device(long_rows)
    with pytest.raises(ValueError, match="exceeds"):
        extract_features_rolled_device(a["ids"], a["values"], a["sort"], a["kind"], kinds=["a"],
                                       default_fc_parameters=settings, rolling_direction=-10_000)
    assert ctx.launch_count() == 0
    # the same rows in windows of at most 21 000 samples are extracted
    check(long_rows, kinds=["a"], default_fc_parameters=settings, rolling_direction=-10_000, max_timeshift=20_999)


def test_errors_before_any_kernel_group():
    ctx = get_context(0)
    rng = np.random.default_rng(18)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    a = on_device(rows)
    kw = dict(kinds=KINDS, default_fc_parameters=EfficientFCParameters(), rolling_direction=3, max_timeshift=40)
    want, want_ids, want_keys, _ = extract_features_rolled_device(a["ids"], a["values"], a["sort"], a["kind"], **kw)

    def raises(match, roll=None, **changed):
        b = dict(a, **changed)
        with pytest.raises(ValueError, match=match):
            extract_features_rolled_device(b["ids"], b["values"], b["sort"], b["kind"], **dict(kw, **(roll or {})))
        assert ctx.launch_count() == 0 and ctx.last_kernels() == []
        X, ids, keys, _ = extract_features_rolled_device(a["ids"], a["values"], a["sort"], a["kind"], **kw)
        assert_same(X, want)
        assert torch.equal(ids, want_ids) and torch.equal(keys, want_keys)
        assert ctx.launch_count() > 0

    # the first four rows of a 1 300-row series share one sort key: the windows named by rows 0 and 3 have one name
    sel = torch.nonzero((a["ids"] == -5) & (a["kind"] == 2)).flatten()
    order = sel[torch.argsort(a["sort"][sel])]
    assert len(order) == 1300
    tied = a["sort"].clone()
    tied[order[:4]] = int(tied[order[0]])
    raises("same name", sort=tied)
    ftied = (a["sort"] + 40).to(torch.float64)
    ftied[order[:3]] = -0.0
    ftied[order[3]] = 0.0                        # -0.0 and 0.0 are one name, as pandas holds them equal
    raises("same name", sort=ftied)
    for kind_of_nan in range(3):
        bad = a["values"].clone()
        bad[int(torch.nonzero(a["kind"] == kind_of_nan)[-1])] = float("nan")
        raises("value column contains NaN", values=bad)
    fsort = a["sort"].to(torch.float64)
    fsort[17] = float("nan")
    raises("sort keys contain NaN", sort=fsort)
    for code in (3, -1):
        bad = a["kind"].clone()
        bad[5] = code
        raises(r"kind code is outside 0 \.\. 2", kind=bad)
    n = 131_073                                  # one window past the spectral group's limit
    raises("exceeds", roll=dict(max_timeshift=None), ids=torch.cat([a["ids"], torch.full((n,), 555, dtype=torch.int64, device=DEV)]),
           values=torch.cat([a["values"], torch.zeros(n, device=DEV)]),
           sort=torch.cat([a["sort"], torch.arange(n, device=DEV)]),
           kind=torch.cat([a["kind"], torch.ones(n, dtype=torch.int64, device=DEV)]))
    with pytest.raises(ValueError, match="Rolling direction of 0"):
        extract_features_rolled_device(a["ids"], a["values"], a["sort"], a["kind"], **dict(kw, rolling_direction=0))
