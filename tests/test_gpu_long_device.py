"""extract_features_long_device on long-format CUDA tensors, bit for bit against extract_features on the equivalent frame
with a kind column (both run the same kernels on the same float32 data), plus its stream contract and the errors it
raises before any kernel group runs."""
import numpy as np
import pandas as pd
import pytest

from tsfresh_b200 import (ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters, extract_features,
                          extract_features_long_device, impute, impute_dataframe_zero)
from tsfresh_b200.extraction import get_context

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)

MOMENTS = {"mean": None, "maximum": None, "minimum": None, "standard_deviation": None, "length": None,
           "skewness": None}                     # every calculator in k_moments: the plan writes its rows directly
KINDS = ["a", "b", "c"]                          # sorted order = code order, as the frame orders its kinds
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
    """spec {kind code: {id: length}} -> dict of row arrays in (kind, id, time) order"""
    cols = {"id": [], "time": [], "kind": [], "value": []}
    for code, series in spec.items():
        for i, n in series.items():
            cols["id"].append(np.full(n, i, dtype=np.int64))
            cols["time"].append(np.arange(n, dtype=np.int64) * 5 - 40)
            cols["kind"].append(np.full(n, code, dtype=np.int64))
            cols["value"].append(rng.standard_normal(n).astype(np.float32))
    return {c: np.concatenate(v) for c, v in cols.items()}


def shuffled(rows, rng):
    p = rng.permutation(len(rows["id"]))
    return {c: v[p] for c, v in rows.items()}


def frame(rows, kinds=KINDS, sort="time"):
    df = pd.DataFrame({"id": rows["id"], "kind": np.array(kinds, dtype=object)[rows["kind"]], "value": rows["value"]})
    if sort is not None:
        df[sort] = rows[sort]
    if "times" in rows:
        df.index = pd.DatetimeIndex(rows["times"])
    return df


def on_device(rows, sort="time", kind_dtype=torch.int64):
    t = {c: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for c, v in rows.items()}
    return dict(ids=t["id"], values=t["value"], sort=t[sort] if sort is not None else None, kind=t["kind"].to(kind_dtype),
                times=t.get("times"))


def check(rows, kinds=KINDS, sort="time", **kw):
    """extract_features_long_device on the rows equals extract_features on their frame, bit for bit"""
    args = on_device(rows, sort)
    X, row_ids, cols = extract_features_long_device(args.pop("ids"), args.pop("values"), args.pop("sort"), args.pop("kind"),
                                                    kinds=kinds, times=args["times"], **kw)
    want = extract_features(frame(rows, kinds, sort), column_id="id", column_sort=sort, column_kind="kind",
                            column_value="value", **kw)
    assert cols == list(want.columns)
    assert X.dtype == torch.float64 and X.device == DEV and tuple(X.shape) == want.shape
    assert row_ids.dtype == torch.int64 and row_ids.device == DEV
    assert row_ids.cpu().numpy().tolist() == want.index.tolist()
    assert_same(X, want.to_numpy())
    return X, row_ids, cols


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


def test_shuffled_kinds_with_their_own_plans():
    rng = np.random.default_rng(1)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    X, row_ids, cols = check(rows, kind_to_fc_parameters=K2FC)
    assert bool(torch.isnan(X).any())            # (id, kind) pairs without rows
    assert get_context(0).launch_count() > 0


def test_ordered_and_shuffled_rows_agree():
    rng = np.random.default_rng(2)
    spec = {k: {i: 200 + 17 * i + 5 * k for i in range(40)} for k in range(3)}     # every kind has every id
    spec[1][40] = 3
    ordered = rows_of(rng, spec)
    X1, ids1, _ = check(ordered, kind_to_fc_parameters=K2FC)
    X2, ids2, _ = check(shuffled(ordered, rng), kind_to_fc_parameters=K2FC)
    assert_same(X2, X1)
    assert torch.equal(ids1, ids2)


def test_sort_none_and_float_keys_with_ties():
    rng = np.random.default_rng(3)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    s = EfficientFCParameters()
    check(rows, sort=None, default_fc_parameters=s)
    rows["ftime"] = rng.integers(0, 6, len(rows["id"])).astype(np.float64) * 0.5 - 1.0    # many equal keys
    check(rows, sort="ftime", default_fc_parameters=s)


def test_times_as_datetime_index():
    rng = np.random.default_rng(4)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    hours = rows["time"].astype(np.int64) * 3_600_000_000_000
    rows["times"] = 1_600_000_000_000_000_000 + hours + rng.integers(0, 10**9, len(hours))
    settings = {"linear_trend_timewise": [{"attr": a} for a in ("pvalue", "rvalue", "intercept", "slope", "stderr")],
                "mean": None}
    X, _, cols = check(rows, default_fc_parameters=settings)
    assert any("linear_trend_timewise" in c for c in cols)


def test_device_impute():
    rng = np.random.default_rng(5)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    rows["value"][rng.choice(len(rows["value"]), 20, replace=False)] = np.inf
    rows["value"][rng.choice(len(rows["value"]), 5, replace=False)] = -np.inf
    for fn in (impute, impute_dataframe_zero):
        X, _, _ = check(rows, default_fc_parameters=EfficientFCParameters(), impute_function=fn)
        assert bool(torch.isfinite(X).all())


def test_value_and_kind_code_dtypes():
    rng = np.random.default_rng(6)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    args = on_device(rows)
    s = EfficientFCParameters()

    def run(values, kind):
        return extract_features_long_device(args["ids"], values, args["sort"], kind, kinds=KINDS, default_fc_parameters=s)

    ref, ref_ids, ref_cols = run(args["values"], args["kind"])
    X, ids, cols = run(args["values"], args["kind"].to(torch.int32))
    assert_same(X, ref)
    assert torch.equal(ids, ref_ids) and cols == ref_cols
    v64 = torch.from_numpy(rng.standard_normal(len(rows["value"]))).to(DEV)
    assert_same(run(v64, args["kind"])[0], run(v64.to(torch.float32), args["kind"])[0])
    for dt in (torch.float16, torch.bfloat16):
        vl = v64.to(dt)
        assert_same(run(vl, args["kind"])[0], run(vl.to(torch.float32), args["kind"])[0])
    strided = torch.stack([args["values"], -args["values"]], 1)[:, 0]          # a non-contiguous view
    assert not strided.is_contiguous()
    assert_same(run(strided, args["kind"])[0], ref)


def test_empty_kinds_and_no_rows():
    rng = np.random.default_rng(7)
    rows = shuffled(rows_of(rng, {0: {1: 10, 2: 20}, 2: {2: 5, 3: 7}}), rng)         # kind "b" has no rows
    X, row_ids, cols = check(rows, default_fc_parameters=MinimalFCParameters())
    assert not any(c.startswith("b__") for c in cols)
    empty_i = torch.empty(0, dtype=torch.int64, device=DEV)
    X, row_ids, cols = extract_features_long_device(empty_i, torch.empty(0, device=DEV), empty_i, empty_i, kinds=KINDS)
    assert tuple(X.shape) == (0, 0) and row_ids.numel() == 0 and cols == []


def test_non_default_stream():
    rng = np.random.default_rng(8)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    args = on_device(rows)
    want, want_ids, _ = extract_features_long_device(args["ids"], args["values"], args["sort"], args["kind"], kinds=KINDS,
                                                     kind_to_fc_parameters=K2FC)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        values = args["values"] * 1.0            # written by a torch kernel on the side stream right before the call
        X, ids, _ = extract_features_long_device(args["ids"], values, args["sort"], args["kind"], kinds=KINDS,
                                                 kind_to_fc_parameters=K2FC)
        host, host_ids = X.cpu(), ids.cpu()
    side.synchronize()
    assert_same(host, want)
    assert torch.equal(host_ids, want_ids.cpu())


def test_errors_before_any_kernel_group():
    ctx = get_context(0)
    rng = np.random.default_rng(9)
    rows = shuffled(rows_of(rng, ragged_spec()), rng)
    args = on_device(rows)
    s = EfficientFCParameters()
    want, want_ids, _ = extract_features_long_device(args["ids"], args["values"], args["sort"], args["kind"], kinds=KINDS,
                                                     default_fc_parameters=s)

    def raises(match, **changed):
        a = dict(args, **changed)
        with pytest.raises(ValueError, match=match):
            extract_features_long_device(a["ids"], a["values"], a["sort"], a["kind"], kinds=KINDS, default_fc_parameters=s)
        assert ctx.launch_count() == 0 and ctx.last_kernels() == []
        X, ids, _ = extract_features_long_device(args["ids"], args["values"], args["sort"], args["kind"], kinds=KINDS,
                                                 default_fc_parameters=s)
        assert_same(X, want)
        assert torch.equal(ids, want_ids)
        assert ctx.launch_count() > 0

    for kind_of_nan in range(3):                 # a NaN value of any kind
        bad = args["values"].clone()
        bad[int(torch.nonzero(args["kind"] == kind_of_nan)[-1])] = float("nan")
        raises("value column contains NaN", values=bad)
    fsort = args["sort"].to(torch.float64)
    fsort[17] = float("nan")
    raises("sort keys contain NaN", sort=fsort)
    for code in (3, -1):
        bad = args["kind"].clone()
        bad[5] = code
        raises(r"kind code is outside 0 \.\. 2", kind=bad)
    n = 131_073                                  # one series past the spectral group's limit
    long_ids = torch.cat([args["ids"], torch.full((n,), 555, dtype=torch.int64, device=DEV)])
    raises("exceeds", ids=long_ids, values=torch.cat([args["values"], torch.zeros(n, device=DEV)]),
           sort=torch.cat([args["sort"], torch.arange(n, device=DEV)]),
           kind=torch.cat([args["kind"], torch.ones(n, dtype=torch.int64, device=DEV)]))
    with pytest.raises(ValueError, match="kind has 3 rows, ids"):          # refused before the library is called
        extract_features_long_device(args["ids"], args["values"], args["sort"], args["kind"][:3], kinds=KINDS)
