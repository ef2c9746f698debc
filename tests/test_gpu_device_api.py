"""extract_features_device on CUDA tensors, bit for bit against the host paths on the same float32 data (both run the
same kernels), plus its stream contract and the errors its checked pass raises before any kernel group runs."""
import numpy as np
import pandas as pd
import pytest

from tsfresh_b200 import (ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters, extract_features,
                          extract_features_device, impute, impute_dataframe_zero, roll_time_series)
from tsfresh_b200._lib import DevicePlan, kernel_variants
from tsfresh_b200.extraction import get_context
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)

MOMENTS = {"mean": None, "maximum": None, "minimum": None, "standard_deviation": None, "length": None,
           "skewness": None}                     # every calculator in k_moments: the plan writes the result directly
SEEN = set()                                     # kernel variants the calls of this module ran


def run(*args, **kw):
    X, cols = extract_features_device(*args, **kw)
    SEEN.update(get_context(0).last_kernels())
    return X, cols


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


def long_frame(x):
    n, L = x.shape
    return pd.DataFrame({"id": np.repeat(np.arange(n), L), "time": np.tile(np.arange(L), n), "value": x.reshape(-1)})


def test_comprehensive_dense_equals_extract_features():
    x = np.random.default_rng(1).standard_normal((1000, 256)).astype(np.float32)
    X, cols = run(torch.from_numpy(x).to(DEV), kinds=["value"])
    want = extract_features(long_frame(x), column_id="id", column_sort="time")
    assert cols == list(want.columns)
    assert X.dtype == torch.float64 and X.device == DEV and tuple(X.shape) == want.shape
    assert_same(X, want.to_numpy())


def test_csr_views_of_many_lengths():
    rng = np.random.default_rng(2)
    lengths = [1, 2, 3, 4, 5, 33, 255, 257, 1300, 21000, 3, 257]
    gap = 7
    R = sum(lengths) + gap * (len(lengths) + 1)
    host = rng.standard_normal(R).astype(np.float32)
    begin, pos = [], gap
    for n in lengths:
        begin.append(pos)
        pos += n + gap
    begin += [begin[7] + 100, begin[9] + 5]      # overlapping views
    lengths += [600, 20000]
    begin, lengths = np.array(begin, np.int64), np.array(lengths, np.int64)
    dev_vals = torch.from_numpy(host).to(DEV)
    dev_vals[begin[0] - 3] = float("nan")        # a NaN no view covers is not read, so not an error
    b, ln = torch.from_numpy(begin).to(DEV), torch.from_numpy(lengths).to(DEV)
    for settings in (ComprehensiveFCParameters(), MOMENTS):
        X, cols = run(dev_vals, b, ln, default_fc_parameters=settings, kinds=["x"])
        plan = Plan(settings)
        assert cols == ["x__" + s for s in plan.suffixes]
        want = DevicePlan(get_context(0), plan).extract_csr(host, begin, lengths.astype(np.int32))
        assert_same(X, want)
    X32, _ = run(dev_vals, b, ln.to(torch.int32), default_fc_parameters=MOMENTS, kinds=["x"])
    assert_same(X32, X)


def test_rolled_windows_as_views():
    rng = np.random.default_rng(3)
    lens = [300, 700, 40]
    df = pd.DataFrame({"id": np.repeat(np.arange(3), lens), "time": np.concatenate([np.arange(n) for n in lens]),
                       "value": rng.standard_normal(sum(lens)).astype(np.float32)})
    rolled = roll_time_series(df, column_id="id", column_sort="time", max_timeshift=255, min_timeshift=0)
    want = extract_features(rolled, default_fc_parameters=EfficientFCParameters())
    X, cols = run(torch.from_numpy(rolled.values["value"]).to(DEV), torch.from_numpy(rolled.begin).to(DEV),
                  torch.from_numpy(rolled.length).to(DEV), default_fc_parameters=EfficientFCParameters(),
                  kinds=["value"])
    assert cols == list(want.columns) and X.shape[0] == len(rolled) == want.shape[0]
    assert_same(X, want.to_numpy())


def test_channels_last_kinds_with_their_own_plans():
    rng = np.random.default_rng(4)
    N, L = 300, 128
    x = rng.standard_normal((N, L, 3)).astype(np.float32)
    k2fc = {"a": MinimalFCParameters(), "b": MOMENTS, "c": EfficientFCParameters()}
    X, cols = run(torch.from_numpy(x).to(DEV), kinds=["a", "b", "c"], kind_to_fc_parameters=k2fc)
    wide = pd.DataFrame({"id": np.repeat(np.arange(N), L), "t": np.tile(np.arange(L), N),
                         "a": x[:, :, 0].reshape(-1), "b": x[:, :, 1].reshape(-1), "c": x[:, :, 2].reshape(-1)})
    want = extract_features(wide, column_id="id", column_sort="t", kind_to_fc_parameters=k2fc)
    assert cols == list(want.columns)
    # k_moments sums dense rows in its own order ("moments/dense"): the long frame (CSR rows) agrees to rounding, the
    # host dense path bit for bit
    np.testing.assert_allclose(X.cpu().numpy(), want.to_numpy(), rtol=1e-10, atol=1e-12)
    c0 = 0
    for k, kind in enumerate("abc"):
        host = DevicePlan(get_context(0), Plan(k2fc[kind])).extract_dense(np.ascontiguousarray(x[:, :, k]))
        assert_same(X[:, c0:c0 + host.shape[1]], host)
        c0 += host.shape[1]
    assert c0 == X.shape[1]
    # default kinds are 0 .. K-1, like the column labels of a wide frame without names
    X0, cols0 = run(torch.from_numpy(x).to(DEV), default_fc_parameters=MOMENTS)
    assert cols0 == ["%d__%s" % (k, s) for k in range(3) for s in Plan(MOMENTS).suffixes]


def test_dtypes_and_layouts():
    rng = np.random.default_rng(5)
    x64 = torch.from_numpy(rng.standard_normal((64, 200))).to(DEV)
    s = EfficientFCParameters()
    ref, _ = run(x64.to(torch.float32), default_fc_parameters=s)
    assert_same(run(x64, default_fc_parameters=s)[0], ref)                  # float64 -> float32 on the device
    for dt in (torch.float16, torch.bfloat16):
        xl = x64.to(dt)
        assert_same(run(xl, default_fc_parameters=s)[0], run(xl.to(torch.float32), default_fc_parameters=s)[0])
    t = x64.to(torch.float32).t().contiguous().t()                          # column-major storage
    assert not t.is_contiguous()
    assert_same(run(t, default_fc_parameters=s)[0], ref)
    wide = torch.from_numpy(rng.standard_normal((64, 450)).astype(np.float32)).to(DEV)
    sl = wide[:, 50:450:2]
    assert_same(run(sl, default_fc_parameters=s)[0], run(sl.contiguous(), default_fc_parameters=s)[0])
    vals = x64.to(torch.float32).reshape(-1)
    begin = torch.arange(64, device=DEV, dtype=torch.int64) * 200
    length = torch.full((64,), 200, device=DEV, dtype=torch.int64)
    assert_same(run(vals.to(torch.float16), begin, length, default_fc_parameters=s)[0],
                run(vals.to(torch.float16).to(torch.float32), begin, length, default_fc_parameters=s)[0])
    two = torch.stack([vals, -vals], 1)                                     # [R, 2] CSR kinds
    X2, cols2 = run(two, begin, length, default_fc_parameters=s, kinds=["p", "q"])
    F = len(cols2) // 2
    assert_same(X2[:, :F], run(vals, begin, length, default_fc_parameters=s)[0])
    assert_same(X2[:, F:], run(-vals, begin, length, default_fc_parameters=s)[0])


def test_out_column_slice():
    rng = np.random.default_rng(6)
    x = torch.from_numpy(rng.standard_normal((100, 256, 2)).astype(np.float32)).to(DEV)
    # the second case is one plan that writes the result directly (k_moments), into a strided slice
    for xs, k2fc in ((x, {0: EfficientFCParameters(), 1: MOMENTS}), (x[..., :1], {0: MOMENTS})):
        want, cols = run(xs, kind_to_fc_parameters=k2fc)
        W = len(cols)
        big = torch.full((100, W + 9), -123.0, dtype=torch.float64, device=DEV)
        X, _ = run(xs, kind_to_fc_parameters=k2fc, out=big[:, 4:4 + W])
        assert X.data_ptr() == big.data_ptr() + 4 * 8 and X.stride() == (W + 9, 1)
        assert_same(big[:, 4:4 + W], want)
        assert bool((big[:, :4] == -123.0).all()) and bool((big[:, 4 + W:] == -123.0).all())


def test_impute_on_the_device():
    rng = np.random.default_rng(7)
    x = rng.standard_normal((200, 128)).astype(np.float32)
    x[3, 10] = np.inf
    x[17, :] = np.inf
    x[40, 5] = -np.inf
    xd = torch.from_numpy(x).to(DEV)
    s = EfficientFCParameters()
    raw, cols = run(xd, default_fc_parameters=s)
    assert not bool(torch.isfinite(raw).all())
    for fn in (impute, impute_dataframe_zero):
        df = pd.DataFrame(raw.cpu().numpy(), columns=cols)
        fn(df)
        got, _ = run(xd, default_fc_parameters=s, impute_function=fn)
        assert_same(got, df.to_numpy())
        big = torch.full((200, len(cols) + 3), 5.0, dtype=torch.float64, device=DEV)
        run(xd, default_fc_parameters=s, impute_function=fn, out=big[:, 1:1 + len(cols)])
        assert_same(big[:, 1:1 + len(cols)], df.to_numpy())
        assert bool((big[:, 0] == 5.0).all()) and bool((big[:, -2:] == 5.0).all())
    # any other callable gets the host DataFrame, as extract_features does
    got, _ = run(xd, default_fc_parameters=s, impute_function=lambda d: d.fillna(-1.0, inplace=True))
    want = raw.cpu().numpy().copy()
    want[np.isnan(want)] = -1.0
    assert_same(got, want)


def test_benford_with_infinite_samples():
    """the reference maps +-inf to +-DBL_MAX (np.nan_to_num) before taking leading digits: digit 1"""
    from oracle.extract import compare, oracle_rows
    rng = np.random.default_rng(10)
    x = rng.standard_normal((4, 50)).astype(np.float32)
    x[0, 3], x[1, :], x[2, [4, 9]] = np.inf, np.inf, [-np.inf, np.inf]
    settings = {"benford_correlation": None}
    X, _ = run(torch.from_numpy(x).to(DEV), default_fc_parameters=settings)
    want = oracle_rows([s.astype(np.float64) for s in x], settings)
    assert not compare(X.cpu().numpy(), want, Plan(settings).suffixes)


def test_stream_ordering():
    """The call runs on torch's current stream: with the default stream held busy by a sleeping kernel, a call on a
    side stream completes while the sleep has not finished, so the call neither enqueued work behind the sleep that it
    waited for nor waited for the default stream itself."""
    rng = np.random.default_rng(8)
    src = torch.from_numpy(rng.standard_normal((200, 256)).astype(np.float32)).to(DEV)
    want, _ = run(src)                           # context, plans and scratch exist: the timed call allocates nothing
    side = torch.cuda.Stream(DEV)
    with torch.cuda.stream(side):                # same for torch's cache of side-stream blocks (an allocation would
        run(src * 1.0)[0].cpu()                  # synchronise the device)
    torch.cuda.synchronize()
    default = torch.cuda.default_stream(DEV)
    with torch.cuda.stream(default):
        torch.cuda._sleep(2_000_000_000)         # about a second
        busy = torch.cuda.Event()
        busy.record(default)
    with torch.cuda.stream(side):
        values = src * 1.0                       # written by a torch kernel on the side stream right before the call
        X, _ = run(values)
        host = X.cpu()
    side.synchronize()
    still_busy = not busy.query()
    torch.cuda.synchronize()
    assert still_busy
    assert_same(host, want)
    with torch.cuda.stream(default):             # the context is rebound to the default stream: same bits
        assert_same(run(src)[0], want)


def test_errors_before_any_kernel_group():
    ctx = get_context(0)
    rng = np.random.default_rng(9)
    x = torch.from_numpy(rng.standard_normal((100, 256)).astype(np.float32)).to(DEV)
    s = EfficientFCParameters()

    def raises(exc, match, *args, **kw):
        run(x, default_fc_parameters=s)
        assert ctx.launch_count() > 0
        with pytest.raises(exc, match=match):
            extract_features_device(*args, **kw)
        assert ctx.launch_count() == 0 and ctx.last_kernels() == []

    bad = x.clone()
    bad[57, 100] = float("nan")
    raises(ValueError, "^Column must not contain NaN values: 0$", bad, default_fc_parameters=s)
    vals = x.reshape(-1)
    R = vals.numel()
    begin = torch.arange(50, device=DEV, dtype=torch.int64) * 300
    length = torch.full((50,), 256, device=DEV, dtype=torch.int32)
    for field, value, series in (("begin", R - 100, 17), ("length", 0, 23), ("begin", -1, 31)):
        b, ln = begin.clone(), length.clone()
        (b if field == "begin" else ln)[series] = value
        raises(ValueError, r"series %d has an invalid \(begin, len\)" % series, vals, b, ln, default_fc_parameters=s)
    nanv = vals.clone()
    nanv[int(begin[8]) + 255] = float("nan")
    raises(ValueError, "^Column must not contain NaN values: 0$", nanv, begin, length, default_fc_parameters=s)
    long = torch.zeros(131_073 + 200, device=DEV)
    raises(ValueError, "exceeds", long, torch.tensor([0, 100, 131_173], device=DEV),
           torch.tensor([100, 131_073, 100], device=DEV), default_fc_parameters=s)
    with pytest.raises(ValueError, match="CUDA tensor"):
        extract_features_device(x.cpu(), default_fc_parameters=s)
    with pytest.raises(ValueError, match="begin is on cpu"):
        extract_features_device(vals, begin.cpu(), length, default_fc_parameters=s)
    W = len(Plan(s).suffixes)
    with pytest.raises(ValueError, match="out is on cpu"):
        extract_features_device(x, default_fc_parameters=s, out=torch.empty((100, W), dtype=torch.float64))
    with pytest.raises(TypeError):
        extract_features_device(x.cpu().numpy(), default_fc_parameters=s)


def test_variant_ledger():
    if not SEEN:
        pytest.skip("no call of this module ran")
    assert SEEN <= set(kernel_variants()), SEEN - set(kernel_variants())
    assert {"basic/w12/shared", "moments/general"} <= SEEN, sorted(SEEN)
    assert any(k.endswith("/global") for k in SEEN), sorted(SEEN)
