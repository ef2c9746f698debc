"""DeviceExtractor on CUDA tensors: bit for bit against extract_features_device on the same data, asynchronous on the
current stream, replayable from a CUDA graph, and with the input errors reported by check() instead of the call."""
import re

import numpy as np
import pytest

from oracle.extract import compare, oracle_rows
from tsfresh_b200 import ComprehensiveFCParameters, DeviceExtractor, EfficientFCParameters, extract_features_device
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)
COMP, EFF = ComprehensiveFCParameters(), EfficientFCParameters()


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


def eager(*args, **kw):
    return extract_features_device(*args, **kw)[0]


def batch(seed, shape, dtype=torch.float32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV, dtype=torch.float64).cumsum(1).to(dtype)


def views(seed, n, max_length, R):
    """n overlapping views on R values, the longest exactly max_length samples"""
    rng = np.random.default_rng(seed)
    length = rng.integers(1, max_length + 1, n)
    length[n // 2] = max_length
    begin = rng.integers(0, R - length + 1)
    return torch.from_numpy(begin).to(DEV), torch.from_numpy(length).to(DEV)


@pytest.mark.parametrize("settings", [COMP, EFF], ids=["comprehensive", "efficient"])
@pytest.mark.parametrize("L", [5, 256, 1000, 21000])
def test_dense_equals_extract_features_device(settings, L):
    n = 40 if L <= 1000 else 3
    ex = DeviceExtractor(n + 3, length=L, default_fc_parameters=settings)
    ex3 = DeviceExtractor(n + 3, length=L, kinds=["a", "b", "c"], default_fc_parameters=settings)
    for dtype in (torch.float32, torch.float64):
        x = batch(L, (n, L), dtype)
        X = ex(x)
        want, cols = extract_features_device(x, default_fc_parameters=settings)
        assert ex.columns == cols and X.dtype == torch.float64 and X.device == DEV
        assert_same(X, want)
        x3 = batch(L + 1, (n, L, 3), dtype)
        want3, cols3 = extract_features_device(x3, default_fc_parameters=settings, kinds=["a", "b", "c"])
        assert ex3.columns == cols3
        assert_same(ex3(x3), want3)
    ex.check()
    ex3.check()


@pytest.mark.parametrize("settings", [COMP, EFF], ids=["comprehensive", "efficient"])
def test_csr_longest_view_at_max_length_equals_extract_features_device(settings):
    R = 20_000
    v = batch(7, (1, R))[0]
    for M in (256, 1000):
        ex = DeviceExtractor(64, max_length=M, default_fc_parameters=settings)
        b, ln = views(M, 50, M, R)
        assert_same(ex(v, b, ln), eager(v, b, ln, default_fc_parameters=settings))
        assert_same(ex(v, b, ln.to(torch.int32)), eager(v, b, ln, default_fc_parameters=settings))
        ex2 = DeviceExtractor(64, max_length=M, kinds=["p", "q"], default_fc_parameters=settings)
        v2 = batch(8, (R, 2))
        assert_same(ex2(v2, b, ln), eager(v2, b, ln, default_fc_parameters=settings, kinds=["p", "q"]))
        ex.check()
        ex2.check()


def test_csr_shorter_views_than_max_length_match_the_oracle():
    rng = np.random.default_rng(11)
    lengths = np.array([1, 2, 3, 5, 17, 64, 100, 255, 256, 257, 300, 511], np.int64)
    host = rng.standard_normal(int(lengths.sum()) + 50).astype(np.float32)
    begin = np.concatenate([[0], np.cumsum(lengths)[:-1]]) + 20
    ex = DeviceExtractor(16, max_length=4000, default_fc_parameters=COMP)
    X = ex(torch.from_numpy(host).to(DEV), torch.from_numpy(begin).to(DEV), torch.from_numpy(lengths).to(DEV))
    ex.check()
    want = oracle_rows([host[b:b + n].astype(np.float64) for b, n in zip(begin, lengths)], COMP)
    assert not compare(X.cpu().numpy(), want, Plan(COMP).suffixes)


def test_call_does_not_block_the_host():
    ex = DeviceExtractor(512, length=256, default_fc_parameters=COMP)
    x = batch(3, (512, 256))
    want = eager(x)
    out = torch.empty((512, len(ex.columns)), dtype=torch.float64, device=DEV)
    ex(x, out=out)                               # modules loaded, stream bound
    torch.cuda.synchronize()
    out.fill_(0)
    torch.cuda._sleep(2_000_000_000)             # about a second on the current stream
    busy = torch.cuda.Event()
    busy.record()
    ex(x, out=out)
    still_busy = not busy.query()
    torch.cuda.synchronize()
    assert still_busy
    ex.check()
    assert_same(out, want)


def capture(fn):
    """fn() run once on a side stream, then captured in a graph"""
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(DEV).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def test_graph_replay_dense_and_csr():
    n, L = 300, 256
    ex = DeviceExtractor(n, length=L, default_fc_parameters=EFF)
    x_in = torch.zeros((n, L), device=DEV)
    x_out = torch.empty((n, len(ex.columns)), dtype=torch.float64, device=DEV)
    g = capture(lambda: ex(x_in, out=x_out))
    R, M = 30_000, 500
    exc = DeviceExtractor(n, max_length=M, default_fc_parameters=EFF)
    v_in, b_in, l_in = torch.zeros(R, device=DEV), torch.zeros(n, dtype=torch.int64, device=DEV), torch.ones(n, dtype=torch.int32, device=DEV)
    c_out = torch.empty((n, len(exc.columns)), dtype=torch.float64, device=DEV)
    gc = capture(lambda: exc(v_in, b_in, l_in, out=c_out))
    for seed in (21, 22):
        x = batch(seed, (n, L))
        x_in.copy_(x)
        g.replay()
        assert_same(x_out, eager(x, default_fc_parameters=EFF))
        v = batch(seed, (1, R))[0]
        b, ln = views(seed, n, M, R)
        v_in.copy_(v)
        b_in.copy_(b)
        l_in.copy_(ln)
        gc.replay()
        assert_same(c_out, eager(v, b, ln, default_fc_parameters=EFF))
    ex.check()
    exc.check()
    assert_same(ex(x), x_out)                    # an eager call on the extractor after its capture


def test_two_graphs_on_two_streams():
    n, L = 2000, 256
    exs = [DeviceExtractor(n, length=L, default_fc_parameters=s) for s in (COMP, EFF)]
    ins = [torch.zeros((n, L), device=DEV) for _ in exs]
    outs = [torch.empty((n, len(e.columns)), dtype=torch.float64, device=DEV) for e in exs]
    graphs = [capture(lambda e=e, i=i, o=o: e(i, out=o)) for e, i, o in zip(exs, ins, outs)]
    xs = [batch(30 + k, (n, L)) for k in range(2)]
    for i, x in zip(ins, xs):
        i.copy_(x)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(DEV) for _ in exs]
    for s, g in zip(streams, graphs):
        with torch.cuda.stream(s):
            g.replay()
    torch.cuda.synchronize()
    for e, o, x, s in zip(exs, outs, xs, (COMP, EFF)):
        e.check()
        assert_same(o, eager(x, default_fc_parameters=s))


def rows_equal_except(X, want, rejected):
    keep = [r for r in range(X.shape[0]) if r not in rejected]
    assert torch.isnan(X[rejected]).all()
    assert_same(X[keep], want)


def test_deferred_errors():
    n, L = 64, 256
    ex = DeviceExtractor(n, length=L, default_fc_parameters=COMP)
    x = batch(40, (n, L))
    bad = x.clone()
    bad[7, 100] = float("nan")
    X = ex(bad)                                  # returns without raising
    torch.cuda.synchronize()
    rows_equal_except(X, eager(x[torch.arange(n, device=DEV) != 7]), [7])
    with pytest.raises(ValueError, match="^Column must not contain NaN values: 0$"):
        eager(bad)
    with pytest.raises(ValueError, match=r"^Column must not contain NaN values: 0 \(first in series 7\)$"):
        ex.check()
    assert_same(ex(x), eager(x))
    ex.check()                                   # cleared, and the clean call reported nothing

    R, M = 20_000, 256
    exc = DeviceExtractor(n, max_length=M, kinds=["v"], default_fc_parameters=COMP)
    v = batch(41, (1, R))[0]
    b, ln = views(41, n, M, R)
    cases = [({3: (R - 10, 256)}, r"series 3 has an invalid \(begin, len\)"),
             ({10: (5, 0)}, r"series 10 has an invalid \(begin, len\)"),
             ({20: (100, M + 1)}, r"^series 20 is longer than max_length=256$"),
             ({3: (R - 10, 256), 10: (5, 0), 20: (100, M + 1)}, r"series 3 has an invalid \(begin, len\)")]
    for change, match in cases:
        bb, ll = b.clone(), ln.clone()
        for s, (b0, l0) in change.items():
            bb[s], ll[s] = b0, l0
        X = exc(v, bb, ll)
        keep = torch.tensor([r not in change for r in range(n)], device=DEV)
        rows_equal_except(X, eager(v, bb[keep], ll[keep], default_fc_parameters=COMP, kinds=["v"]), sorted(change))
        if "invalid" in match:
            with pytest.raises(ValueError) as e:
                eager(v, bb, ll, default_fc_parameters=COMP, kinds=["v"])
            assert re.search(match, str(e.value))           # the series the eager call names
        with pytest.raises(ValueError, match=match):
            exc.check()
        exc(v, b, ln)
        exc.check()
    for s in range(n):                           # a NaN that the view of max_length samples does not cover
        at = int(b[s]) + int(ln[s]) - 1
        covering = [r for r in range(n) if b[r] <= at < b[r] + ln[r]]
        if n // 2 not in covering:
            break
    nanv = v.clone()
    nanv[at] = float("nan")
    X = exc(nanv, b, ln)
    keep = torch.tensor([r not in covering for r in range(n)], device=DEV)
    rows_equal_except(X, eager(v, b[keep], ln[keep], default_fc_parameters=COMP, kinds=["v"]), covering)
    with pytest.raises(ValueError, match=r"^Column must not contain NaN values: v \(first in series %d\)$" % covering[0]):
        exc.check()


def test_deferred_errors_first_call_and_kind():
    """check() reports the first bad call since the last check(), and names the kind whose values held the NaN"""
    n, L = 32, 128
    ex = DeviceExtractor(n, length=L, kinds=["a", "b"], default_fc_parameters=EFF)
    x = batch(50, (n, L, 2))
    b1, b2 = x.clone(), x.clone()
    b1[5, 3, 1] = float("nan")
    b2[2, 3, 0] = float("nan")
    ex(x)
    ex(b1)
    ex(b2)
    with pytest.raises(ValueError, match=r"^Column must not contain NaN values: b \(first in series 5\)$"):
        ex.check()
    ex.check()


def test_graph_replayed_on_bad_data():
    n, L = 100, 256
    ex = DeviceExtractor(n, length=L, default_fc_parameters=EFF)
    x_in = torch.zeros((n, L), device=DEV)
    x_out = torch.empty((n, len(ex.columns)), dtype=torch.float64, device=DEV)
    g = capture(lambda: ex(x_in, out=x_out))
    ex.check()
    x = batch(60, (n, L))
    bad = x.clone()
    bad[7, 0] = float("nan")
    x_in.copy_(bad)
    g.replay()
    torch.cuda.synchronize()
    rows_equal_except(x_out, eager(x[torch.arange(n, device=DEV) != 7], default_fc_parameters=EFF), [7])
    with pytest.raises(ValueError, match=r"first in series 7\)$"):
        ex.check()
    x_in.copy_(x)
    g.replay()
    ex.check()
    assert_same(x_out, eager(x, default_fc_parameters=EFF))


def test_strided_out_keeps_the_other_columns():
    n, L = 50, 256
    ex = DeviceExtractor(n, length=L, default_fc_parameters=EFF)
    W = len(ex.columns)
    big = torch.full((n, W + 5), 7.0, dtype=torch.float64, device=DEV)
    bad = batch(70, (n, L))
    bad[9, 9] = float("nan")
    ex(bad, out=big[:, 2:2 + W])
    torch.cuda.synchronize()
    assert (big[:, :2] == 7).all() and (big[:, 2 + W:] == 7).all()
    assert torch.isnan(big[9, 2:2 + W]).all()
    with pytest.raises(ValueError, match="series 9"):
        ex.check()
