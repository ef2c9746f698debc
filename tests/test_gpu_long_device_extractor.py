"""DeviceLongExtractor on long-format CUDA tensors: bit for bit against extract_features_long_device on the same rows,
asynchronous on the current stream, replayable from a CUDA graph with a new row count, and with the data errors
reported by check() instead of the call."""
import numpy as np
import pytest

from oracle.extract import compare, oracle_rows
from tsfresh_b200 import (ComprehensiveFCParameters, DeviceLongExtractor, EfficientFCParameters, MinimalFCParameters,
                          extract_features_long_device)
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)
COMP, EFF = ComprehensiveFCParameters(), EfficientFCParameters()
MOMENTS = {"mean": None, "maximum": None, "minimum": None, "standard_deviation": None, "length": None, "skewness": None}
KINDS = ["a", "b", "c"]
K2FC = {"a": COMP, "b": MinimalFCParameters(), "c": MOMENTS}
PAD = (1 << 63) - 1
L = 300                                          # every kind's longest series in the bit-for-bit tests


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
    """spec {kind code: {id: length}} -> dict of row arrays in (kind, id, time) order, shuffled"""
    cols = {"id": [], "time": [], "kind": [], "value": []}
    for code, series in spec.items():
        for i, n in series.items():
            cols["id"].append(np.full(n, i, dtype=np.int64))
            cols["time"].append(np.arange(n, dtype=np.int64) * 5 - 40)
            cols["kind"].append(np.full(n, code, dtype=np.int64))
            cols["value"].append(rng.standard_normal(n).astype(np.float32))
    rows = {c: np.concatenate(v) for c, v in cols.items()}
    rows["ftime"] = (rows["time"] // 10).astype(np.float64) * 0.5        # float64 keys with ties
    p = rng.permutation(len(rows["id"]))
    return {c: v[p] for c, v in rows.items()}


def spec3(n_kinds=3):
    """negative, sparse and large ids, lengths 1 .. L, some ids missing from some kinds, every kind's longest L"""
    ids = [-(1 << 62), -5, 0, 3, 7, 1 << 40, 123456789012, 99]
    lens = [1, 2, 3, 100, 255, L, 17]
    spec = {k: {} for k in range(n_kinds)}
    for j, i in enumerate(ids):
        for k in range(n_kinds):
            if (j + k) % 4 != 3:
                spec[k][i] = lens[(j + 2 * k) % len(lens)]
    for k in range(n_kinds):
        spec[k][ids[k]] = L
    return spec


def tensors(rows, sort="time"):
    t = {c: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for c, v in rows.items()}
    return t["id"], t["value"], (t[sort] if sort else None), t["kind"]


def eager(rows, kinds=KINDS, sort="time", **kw):
    ids, values, s, kind = tensors(rows, sort)
    return extract_features_long_device(ids, values, s, kind, kinds=kinds, **kw)


def assert_rows(ex, got, want, n):
    """the extractor's (X, row_ids, n_ids) against an eager (X, row_ids, columns) over the kinds the eager call has"""
    X, row_ids, n_ids = got
    wX, wids, wcols = want
    assert int(n_ids) == n == wX.shape[0]
    assert row_ids[:n].tolist() == wids.tolist()
    assert (row_ids[n:] == PAD).all()
    keep = [ex.columns.index(c) for c in wcols]
    assert_same(X[:n, keep], wX)
    rest = [c for c in range(len(ex.columns)) if c not in keep]
    assert bool(torch.isnan(X[:n, rest]).all()) and bool(torch.isnan(X[n:]).all())


@pytest.mark.parametrize("sort", ["time", "ftime", None])
def test_three_kinds_equal_extract_features_long_device(sort):
    rng = np.random.default_rng(1)
    rows = rows_of(rng, spec3())
    want = eager(rows, sort=sort, kind_to_fc_parameters=K2FC)
    n = want[0].shape[0]
    ex = DeviceLongExtractor(len(rows["id"]) + 50, n + 5, L, kinds=KINDS, kind_to_fc_parameters=K2FC)
    assert ex.columns == want[2]
    got = ex(*tensors(rows, sort))
    assert got[0].shape == (n + 5, len(ex.columns)) and got[0].dtype == torch.float64
    assert_rows(ex, got, want, n)
    ids, values, s, kind = tensors(rows, sort)
    assert_rows(ex, ex(ids, values.double(), s, kind.to(torch.int32)), want, n)     # float64 values, int32 codes
    ex.check()


def test_one_kind_and_a_kind_without_rows():
    rng = np.random.default_rng(2)
    rows = rows_of(rng, {0: spec3()[0]})
    ex1 = DeviceLongExtractor(len(rows["id"]), 8, L, default_fc_parameters=COMP)
    ids, values, s, _ = tensors(rows)
    want = extract_features_long_device(ids, values, s, default_fc_parameters=COMP)
    assert_rows(ex1, ex1(ids, values, s), want, want[0].shape[0])
    for dt in (torch.float16, torch.bfloat16):
        v = values.to(dt)
        want = extract_features_long_device(ids, v, s, default_fc_parameters=COMP)
        assert_rows(ex1, ex1(ids, v, s), want, want[0].shape[0])
    ex1.check()
    spec = spec3()
    del spec[1]                                  # kind "b" has no rows: NaN columns, the others unchanged
    rows = rows_of(rng, spec)
    want = eager(rows, kind_to_fc_parameters=K2FC)
    assert not any(c.startswith("b__") for c in want[2])
    ex = DeviceLongExtractor(len(rows["id"]), 10, L, kinds=KINDS, kind_to_fc_parameters=K2FC)
    assert_rows(ex, ex(*tensors(rows)), want, want[0].shape[0])
    ex.check()


def test_shorter_series_match_the_oracle():
    rng = np.random.default_rng(3)
    lengths = [1, 2, 3, 5, 17, 64, 100, 255, 256, 257, 300, 511]
    rows = rows_of(rng, {0: {i * 7 - 20: n for i, n in enumerate(lengths)}})
    ex = DeviceLongExtractor(len(rows["id"]), 16, 4000, default_fc_parameters=COMP)
    X, row_ids, n_ids = ex(*tensors(rows)[:3])
    ex.check()
    n = int(n_ids)
    order = np.lexsort((rows["time"], rows["id"]))
    series = [rows["value"][order][rows["id"][order] == i].astype(np.float64) for i in row_ids[:n].tolist()]
    want = oracle_rows(series, COMP)
    assert not compare(X[:n].cpu().numpy(), want, Plan(COMP).suffixes)


def test_n_rows_equals_the_sliced_call():
    rng = np.random.default_rng(4)
    rows = rows_of(rng, spec3())
    ids, values, s, kind = tensors(rows)
    ex = DeviceLongExtractor(len(rows["id"]), 10, 4000, kinds=KINDS, kind_to_fc_parameters=K2FC)
    for m in (len(rows["id"]), len(rows["id"]) - 400, 37, 0):
        got = ex(ids, values, s, kind, n_rows=torch.tensor(m, device=DEV))
        X, row_ids, n_ids = [t.clone() for t in got]
        want = ex(ids[:m], values[:m], s[:m], kind[:m])
        assert int(n_ids) == int(want[2])
        assert torch.equal(row_ids, want[1])
        assert_same(X, want[0])
    ex.check()


def test_call_does_not_block_the_host():
    rng = np.random.default_rng(5)
    rows = rows_of(rng, spec3())
    ex = DeviceLongExtractor(len(rows["id"]), 10, L, kinds=KINDS, kind_to_fc_parameters=K2FC)
    args = tensors(rows)
    want = eager(rows, kind_to_fc_parameters=K2FC)
    out = torch.empty((10, len(ex.columns)), dtype=torch.float64, device=DEV)
    ex(*args, out=out)                           # modules loaded, stream bound
    torch.cuda.synchronize()
    out.fill_(0)
    torch.cuda._sleep(2_000_000_000)             # about a second on the current stream
    busy = torch.cuda.Event()
    busy.record()
    got = ex(*args, out=out)
    still_busy = not busy.query()
    torch.cuda.synchronize()
    assert still_busy
    ex.check()
    assert_rows(ex, got, want, want[0].shape[0])


def capture(fn):
    """fn() run once on a side stream, then captured in a graph; returns (graph, fn's result inside the graph)"""
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream(DEV).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = fn()
    return g, res


class Static:
    """static input tensors of a captured call, refilled with the first m rows of new data"""

    def __init__(self, max_rows, sort_dtype=torch.int64):
        self.ids = torch.zeros(max_rows, dtype=torch.int64, device=DEV)
        self.values = torch.zeros(max_rows, device=DEV)
        self.sort = torch.zeros(max_rows, dtype=sort_dtype, device=DEV)
        self.kind = torch.zeros(max_rows, dtype=torch.int64, device=DEV)
        self.n = torch.zeros((), dtype=torch.int64, device=DEV)

    def args(self):
        return self.ids, self.values, self.sort, self.kind

    def fill(self, ids, values, sort, kind):
        m = ids.shape[0]
        for dst, src in zip(self.args(), (ids, values, sort, kind)):
            dst[:m].copy_(src)
            dst[m:].fill_(7)                     # rows past n_rows do not count, whatever they hold
        self.n.fill_(m)


def test_graph_replay_with_new_rows_and_two_streams():
    specs = [spec3(), {k: {i: L - 3 * k - (i % 5) for i in range(-3, 30)} for k in range(3)}]
    for k in range(3):
        specs[1][k][5] = L
    max_rows = 40 * 3 * L
    exs = [DeviceLongExtractor(max_rows, 40, L, kinds=KINDS, kind_to_fc_parameters=K2FC),
           DeviceLongExtractor(max_rows, 40, L, kinds=KINDS, default_fc_parameters=EFF)]
    st = [Static(max_rows) for _ in exs]
    captured = [capture(lambda e=e, s=s: e(*s.args(), n_rows=s.n)) for e, s in zip(exs, st)]
    streams = [torch.cuda.Stream(DEV) for _ in exs]
    for seed, spec in enumerate(specs):
        rng = np.random.default_rng(60 + seed)
        rows = rows_of(rng, spec)
        assert len(rows["id"]) <= max_rows
        for s in st:
            s.fill(*tensors(rows))
        torch.cuda.synchronize()
        for stream, (g, _) in zip(streams, captured):
            with torch.cuda.stream(stream):
                g.replay()
        torch.cuda.synchronize()
        for ex, (_, got), kw in zip(exs, captured, ({"kind_to_fc_parameters": K2FC}, {"default_fc_parameters": EFF})):
            want = eager(rows, **kw)
            assert_rows(ex, got, want, want[0].shape[0])
            ex.check()


def drop(rows, keep):
    return {c: v[keep] for c, v in rows.items()}


def eager_error(rows, **kw):
    with pytest.raises(ValueError) as e:
        eager(rows, **kw)
    return type(e.value), str(e.value)


def test_deferred_errors():
    rng = np.random.default_rng(7)
    spec = spec3()
    rows = rows_of(rng, spec)
    n_all = len(rows["id"])
    ex = DeviceLongExtractor(n_all + 300, 9, L, kinds=KINDS, kind_to_fc_parameters=K2FC)
    good = eager(rows, kind_to_fc_parameters=K2FC)
    n = good[0].shape[0]

    def reports(exc, message):
        with pytest.raises(exc) as e:
            ex.check()
        assert str(e.value) == message
        ex.check()                               # cleared

    # a NaN value in the series (id 3, kind "c"): that series' cells NaN, every other cell as without the NaN
    sel = (rows["id"] == 3) & (rows["kind"] == 2)
    bad = {c: v.copy() for c, v in rows.items()}
    bad["value"][np.nonzero(sel)[0][-1]] = np.nan
    X, row_ids, n_ids = ex(*tensors(bad))
    r, c_cols = good[1].tolist().index(3), [j for j, c in enumerate(ex.columns) if c.startswith("c__")]
    want = good[0].clone()
    want[r, c_cols] = float("nan")
    assert_rows(ex, (X, row_ids, n_ids), (want, good[1], good[2]), n)
    reports(*eager_error(bad, kind_to_fc_parameters=K2FC))
    assert_rows(ex, ex(*tensors(rows)), good, n)
    ex.check()

    # kind "a"'s last series (its largest id, so the rows of the others keep their places) of L + 1 rows: its cells
    # NaN, every other cell as without it
    big = max(spec[0])
    longer = rows_of(rng, {**spec, 0: {**spec[0], big: L + 1}})
    sel = (longer["id"] == big) & (longer["kind"] == 0)
    assert_rows(ex, ex(*tensors(longer)), eager(drop(longer, ~sel), kind_to_fc_parameters=K2FC), n)
    too_long = "the series of id %d and kind 'a' is longer than max_length=%d" % (big, L)
    reports(ValueError, too_long)

    def rejected(got):
        X, row_ids, n_ids = got
        torch.cuda.synchronize()
        assert int(n_ids) == 0 and (row_ids == PAD).all() and bool(torch.isnan(X).all())

    # a NaN float64 sort key, a kind code out of range, more than max_ids ids: the whole call
    fbad = {c: v.copy() for c, v in rows.items()}
    fbad["ftime"][17] = np.nan
    rejected(ex(*tensors(fbad, "ftime")))
    reports(*eager_error(fbad, sort="ftime", kind_to_fc_parameters=K2FC))
    for code in (3, -1):
        kbad = {c: v.copy() for c, v in rows.items()}
        kbad["kind"][5] = code
        rejected(ex(*tensors(kbad)))
        reports(*eager_error(kbad, kind_to_fc_parameters=K2FC))
    more = rows_of(rng, {**spec, 1: {**spec[1], 1000: 4, 1001: 5}})     # 10 ids
    rejected(ex(*tensors(more)))
    reports(ValueError, "10 distinct ids, more than max_ids=9: id %d is the first past them" % sorted(set(more["id"]))[9])
    assert_rows(ex, ex(*tensors(rows)), good, n)
    ex.check()

    # the first bad call since the last check() is the one reported
    ex(*tensors(rows))
    ex(*tensors(longer))
    ex(*tensors(more))
    reports(ValueError, too_long)


def test_graph_replayed_on_bad_rows():
    rng = np.random.default_rng(8)
    rows = rows_of(rng, spec3())
    ex = DeviceLongExtractor(len(rows["id"]) + 10, 12, L, kinds=KINDS, kind_to_fc_parameters=K2FC)
    s = Static(len(rows["id"]) + 10)
    g, got = capture(lambda: ex(*s.args(), n_rows=s.n))
    ex.check()
    bad = {c: v.copy() for c, v in rows.items()}
    bad["kind"][3] = 5
    s.fill(*tensors(bad))
    g.replay()
    torch.cuda.synchronize()
    assert int(got[2]) == 0 and bool(torch.isnan(got[0]).all())
    with pytest.raises(ValueError, match=r"^tsfx_stage_long_stacked: a kind code is outside 0 \.\. 2$"):
        ex.check()
    s.fill(*tensors(rows))
    g.replay()
    ex.check()
    want = eager(rows, kind_to_fc_parameters=K2FC)
    assert_rows(ex, got, want, want[0].shape[0])
