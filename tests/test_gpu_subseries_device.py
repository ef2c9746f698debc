"""extract_features_sub_device on long-format CUDA tensors: against the reference's add_sub_time_series_index +
extract_features answers (tests/golden/subseries.npz, oracle/make_golden_subseries.py), against the oracle on packages cut
in numpy, the kernel variants that packages select, a recording past the per-series length limit, its input options,
its errors (raised before any feature kernel runs) and its interplay with the rolled windows on one context."""
import json
import os

import numpy as np
import pandas as pd
import pytest

from oracle import make_golden_subseries as mk
from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from oracle.impute import impute as oracle_impute
from tsfresh_b200 import (ComprehensiveFCParameters, EfficientFCParameters, MinimalFCParameters, add_sub_time_series_index,
                          extract_features, extract_features_long_device, extract_features_rolled_device,
                          extract_features_sub_device, impute)
from tsfresh_b200.extraction import get_context
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda", 0)

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "subseries.npz"))
DOC = json.loads(str(Z["doc"]))
SETTINGS = {"comprehensive": ComprehensiveFCParameters, "efficient": EfficientFCParameters, "minimal": MinimalFCParameters}
MOMENTS = {"mean": None, "maximum": None, "minimum": None, "standard_deviation": None, "length": None, "skewness": None}


def bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64)
    return np.where(np.isnan(a), np.nan, a).view(np.int64)


def golden_rows(name):
    return mk.cases()[name][0]


def on_device(rows):
    return {c: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for c, v in rows.items()}


def cut(rows, sub_length, with_id=True):
    """numpy restatement of the packaging: {(package number, parent id): {kind code: float64 values}}, names ascending"""
    n = len(rows["value"])
    ids = rows["id"] if with_id else np.zeros(n, np.int64)
    key = rows["sort"] if rows.get("sort") is not None else np.arange(n)
    order = np.lexsort((key, ids, rows["kind"]))             # stable: equal keys keep their input order
    out = {}
    k, i, v = rows["kind"][order], ids[order], rows["value"][order].astype(np.float64)
    starts = np.flatnonzero(np.r_[True, (k[1:] != k[:-1]) | (i[1:] != i[:-1])])
    for s, e in zip(starts, np.r_[starts[1:], n]):
        for p, b in enumerate(range(s, e, sub_length)):
            out.setdefault((p, int(i[s])), {})[int(k[s])] = v[b:min(b + sub_length, e)]
    return dict(sorted(out.items()))


def expected(packages, kinds, plans_of):
    """the oracle's matrix for cut() packages: one column block per kind with rows, NaN where a kind has no package"""
    present = sorted({c for p in packages.values() for c in p})
    blocks, suffixes = [], []
    for c in present:
        settings = plans_of(kinds[c])
        names = list(packages)
        have = [j for j, name in enumerate(names) if c in packages[name]]
        width = len(Plan(settings).suffixes)
        block = np.full((len(names), width), np.nan)
        block[have] = oracle_rows([packages[names[j]][c] for j in have], settings)
        blocks.append(block)
        suffixes += Plan(settings).suffixes
    return np.concatenate(blocks, axis=1), suffixes


def assert_close(got, want, suffixes, packages=None):
    """compare()'s parity rule; packages of at most 5 samples (and exact integer inputs) get compare()'s noise floor"""
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape
    short = np.zeros(len(got), bool)
    if packages is not None:
        short = np.array([min(len(v) for v in p.values()) <= 5 for p in packages.values()])
    for rows, atol in ((~short, 0.0), (short, NOISE_FLOOR)):
        if rows.any():
            bad = compare(got[rows], want[rows], suffixes, atol=atol)
            assert not bad, bad[:5]


@pytest.mark.parametrize("name", sorted(DOC))
def test_reference_answers(name):
    d = DOC[name]
    rows = golden_rows(name)
    a = on_device(rows)
    settings = SETTINGS[d["settings"]]()
    kinds = d["kinds"]
    X, pnum, pid, cols = extract_features_sub_device(a["id"] if d["with_id"] else None, a["value"], a["sort"],
                                                     a["kind"] if len(kinds) > 1 else None, kinds=kinds,
                                                     sub_length=d["sub_length"], default_fc_parameters=settings)
    assert cols == d["columns"]
    assert pnum.dtype == torch.int64 and np.array_equal(pnum.cpu().numpy(), Z["%s/package" % name])
    if d["with_id"]:
        assert pid.dtype == torch.int64 and np.array_equal(pid.cpu().numpy(), Z["%s/parent" % name])
    else:
        assert pid is None
    want = Z["%s/X" % name]
    suffixes = [c.split("__", 1)[1] for c in cols]
    packages = cut(rows, d["sub_length"], d["with_id"])
    exact_inputs = bool(np.all(rows["value"] == np.round(rows["value"])))
    if exact_inputs:
        assert_close(X, want, suffixes, {k: {0: np.zeros(1)} for k in packages})
    else:
        assert_close(X, want, suffixes, packages)


@pytest.mark.parametrize("name", ["id_parameters", "sort_parameters", "ragged_7", "ragged_no_id_256"])
def test_host_drop_in_gives_the_reference_index(name):
    """extract_features(add_sub_time_series_index(df, ...), column_id="id") through this project"""
    d = DOC[name]
    rows = golden_rows(name)
    kinds = d["kinds"]
    df = pd.DataFrame({"value": rows["value"].astype(np.float64)})
    if d["with_id"]:
        df["ID"] = rows["id"]
    kind = "kind" if len(kinds) > 1 else None
    if kind:
        df["kind"] = np.asarray(kinds, dtype=object)[rows["kind"]]
    sort = None if rows["sort"] is None else "sort"
    if sort:
        df["sort"] = rows["sort"]
    data = add_sub_time_series_index(df, d["sub_length"], column_id="ID" if d["with_id"] else None, column_sort=sort,
                                     column_kind=kind)
    if d["with_id"]:
        data = data.drop(columns="ID")
    got = extract_features(data, column_id="id", column_sort=sort, column_kind=kind,
                           default_fc_parameters=SETTINGS[d["settings"]]())
    want_index = (list(zip(Z["%s/package" % name].tolist(), Z["%s/parent" % name].tolist())) if d["with_id"]
                  else Z["%s/package" % name].tolist())
    assert got.index.tolist() == want_index
    assert list(got.columns) == d["columns"]
    a = on_device(rows)
    X, _, _, _ = extract_features_sub_device(a["id"] if d["with_id"] else None, a["value"], a["sort"],
                                             a["kind"] if kind else None, kinds=kinds, sub_length=d["sub_length"],
                                             default_fc_parameters=SETTINGS[d["settings"]]())
    assert_close(X, got.to_numpy(), [c.split("__", 1)[1] for c in d["columns"]], cut(rows, d["sub_length"], d["with_id"]))


def random_rows(rng, spec, float_keys=False):
    """spec {kind code: {id: length}} -> rows, shuffled, distinct sort keys inside a series"""
    cols = {"id": [], "sort": [], "kind": [], "value": [], "time": []}
    for code, series in spec.items():
        for i, n in series.items():
            cols["id"].append(np.full(n, i, np.int64))
            keys = rng.permutation(n).astype(np.int64) * 7 - 1000
            cols["sort"].append(keys * 0.125 if float_keys else keys)
            cols["kind"].append(np.full(n, code, np.int64))
            cols["value"].append(rng.standard_normal(n).astype(np.float32))
            ticks = np.sort(rng.choice(10 ** 6, n, replace=False)).astype(np.int64)
            cols["time"].append(ticks[np.argsort(np.argsort(keys))] * 37_000_000_000)     # rising with the sort key
    rows = {c: np.concatenate(v) for c, v in cols.items()}
    p = rng.permutation(len(rows["id"]))
    return {c: v[p] for c, v in rows.items()}


KINDS = ["a", "b", "c"]
K2FC = {"a": ComprehensiveFCParameters(), "b": MinimalFCParameters(), "c": MOMENTS}


def spec_ragged():
    return {0: {-4: 300, 2: 77, 9: 1}, 1: {-4: 13, 5: 259, 9: 64}, 2: {2: 511, 5: 6, 1 << 50: 40}}


@pytest.mark.parametrize("sub_length", [1, 13, 64, 256, 1000])
def test_random_frames_against_the_oracle(sub_length):
    rng = np.random.default_rng(sub_length)
    rows = random_rows(rng, spec_ragged())
    a = on_device(rows)
    X, pnum, pid, cols = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], kinds=KINDS,
                                                     sub_length=sub_length, kind_to_fc_parameters=K2FC)
    packages = cut(rows, sub_length)
    assert list(zip(pnum.cpu().tolist(), pid.cpu().tolist())) == list(packages)
    want, suffixes = expected(packages, KINDS, K2FC.get)
    assert_close(X, want, suffixes, packages)
    # NaN blocks exactly where a kind has no package of that name
    widths = [len(Plan(K2FC[k]).suffixes) for k in KINDS]
    c0 = np.cumsum([0] + widths)
    nan_rows = np.isnan(X.cpu().numpy())
    for c in range(3):
        missing = np.array([c not in p for p in packages.values()])
        assert np.array_equal(nan_rows[:, c0[c]:c0[c + 1]].all(axis=1), missing)
    assert get_context(0).launch_count() > 0


def test_input_options():
    rng = np.random.default_rng(5)
    rows = random_rows(rng, spec_ragged(), float_keys=True)
    a = on_device(rows)
    settings = EfficientFCParameters()
    # float64 sort keys
    X, pnum, pid, cols = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], kinds=KINDS, sub_length=50,
                                                     default_fc_parameters=settings)
    packages = cut(rows, 50)
    assert list(zip(pnum.cpu().tolist(), pid.cpu().tolist())) == list(packages)
    want, suffixes = expected(packages, KINDS, lambda k: settings)
    assert_close(X, want, suffixes, packages)
    # ids=None: every kind is one series
    Xn, pn, pidn, _ = extract_features_sub_device(None, a["value"], a["sort"], a["kind"], kinds=KINDS, sub_length=50,
                                                  default_fc_parameters=settings)
    packages = cut(rows, 50, with_id=False)
    assert pidn is None and pn.cpu().tolist() == [p for p, _ in packages]
    want, suffixes = expected(packages, KINDS, lambda k: settings)
    assert_close(Xn, want, suffixes, packages)
    # sort=None: rows keep their input order
    Xs, ps, ids_s, _ = extract_features_sub_device(a["id"], a["value"], None, a["kind"], kinds=KINDS, sub_length=50,
                                                   default_fc_parameters=settings)
    packages = cut(dict(rows, sort=None), 50)
    assert list(zip(ps.cpu().tolist(), ids_s.cpu().tolist())) == list(packages)
    want, suffixes = expected(packages, KINDS, lambda k: settings)
    assert_close(Xs, want, suffixes, packages)
    # impute_function=impute: the imputed matrix of the plain one
    Xi, _, _, _ = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], kinds=KINDS, sub_length=50,
                                              default_fc_parameters=settings, impute_function=impute)
    assert np.array_equal(bits(Xi), bits(oracle_impute(X.cpu().numpy())))
    plain = pd.DataFrame(X.cpu().numpy())
    impute(plain)
    assert np.array_equal(bits(Xi), bits(plain.to_numpy()))
    # a side stream gives the same bits
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        Xd, pd_, idd, _ = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], kinds=KINDS,
                                                      sub_length=50, default_fc_parameters=settings)
    side.synchronize()
    assert np.array_equal(bits(Xd), bits(X)) and torch.equal(pd_, pnum) and torch.equal(idd, pid)


def test_times_give_linear_trend_timewise():
    rng = np.random.default_rng(6)
    rows = random_rows(rng, {0: {1: 200, 3: 45}, 1: {1: 90}})
    a = on_device(rows)
    settings = {"linear_trend_timewise": [{"attr": k} for k in ("pvalue", "rvalue", "intercept", "slope", "stderr")],
                "mean": None}
    X, pnum, pid, cols = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], kinds=["a", "b"],
                                                     times=a["time"], sub_length=32, default_fc_parameters=settings)
    assert any("linear_trend_timewise" in c for c in cols)
    at = cut(dict(rows, value=np.arange(len(rows["time"]))), 32)           # row numbers of every package
    timed = {name: {c: rows["time"][r.astype(np.int64)] for c, r in p.items()} for name, p in at.items()}
    packages = cut(rows, 32)
    blocks = []
    for c in range(2):
        names = [n for n in packages if c in packages[n]]
        block = np.full((len(packages), 6), np.nan)
        block[[list(packages).index(n) for n in names]] = oracle_rows(
            [packages[n][c] for n in names], settings, skip=(), times=[timed[n][c] for n in names])
        blocks.append(block)
    assert_close(X, np.concatenate(blocks, axis=1), [c.split("__", 1)[1] for c in cols], packages)


@pytest.mark.parametrize("sub_length, small", [(256, True), (1000, False)])
def test_kernel_variants_follow_the_package_length(sub_length, small):
    rng = np.random.default_rng(7)
    rows = random_rows(rng, {0: {i: 4_000 for i in range(8)}})
    a = on_device(rows)
    extract_features_sub_device(a["id"], a["value"], a["sort"], None, kinds=["v"], sub_length=sub_length,
                                default_fc_parameters=ComprehensiveFCParameters())
    kernels = get_context(0).last_kernels()
    for compact in ("entropy/rank-g1", "seq/small", "la/small", "peaks/small"):
        assert (compact in kernels) == small, kernels
    if not small:
        assert any(k.startswith("seq/general") for k in kernels), kernels


def test_long_recording():
    """two recordings of 1 000 000 samples: whole series are past the 131 072-sample limit, packages of 1 000 are not"""
    rng = np.random.default_rng(8)
    n = 1_000_000
    ids = torch.repeat_interleave(torch.tensor([3, 11], dtype=torch.int64, device=DEV), n)
    x = np.cumsum(rng.standard_normal(2 * n)).astype(np.float32)
    values = torch.from_numpy(x).to(DEV)
    sort = torch.arange(2 * n, dtype=torch.int64, device=DEV) % n
    settings = ComprehensiveFCParameters()
    X, pnum, pid, cols = extract_features_sub_device(ids, values, sort, sub_length=1_000, default_fc_parameters=settings)
    assert X.shape == (2_000, len(Plan(settings).suffixes))
    assert pnum.cpu().tolist() == [p for p in range(1_000) for _ in (3, 11)]
    assert pid.cpu().tolist() == [3, 11] * 1_000
    picks = [0, 1, 997, 1_998, 1_999]
    want = oracle_rows([x[(r % 2) * n + (r // 2) * 1_000:][:1_000].astype(np.float64) for r in picks], settings)
    bad = compare(X[picks].cpu().numpy(), want, Plan(settings).suffixes)
    assert not bad, bad[:5]
    with pytest.raises(ValueError, match="exceeds"):
        extract_features_long_device(ids, values, sort, default_fc_parameters=settings)


def test_errors_before_any_kernel_group():
    ctx = get_context(0)
    rng = np.random.default_rng(9)
    rows = random_rows(rng, spec_ragged())
    a = on_device(rows)
    kw = dict(kinds=KINDS, default_fc_parameters=EfficientFCParameters(), sub_length=40)
    want, want_n, want_ids, _ = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], **kw)

    def raises(error, match, **changed):
        """argument errors leave the context alone; data errors come from the staging calls, before any kernel group"""
        b = dict(a, **{k: v for k, v in changed.items() if k in a})
        args = dict(kw, **{k: v for k, v in changed.items() if k not in a})
        before = ctx.launch_count()
        with pytest.raises(error, match=match):
            extract_features_sub_device(b["id"], b["value"], b["sort"], b["kind"], **args)
        if error is ValueError:
            assert ctx.launch_count() == 0 and ctx.last_kernels() == []
        else:
            assert ctx.launch_count() == before > 0
        X, pn, ids, _ = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], **kw)
        assert np.array_equal(bits(X), bits(want))
        assert torch.equal(pn, want_n) and torch.equal(ids, want_ids)
        assert ctx.launch_count() > 0

    raises(ZeroDivisionError, "division", sub_length=0)
    raises(AssertionError, "positive integer", sub_length=-3)
    raises(AssertionError, "positive integer", sub_length=2.5)
    raises(TypeError, "unsupported operand", sub_length=None)
    bad = a["value"].clone()
    bad[int(torch.nonzero(a["kind"] == 1)[-1])] = float("nan")
    raises(ValueError, "value column contains NaN", value=bad)
    fsort = a["sort"].to(torch.float64)
    fsort[17] = float("nan")
    raises(ValueError, "sort keys contain NaN", sort=fsort)
    badk = a["kind"].clone()
    badk[5] = 3
    raises(ValueError, r"kind code is outside 0 \.\. 2", kind=badk)
    n = 25_000                                   # one package past sample_entropy's 21 000-sample limit
    raises(ValueError, "exceeds", sub_length=30_000, default_fc_parameters={"sample_entropy": None, "mean": None},
           id=torch.cat([a["id"], torch.full((n,), 555, dtype=torch.int64, device=DEV)]),
           value=torch.cat([a["value"], torch.zeros(n, device=DEV)]),
           sort=torch.cat([a["sort"], torch.arange(n, device=DEV)]),
           kind=torch.cat([a["kind"], torch.ones(n, dtype=torch.int64, device=DEV)]))


def test_determinism_and_rolls_between_packagings():
    rng = np.random.default_rng(10)
    rows = random_rows(rng, spec_ragged())
    a = on_device(rows)
    kw = dict(kinds=KINDS, default_fc_parameters=EfficientFCParameters())
    first = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], sub_length=33, **kw)
    again = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], sub_length=33, **kw)
    assert np.array_equal(bits(first[0]), bits(again[0]))
    assert torch.equal(first[1], again[1]) and torch.equal(first[2], again[2])
    rolled = extract_features_rolled_device(a["id"], a["value"], a["sort"], a["kind"], rolling_direction=5,
                                            max_timeshift=30, **kw)
    packaged = extract_features_sub_device(a["id"], a["value"], a["sort"], a["kind"], sub_length=33, **kw)
    rolled_again = extract_features_rolled_device(a["id"], a["value"], a["sort"], a["kind"], rolling_direction=5,
                                                  max_timeshift=30, **kw)
    assert np.array_equal(bits(packaged[0]), bits(first[0])) and torch.equal(packaged[1], first[1])
    assert np.array_equal(bits(rolled_again[0]), bits(rolled[0])) and torch.equal(rolled_again[2], rolled[2])
    packages = cut(rows, 33)
    want, suffixes = expected(packages, KINDS, lambda k: kw["default_fc_parameters"])
    assert_close(packaged[0], want, suffixes, packages)


def test_staged_calls_refuse_a_second_reshape():
    """the C calls: packaging after a roll (or twice), or rolling packages, is refused until the rows are staged again"""
    from tsfresh_b200 import _lib
    ctx = get_context(0)
    rng = np.random.default_rng(12)
    rows = random_rows(rng, {0: {1: 50, 2: 70}})
    a = on_device(rows)
    with ctx.lock:
        ctx.set_stream(_lib.STREAM_LEGACY)
        try:
            def stage():
                return ctx.stage_long_stacked(a["id"].data_ptr(), a["sort"].data_ptr(), False, a["value"].data_ptr(), 0,
                                              False, 1, 0, len(rows["id"]), keep_sort_keys=True)
            stage()
            assert ctx.sub_staged(16, 1)[0] == 9             # 4 + 5 packages of 16 rows
            for call in (lambda: ctx.sub_staged(16, 1), lambda: ctx.roll_staged(1, 5, 0, 1)):
                with pytest.raises(ValueError, match="no unrolled, unpackaged rows staged"):
                    call()
            stage()
            ctx.roll_staged(1, 5, 0, 1)
            with pytest.raises(ValueError, match="no unrolled, unpackaged rows staged"):
                ctx.sub_staged(16, 1)
            stage()
            with pytest.raises(ValueError, match="bad arguments"):
                ctx.sub_staged(0, 1)
        finally:
            ctx.set_stream(None)
