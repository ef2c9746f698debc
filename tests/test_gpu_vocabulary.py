"""The parameter values beyond the Comprehensive grid on the GPU, against the oracle, in every kernel variant that runs
them: the numpy f_agg of agg_autocorrelation (BASIC) and change_quantiles (SORTED), linregress attr "intercept_stderr"
(BASIC), and augmented_dickey_fuller with autolag "t-stat" and case-insensitive names (LA, the compact kernel and every
general geometry up to the three-round autolag of the longest series).

Comparison rules (oracle/extract.py:compare): usedlag and the max / min of change_quantiles bit-exact (they select one
value; a difference of two float32 samples is exact in float64 on these data), everything else rtol 1e-5 with NaN equal
to NaN, and NOISE_FLOOR on the degenerate rows.  One waiver: where the oracle's |t| of a model between the two lags lies
within 1e-9 relative of the 1.6449 stop value, the t-stat search may stop at either side; the statistic is then compared
with the oracle's at the lag the kernel chose, and the test prints how many rows used the waiver.  The same-bits check:
the new columns appended to a plan leave the plan's own columns untouched.  The ledger at the end: every variant named
above ran (the SORTED global region in a process with TSFX_GLOBAL_ABOVE=1)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from tests.helpers import to_csr
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu

AGGS = ("mean", "median", "var", "std", "max", "amax", "min", "amin", "ptp", "sum", "prod", "average",
        "nanmean", "nanmedian", "nanvar", "nanstd", "nanmax", "nanmin", "nansum", "nanprod")
EXACT_CQ = ('f_agg_"max"', 'f_agg_"min"', 'f_agg_"amax"', 'f_agg_"amin"', 'f_agg_"nanmax"', 'f_agg_"nanmin"')
REACHED = set()
WAIVED = []
STOP = 1.6448536269514722


def settings(group, n):
    if group in ("basic", "basic_light"):     # light: no lag past the grid's 40, so that 12 warps share a CTA
        lags = (1, 5, 40) if group == "basic_light" else (1, 5, 40, min(n, 300))
        return {"agg_autocorrelation": [{"f_agg": f, "maxlag": m} for f in AGGS for m in lags]
                + [{"f_agg": f, "maxlag": 0} for f in ("mean", "sum", "prod", "nansum", "nanprod", "median", "nanvar")],
                "linear_trend": [{"attr": a} for a in ("intercept_stderr", "stderr", "slope")],
                "agg_linear_trend": [{"attr": "intercept_stderr", "chunk_len": c, "f_agg": f} for c in (5, 50)
                                     for f in ("max", "mean")]}
    if group == "sorted":
        return {"change_quantiles": [{"ql": ql, "qh": qh, "isabs": b, "f_agg": f}
                                     for ql, qh in ((0.0, 0.2), (0.2, 0.8), (0.4, 0.9), (0.8, 0.6)) for b in (False, True)
                                     for f in AGGS],
                "median": None}
    if group == "la":
        return {"augmented_dickey_fuller": [{"attr": a, "autolag": al} for al in ("t-stat", "aic", "Bic", "t-stats")
                                            for a in ("teststat", "pvalue", "usedlag")]}
    raise KeyError(group)


def _rng(n, seed, walk):
    x = np.random.default_rng(seed).standard_normal(n)
    return (x.cumsum() if walk else x).astype(np.float32)


def level_series(n, seed):
    """level + spread * z: a large level next to small changes"""
    return (1000.0 + 0.01 * np.random.default_rng(seed).standard_normal(n)).astype(np.float32)


def call_series(n, seed):
    """(series, degenerate flags): a random and a walk of n samples, a level series, short and constant ones"""
    s = [_rng(n, seed, False), _rng(n, seed + 1, True), level_series(n, seed + 2)]
    deg = [False, False, False]
    for m in (1, 2, 3, 5, 33):
        s.append(_rng(m, seed + m, False))
        deg.append(True)
    s.append(np.full(40, 2.5, np.float32))
    deg.append(True)
    inf = _rng(60, seed + 7, False)
    inf[[10, 11, 30, 31]] = [np.inf, -np.inf, np.inf, np.inf]
    s.append(inf)
    deg.append(True)
    return s, deg


# (group, longest series, dense, variant the call must run)
CASES = [("basic_light", 300, False, "basic/w12/shared"), ("basic", 300, False, "basic/w4/shared"), ("basic", 700, False, "basic/w4/shared"),
         ("basic", 1500, False, "basic/w2/shared"), ("basic", 5000, False, "basic/w1/shared"),
         ("basic", 12000, False, "basic/w4/global"), ("basic", 1024, True, "basic/w2/shared"),
         ("sorted", 300, False, "sorted/w8/shared"), ("sorted", 1500, False, "sorted/w4/shared"),
         ("sorted", 3000, False, "sorted/w2/shared"), ("sorted", 5000, False, "sorted/w1/shared"),
         ("sorted", 24001, False, "sorted/w1/shared"), ("sorted", 1000, True, "sorted/w8/shared"),
         ("la", 200, False, "la/small"), ("la", 256, True, "la/small"), ("la", 300, False, "la/w8/shared"),
         ("la", 700, False, "la/w4/shared"), ("la", 1500, False, "la/w2/shared"), ("la", 5000, False, "la/w1/shared"),
         ("la", 12000, False, "la/w4/global"), ("la", 71260, False, "la/w4/global"), ("la", 131072, False, "la/w4/global")]


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def extract(ctx, st, series, dense):
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(st))
    try:
        got = dp.extract_dense(np.stack(series)) if dense else dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
    return got, kernels


def check(got, want, suffixes, degenerate):
    bad = []
    for r in range(got.shape[0]):
        atol = NOISE_FLOOR if degenerate[r] else 0.0
        bad += [(r,) + b[1:] for b in compare(got[r:r + 1], want[r:r + 1], suffixes, atol=atol)]
    for c, suf in enumerate(suffixes):           # bit-exact: the selecting reducers of change_quantiles
        if suf.startswith("change_quantiles") and any(k in suf for k in EXACT_CQ):
            g, w = got[:, c], want[:, c]
            for r in np.nonzero(~((g == w) | (np.isnan(g) & np.isnan(w))))[0]:
                bad.append((int(r), suf, float(g[r]), float(w[r])))
    return bad


@pytest.mark.parametrize("group,n,dense,variant", CASES, ids=["%s_%d%s" % (g, n, "_dense" if d else "") for g, n, d, _ in CASES])
def test_vocabulary(ctx, group, n, dense, variant):
    st = settings(group, n)
    if dense:
        series = [_rng(n, n, False), _rng(n, n + 1, True), level_series(n, n + 2), np.full(n, 2.5, np.float32)]
        degenerate = [False, False, False, True]
    elif n > 20000:
        series, degenerate = [_rng(n, n, True), level_series(n, n + 2)], [False, False]
    else:
        series, degenerate = call_series(n, n)
    if group.startswith("basic"):   # statsmodels' acf raises on inf: the reference's agg_autocorrelation has no value there
        keep = [i for i, s in enumerate(series) if np.isfinite(s).all()]
        series, degenerate = [series[i] for i in keep], [degenerate[i] for i in keep]
    got, kernels = extract(ctx, st, series, dense)
    REACHED.update(kernels)
    assert variant in kernels, kernels
    want = oracle_rows([s.astype(np.float64) for s in series], st)
    bad = check(got, want, Plan(st).suffixes, degenerate)
    if group == "la":
        bad = _tstat_waiver(bad, got, Plan(st).suffixes, series)
    assert not bad, "\n".join("row %d %s: gpu=%r oracle=%r" % b for b in bad[:40]) + "\n(%d mismatches)" % len(bad)


# ---------------------------------------------------------------------------------------------- t-stat waiver
def _adf_design(x, lags):
    """adfuller's design with `lags` lagged differences: (y, [const, level, dlag1..])"""
    from oracle import thirdparty as tp
    d = np.diff(x)
    xdall = tp._lagmat_both_in(d, lags)
    nobs = xdall.shape[0]
    xdall[:, 0] = x[-nobs - 1: -1]
    return d[-nobs:], np.column_stack([np.ones(nobs), xdall])


def _model_t(x):
    """|t| of the last regressor of every model of the oracle's t-stat search, by lag count"""
    from oracle import thirdparty as tp
    n = len(x)
    maxlag = min(n // 2 - 2, int(np.ceil(12.0 * np.power(n / 100.0, 1 / 4.0))))
    y, full = _adf_design(x, maxlag)
    out = {}
    for ncol in range(2 + maxlag, 2, -1):
        beta, ssr, xtxi = tp._ols(y, full[:, :ncol])
        out[ncol - 2] = abs(beta[-1] / np.sqrt(ssr / (len(y) - ncol) * xtxi[-1, -1]))
    return out


def _stat_at(x, lag):
    """the oracle's teststat with usedlag forced to `lag`"""
    from oracle import thirdparty as tp
    y, full = _adf_design(x, lag)
    X = np.column_stack([full[:, 1:], np.ones(len(y))])
    beta, ssr, xtxi = tp._ols(y, X)
    return beta[0] / np.sqrt(ssr / (len(y) - X.shape[1]) * xtxi[0, 0])


def _tstat_waiver(bad, got, suffixes, series):
    """drops the t-stat mismatches of rows whose search decided within 1e-9 relative of the stop value, where the kernel's
    lag is the other side of that decision and its statistic matches the oracle's at that lag"""
    col = {s: c for c, s in enumerate(suffixes)}
    rows = {r for r, suf, _, _ in bad if 'autolag_"t-stat"' in suf}
    waived = set()
    for r in rows:
        x = np.asarray(series[r], np.float64)
        if x.max() == x.min():
            continue
        lag = int(got[r, col['augmented_dickey_fuller__attr_"usedlag"__autolag_"t-stat"']])
        ts = _model_t(x)
        want = next((k for k in sorted(ts, reverse=True) if ts[k] >= STOP), 0)
        lo, hi = min(lag, want), max(lag, want)
        near = any(abs(ts[k] / STOP - 1.0) <= 1e-9 for k in ts if lo <= k <= hi)
        stat = got[r, col['augmented_dickey_fuller__attr_"teststat"__autolag_"t-stat"']]
        if near and np.isclose(stat, _stat_at(x, lag), rtol=1e-5, atol=0):
            waived.add(r)
    WAIVED.extend(waived)
    if waived:
        print("t-stat waiver used on %d rows" % len(waived))
    return [b for b in bad if not (b[0] in waived and 'autolag_"t-stat"' in b[1])]


def test_same_bits_with_new_columns_appended(ctx):
    """today's grid alone, and the same plan with the new columns after it: identical values in the shared columns"""
    from tsfresh_b200.settings import ComprehensiveFCParameters
    base = dict(ComprehensiveFCParameters())
    more = dict(base)
    for g in ("basic", "sorted", "la"):
        # maxlag 40 at most: a longer lag than the grid's would change how the lag products are formed (tensor cores up
        # to lag 63), and with them the bits of the grid's autocorrelation columns
        for k, v in settings(g, 40).items():
            more[k] = list(more.get(k) or []) + list(v or []) if v is not None else more.get(k)
    for n in (200, 1000):
        series, _ = call_series(n, 3 * n)
        series = [s for s in series if np.isfinite(s).all()]
        a, _ = extract(ctx, base, series, False)
        b, _ = extract(ctx, more, series, False)
        names_a, names_b = Plan(base).suffixes, Plan(more).suffixes
        idx = [names_b.index(s) for s in names_a]
        assert np.array_equal(a, b[:, idx], equal_nan=True)


def test_through_extract_features_and_roll(ctx):
    """the public entry points: a long frame, a wide frame with kinds, rolled windows"""
    import pandas as pd

    from tsfresh_b200 import extract_features
    from tsfresh_b200.rolling import roll_time_series
    st = {"agg_autocorrelation": [{"f_agg": "ptp", "maxlag": 5}, {"f_agg": "nansum", "maxlag": 3}],
          "change_quantiles": [{"ql": 0.2, "qh": 0.8, "isabs": False, "f_agg": "max"}],
          "linear_trend": [{"attr": "intercept_stderr"}],
          "augmented_dickey_fuller": [{"attr": "usedlag", "autolag": "t-stat"}]}
    rng = np.random.default_rng(9)
    df = pd.DataFrame({"id": np.repeat([1, 2, 3], 80), "time": np.tile(np.arange(80), 3),
                       "a": rng.standard_normal(240).astype(np.float32), "b": rng.standard_normal(240).cumsum().astype(np.float32)})
    X = extract_features(df, column_id="id", column_sort="time", default_fc_parameters=st, disable_progressbar=True)
    suffixes = Plan(st).suffixes
    for kind in ("a", "b"):
        series = [df[df.id == i][kind].to_numpy() for i in (1, 2, 3)]
        want = oracle_rows([s.astype(np.float64) for s in series], st)
        got = X[[kind + "__" + s for s in suffixes]].to_numpy()
        assert not compare(got, want, suffixes)
    rolled = roll_time_series(df[["id", "time", "a"]], column_id="id", column_sort="time", max_timeshift=30, min_timeshift=20)
    R = extract_features(rolled, column_id="id", column_sort="time", default_fc_parameters=st, disable_progressbar=True)
    assert R.shape[1] == len(suffixes) and len(R) == 3 * 60
    windows = []
    for key in R.index:                  # window (id, t): the rows of id with time in [t - 30, t]
        i, t = key
        w = df[(df.id == i) & (df.time >= t - 30) & (df.time <= t)].sort_values("time")
        windows.append(w["a"].to_numpy().astype(np.float64))
    got = R[["a__" + s for s in suffixes]].to_numpy()
    bad = compare(got, oracle_rows(windows, st), suffixes)
    assert not bad, bad[:10]


def test_change_quantiles_median_is_the_median(ctx):
    """f_agg "median" of change_quantiles is np.median of the corridor's changes (it used to give their variance)"""
    st = {"change_quantiles": [{"ql": ql, "qh": qh, "isabs": b, "f_agg": "median"} for ql, qh in ((0.0, 0.6), (0.2, 0.8))
                               for b in (False, True)]}
    series = [_rng(n, n, walk) for n in (40, 301, 2000) for walk in (False, True)]
    got, _ = extract(ctx, st, series, False)
    assert not check(got, oracle_rows([s.astype(np.float64) for s in series], st), Plan(st).suffixes, [False] * len(series))


_GLOBAL_WORKER = """
import json, sys
import numpy as np
sys.path.insert(0, %r)
from tests.test_gpu_vocabulary import call_series, extract, settings
from tsfresh_b200._lib import Context
ctx = Context(0)
series, _ = call_series(1500, 1500)
got, kernels = extract(ctx, settings("sorted", 1500), series, False)
np.save(%r, got)
print(json.dumps(kernels))
ctx.close()
"""


def test_sorted_global_region(tmp_path):
    """the SORTED global region (TSFX_GLOBAL_ABOVE=1, read once per process: a process of its own)"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    path = str(tmp_path / "sorted_global.npy")
    env = {k: v for k, v in os.environ.items() if not k.startswith("TSFX_")}
    env["TSFX_GLOBAL_ABOVE"] = "1"
    r = subprocess.run([sys.executable, "-c", _GLOBAL_WORKER % (root, path)], env=env, cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    kernels = json.loads(r.stdout.strip().splitlines()[-1])
    REACHED.update(kernels)
    assert "sorted/w4/global" in kernels, kernels
    series, degenerate = call_series(1500, 1500)
    st = settings("sorted", 1500)
    bad = check(np.load(path), oracle_rows([s.astype(np.float64) for s in series], st), Plan(st).suffixes, degenerate)
    assert not bad, bad[:10]


def test_plan_create_refuses_unknown_codes(ctx):
    """codes outside the documented sets reach tsfx_plan_create only through the C ABI: refused there, before any launch"""
    from tsfresh_b200._lib import DevicePlan
    cq = {"ql": 0.2, "qh": 0.8, "isabs": False, "f_agg": "mean"}
    cases = [({"agg_autocorrelation": [{"f_agg": "mean", "maxlag": 3}]}, "attr", v) for v in (9, 15, 22, 25, -1)]
    cases += [({"change_quantiles": [cq]}, "attr", v) for v in (9, 22, 31)]
    cases += [({"agg_linear_trend": [{"attr": "slope", "chunk_len": 5, "f_agg": "max"}]}, "i1", v) for v in (6, 16, 20)]
    cases += [({"agg_linear_trend": [{"attr": "slope", "chunk_len": 5, "f_agg": "max"}]}, "attr", 6),
              ({"linear_trend": [{"attr": "slope"}]}, "attr", 6),
              ({"augmented_dickey_fuller": [{"attr": "teststat", "autolag": "AIC"}]}, "i0", 4)]
    for st, field, value in cases:
        plan = Plan(st)
        plan.descs[field] = value
        with pytest.raises(NotImplementedError):
            DevicePlan(ctx, plan)


def test_ledger():
    """runs last: every variant the new cases are meant to run in did run"""
    want = {v for _, _, _, v in CASES} | {"sorted/w4/global"}
    assert want <= REACHED, sorted(want - REACHED)
    print("t-stat waiver rows: %d" % len(WAIVED))
