"""CPU checks of the parameter values beyond the Comprehensive grid: every numpy f_agg of agg_autocorrelation and
change_quantiles, attr "intercept_stderr" of the three linregress calculators, and augmented_dickey_fuller's autolag
"t-stat" and case-insensitive names.  Column names and descriptors, from_columns, the refusals that remain, the plan-time
errors numpy raises on an empty lag vector, the oracle against the reference (tests/golden/vocabulary.npz, written by
oracle/make_golden_vocabulary.py) and the t-stat lag search against explicit least-squares designs."""
import os

import numpy as np
import pytest

from oracle.make_golden_vocabulary import RAISE_ON_EMPTY, series, settings, times
from tsfresh_b200.plan import AGG_NANSKIP, CALC, Plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODES = {"mean": 0, "median": 1, "var": 2, "std": 3, "max": 4, "amax": 4, "min": 5, "amin": 5, "ptp": 6, "sum": 7,
         "prod": 8, "average": 0, "nanmean": 16, "nanmedian": 17, "nanvar": 18, "nanstd": 19, "nanmax": 20, "nanmin": 21,
         "nansum": 23, "nanprod": 24}


def _header_value(name):
    import re
    text = open(os.path.join(ROOT, "include", "tsfx.h")).read()
    m = re.search(r"#define %s (\d+)" % name, text)
    if m:
        return int(m.group(1))
    for body in re.findall(r"enum \{([^}]*)\}", text):
        names = [t.split("=")[0].strip() for t in body.split(",")]
        if name in names:
            return names.index(name)
    raise KeyError(name)


def test_codes_match_the_header():
    assert AGG_NANSKIP == _header_value("TSFX_AGG_NANSKIP")
    for f, code in CODES.items():
        base = f[3:] if f.startswith("nan") else f
        base = {"amax": "max", "amin": "min", "average": "mean"}.get(base, base)
        assert code == _header_value("TSFX_AGG_" + base.upper()) | (AGG_NANSKIP if f.startswith("nan") else 0), f
    assert _header_value("TSFX_LR_INTERCEPT_STDERR") == 5 and _header_value("TSFX_AUTOLAG_TSTAT") == 3


def test_column_names_and_descriptors():
    p = Plan({"agg_autocorrelation": [{"f_agg": f, "maxlag": 7} for f in CODES],
              "change_quantiles": [{"ql": 0.2, "qh": 0.8, "isabs": True, "f_agg": f} for f in CODES]})
    for i, f in enumerate(CODES):
        assert p.suffixes[i] == 'agg_autocorrelation__f_agg_"%s"__maxlag_7' % f
        assert p.descs[i]["calc"] == CALC["TSFX_AGG_AUTOCORRELATION"] and p.descs[i]["attr"] == CODES[f] and p.descs[i]["i0"] == 7
        j = len(CODES) + i
        assert p.suffixes[j] == 'change_quantiles__f_agg_"%s"__isabs_True__qh_0.8__ql_0.2' % f
        assert p.descs[j]["calc"] == CALC["TSFX_CHANGE_QUANTILES"] and p.descs[j]["attr"] == CODES[f]
        assert (p.descs[j]["i0"], p.descs[j]["p0"], p.descs[j]["p1"]) == (1, 0.2, 0.8)
    p = Plan({"linear_trend": [{"attr": "intercept_stderr"}],
              "agg_linear_trend": [{"attr": "intercept_stderr", "chunk_len": 5, "f_agg": "max"}],
              "linear_trend_timewise": [{"attr": "intercept_stderr"}]}, has_datetime_index=True)
    assert p.suffixes == ['linear_trend__attr_"intercept_stderr"',
                          'agg_linear_trend__attr_"intercept_stderr"__chunk_len_5__f_agg_"max"',
                          'linear_trend_timewise__attr_"intercept_stderr"']
    assert list(p.descs["attr"]) == [5, 5, 5] and p.descs[1]["i0"] == 5 and p.descs[1]["i1"] == 4
    names = ("t-stat", "T-Stat", "aic", "Aic", "AIC", "bic", "BIC", None, "t-stats", "xyz")
    p = Plan({"augmented_dickey_fuller": [{"attr": "usedlag", "autolag": al} for al in names]})
    assert p.suffixes == ['augmented_dickey_fuller__attr_"usedlag"__autolag_"%s"' % al for al in names]
    adf, nan = CALC["TSFX_AUGMENTED_DICKEY_FULLER"], CALC["TSFX_CONST_NAN"]
    assert [(int(d["calc"]), int(d["i0"])) for d in p.descs] == \
        [(adf, 3), (adf, 3), (adf, 0), (adf, 0), (adf, 0), (adf, 1), (adf, 1), (adf, 2), (nan, 0), (nan, 0)]
    assert all(d["attr"] == 2 for d in p.descs[:8])


def test_from_columns_round_trip():
    from tsfresh_b200 import from_columns
    st = dict(settings())
    st.pop("linear_trend_timewise")
    suffixes = [s for s in Plan(st).suffixes if "intercept_stderr" not in s]
    back = from_columns(["x__" + s for s in suffixes])["x"]
    assert sorted(Plan(back).suffixes) == sorted(suffixes)
    # the reference splits every parameter at its last "_" (string_manipulation.py:29-30), so it cannot read back
    # attr_"intercept_stderr" either: literal_eval('stderr"') raises SyntaxError there too
    with pytest.raises(SyntaxError):
        from_columns(['x__linear_trend__attr_"intercept_stderr"'])


def test_what_is_still_refused():
    """layout limits and calculators without a GPU path; the ordinary values the reference documents all plan"""
    refused = [{(lambda x: 0): None}, {"approximate_entropy": [{"m": 3, "r": 0.1}]},
               {"query_similarity_count": [{"query": [1.0, 2.0, 3.0], "threshold": 0.0}]},
               {"friedrich_coefficients": [{"coeff": 0, "m": 2, "r": 30}]}, {"max_langevin_fixed_point": [{"m": 5, "r": 30}]},
               {"matrix_profile": [{"threshold": 0.98, "feature": "min"}]},
               {"autocorrelation": [{"lag": 4097}]}, {"ar_coefficient": [{"coeff": 0, "k": 33}]},
               {"lempel_ziv_complexity": [{"bins": 65536}]}, {"agg_autocorrelation": [{"f_agg": "cumsum", "maxlag": 3}]},
               {"change_quantiles": [{"ql": 0.1, "qh": 0.9, "isabs": False, "f_agg": "quantile"}]},
               {"augmented_dickey_fuller": [{"attr": "teststat", "autolag": 3}]}]
    for st in refused:
        with pytest.raises(NotImplementedError):
            Plan(st)
    assert Plan(settings(), has_datetime_index=True).n_cols == sum(len(v) for v in settings().values())
    for calc in ("linear_trend", "linear_trend_timewise"):
        with pytest.raises(AttributeError):
            Plan({calc: [{"attr": "slope_stderr"}]}, has_datetime_index=True)
    with pytest.raises(AttributeError):
        Plan({"agg_linear_trend": [{"attr": "nope", "chunk_len": 5, "f_agg": "max"}]})


@pytest.mark.parametrize("f_agg", list(CODES))
def test_maxlag_zero(f_agg):
    """numpy on the empty a[:0]: the reducers that raise there raise the same error from Plan"""
    st = {"agg_autocorrelation": [{"f_agg": f_agg, "maxlag": 0}]}
    if f_agg in RAISE_ON_EMPTY:
        with pytest.raises(ValueError) as ours:
            Plan(st)
        with pytest.raises(ValueError) as theirs:
            getattr(np, f_agg)(np.zeros(0))
        assert str(ours.value) == str(theirs.value)
    else:
        assert Plan(st).n_cols == 1


def _oracle_row(i, x):
    """the oracle's row; agg_autocorrelation is NaN on a series with inf, where both raise (statsmodels' acf)"""
    from oracle.extract import oracle_rows
    st = settings()
    if np.isfinite(x).all():
        return oracle_rows([x.astype(np.float64)], st, times=[times(len(x), i)])[0]
    skip = len(st.pop("agg_autocorrelation"))
    return np.concatenate([np.full(skip, np.nan), oracle_rows([x.astype(np.float64)], st, times=[times(len(x), i)])[0]])


def test_oracle_matches_the_reference():
    golden = np.load(os.path.join(ROOT, "tests", "golden", "vocabulary.npz"))
    suffixes = Plan(settings(), has_datetime_index=True).suffixes
    for i, (name, x) in enumerate(series()):
        want, got = golden[name], _oracle_row(i, x)
        assert got.shape == want.shape
        for c, suf in enumerate(suffixes):
            if name == "inf_pairs" and suf.startswith("agg_autocorrelation"):
                continue        # the reference raises (statsmodels' acf refuses inf)
            g, w = got[c], want[c]
            assert (np.isnan(g) and np.isnan(w)) or g == w or np.isclose(g, w, rtol=1e-12, atol=0), (name, suf, g, w)


def _tstat_lstsq(x):
    """adfuller(x, autolag="t-stat", regression="c") from explicit designs and numpy.linalg.lstsq: (usedlag, teststat)"""
    x = np.asarray(x, np.float64)
    x = x - x.mean()            # the level column, centred: the same fits next to the constant, better conditioned
    n = len(x)
    maxlag = min(n // 2 - 2, int(np.ceil(12.0 * (n / 100.0) ** 0.25)))
    d = np.diff(x)

    def design(lags):
        rows = np.arange(lags, n - 1)
        cols = [np.ones(len(rows)), x[rows]] + [d[rows - j] for j in range(1, lags + 1)]
        return np.column_stack(cols), d[rows]

    full, y = design(maxlag)
    used = 0
    for q in range(maxlag + 2, 2, -1):
        X = full[:, :q]
        beta, *_ = np.linalg.lstsq(X, y, rcond=None)
        r = y - X @ beta
        cov = np.linalg.inv(X.T @ X) * (r @ r) / (len(y) - q)
        if abs(beta[-1] / np.sqrt(cov[-1, -1])) >= 1.6448536269514722:
            used = q - 2
            break
    X, y = design(used)
    beta, *_ = np.linalg.lstsq(X, y, rcond=None)
    r = y - X @ beta
    cov = np.linalg.inv(X.T @ X) * (r @ r) / (len(y) - X.shape[1])
    return used, beta[1] / np.sqrt(cov[1, 1])


def test_tstat_independent_route():
    from oracle import thirdparty as tp
    rng = np.random.default_rng(5)
    xs = [rng.standard_normal(n).cumsum() for n in (30, 100, 257, 1000)] + [rng.standard_normal(n) for n in (40, 500)]
    xs += [(1000.0 + 0.01 * rng.standard_normal(300)).astype(np.float32).astype(np.float64) for _ in range(3)]   # level series
    lags = set()
    for x in xs:
        stat, _, used = tp.adfuller(x, autolag="t-stat")
        u2, s2 = _tstat_lstsq(x)
        assert used == u2, (len(x), used, u2)
        assert np.isclose(stat, s2, rtol=1e-8, atol=0), (len(x), stat, s2)
        lags.add(used)
    assert len(lags) > 2, lags          # the search stops at different lags on these series
