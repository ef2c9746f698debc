"""TEST INFRASTRUCTURE (build container only): what the UNMODIFIED reference answers for the parameter values beyond the
Comprehensive grid that the plan compiler accepts -> tests/golden/vocabulary.npz, read by tests/test_vocabulary_host.py:

  * every numpy f_agg of agg_autocorrelation (maxlag 0, 1, 5, 40; NaN on the +-inf series, where statsmodels' acf
    raises and with it the reference's whole extraction) and change_quantiles (the Comprehensive corridors,
    isabs False and True);
  * attr "intercept_stderr" of linear_trend, agg_linear_trend and linear_trend_timewise;
  * augmented_dickey_fuller with autolag "t-stat", lower- and mixed-case names, and names adfuller refuses.

The aggregator and linregress columns are the reference on the installed numpy and scipy.  adfuller comes from
oracle/thirdparty.py through oracle/ref_shim.py (statsmodels is not installed), so the ADF columns pin the reference's
handling of the names, not statsmodels itself.  The series and settings are built by the functions below, which the
test imports too."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

AGGS = ("mean", "median", "var", "std", "max", "amax", "min", "amin", "ptp", "sum", "prod", "average",
        "nanmean", "nanmedian", "nanvar", "nanstd", "nanmax", "nanmin", "nansum", "nanprod")
RAISE_ON_EMPTY = ("max", "amax", "min", "amin", "ptp", "nanmax", "nanmin")
MAXLAGS = (0, 1, 5, 40)
CORRIDORS = [(ql, qh) for ql in (0.0, 0.2, 0.4, 0.6, 0.8) for qh in (0.2, 0.4, 0.6, 0.8, 1.0)]
AUTOLAGS = ("t-stat", "aic", "Aic", "bic", "T-STAT", "t-stats", "xyz")


def series():
    """(name, float32 series): random, walk, tied, constant, 1-5 samples, and +-inf pairs"""
    rng = np.random.default_rng(2027)
    out = [("random_%d" % n, rng.standard_normal(n)) for n in (60, 257)]
    out += [("walk_%d" % n, rng.standard_normal(n).cumsum()) for n in (100, 300)]
    out += [("tied", np.repeat(rng.integers(0, 4, 30), 3).astype(np.float64)), ("constant", np.full(50, 1.5))]
    out += [("short_%d" % n, rng.standard_normal(n)) for n in range(1, 6)]
    inf = rng.standard_normal(80)
    inf[[10, 11, 40, 41]] = [np.inf, -np.inf, np.inf, np.inf]     # inf - inf and inf - (-inf) among the changes
    out.append(("inf_pairs", inf))
    return [(k, np.asarray(v, dtype=np.float32)) for k, v in out]


def settings():
    """the settings of the golden rows, in column order (linear_trend_timewise needs the rows' timestamps)"""
    return {
        "agg_autocorrelation": [{"f_agg": f, "maxlag": m} for f in AGGS for m in MAXLAGS
                                if not (m == 0 and f in RAISE_ON_EMPTY)],
        "change_quantiles": [{"ql": ql, "qh": qh, "isabs": b, "f_agg": f} for ql, qh in CORRIDORS
                             for b in (False, True) for f in AGGS],
        "linear_trend": [{"attr": a} for a in ("intercept_stderr", "stderr", "intercept")],
        "agg_linear_trend": [{"attr": "intercept_stderr", "chunk_len": c, "f_agg": f} for c in (2, 5, 10)
                             for f in ("max", "mean", "var")],
        "augmented_dickey_fuller": [{"attr": a, "autolag": al} for al in AUTOLAGS for a in ("teststat", "pvalue", "usedlag")],
        "linear_trend_timewise": [{"attr": a} for a in ("intercept_stderr", "stderr")],
    }


def times(n, seed):
    """int64 nanosecond timestamps of n rows, irregular gaps"""
    rng = np.random.default_rng(seed)
    return (rng.integers(1, 5000, n).cumsum() * 10 ** 9 + rng.integers(0, 10 ** 9, n)).astype(np.int64)


def main():
    import pandas as pd

    from oracle import ref_shim
    from tsfresh_b200.plan import param_string
    ref_shim.load()
    from tsfresh.feature_extraction import feature_calculators as fc

    arrays = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with np.errstate(all="ignore"):
            for i, (name, x32) in enumerate(series()):
                x = x32.astype(np.float64)
                row = []
                for calc, plist in settings().items():
                    if calc == "linear_trend_timewise":
                        s = pd.Series(x, index=pd.DatetimeIndex(times(len(x), i).astype("datetime64[ns]")))
                        row += [v for _, v in fc.linear_trend_timewise(s, plist)]
                    elif calc == "change_quantiles":
                        row += [fc.change_quantiles(x, **p) for p in plist]
                    elif calc == "agg_autocorrelation" and not np.isfinite(x).all():
                        row += [np.nan] * len(plist)        # acf raises on inf: the reference's extraction fails
                    else:
                        got = dict(getattr(fc, calc)(x, plist))
                        row += [got[k] for k in _combiner_keys(calc, plist, param_string)]
                arrays[name] = np.asarray(row, dtype=np.float64)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "vocabulary.npz"), **arrays)


def _combiner_keys(calc, plist, param_string):
    if calc == "agg_autocorrelation":
        return ['f_agg_"%s"__maxlag_%s' % (p["f_agg"], p["maxlag"]) for p in plist]
    if calc == "linear_trend":
        return ['attr_"%s"' % p["attr"] for p in plist]
    if calc == "agg_linear_trend":
        return ['attr_"%s"__chunk_len_%s__f_agg_"%s"' % (p["attr"], p["chunk_len"], p["f_agg"]) for p in plist]
    if calc == "augmented_dickey_fuller":
        return ['attr_"%s"__autolag_"%s"' % (p["attr"], p["autolag"]) for p in plist]
    raise KeyError(calc)


if __name__ == "__main__":
    main()
