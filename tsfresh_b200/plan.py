"""Plan compiler: FC-parameters dict -> ordered output columns + flat tsfx_feature_desc table.

Restates, for the GPU path, what the reference's per-series loop does with the settings dict
(tsfresh/feature_extraction/extraction.py:339-378): iterate the dict in order, expand each
calculator's parameter list, and name every value `{kind}__{calculator}[__{params}]`
(parameter strings: utilities/string_manipulation.py:47-74 for "simple" calculators, the literal
f-strings of each "combiner" in feature_calculators.py).  Callable keys and parameter values without
a GPU implementation raise NotImplementedError -- there is no CPU fallback.
"""
import ctypes
import math
import os
import re

import numpy as np

_HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include", "tsfx.h")


def _parse_calc_enum():
    text = open(_HEADER).read()
    body = re.search(r"enum tsfx_calc \{(.*?)\};", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [t.split("=")[0].strip() for t in body.split(",") if t.strip()]
    return {n: i for i, n in enumerate(names)}


CALC = _parse_calc_enum()
CALC_NAME = {v: k for k, v in CALC.items()}

AGG = {"mean": 0, "median": 1, "var": 2, "std": 3, "max": 4, "min": 5}
AGG_NANSKIP = 16            # TSFX_AGG_NANSKIP: the np.nan* variant of a reducer
# numpy functions agg_autocorrelation and change_quantiles accept as f_agg (the reference calls getattr(np, f_agg))
AGG_NUMPY = dict(AGG, amax=4, amin=5, ptp=6, sum=7, prod=8, average=0,
                 **{"nan" + k: v | AGG_NANSKIP for k, v in (("mean", 0), ("median", 1), ("var", 2), ("std", 3), ("max", 4),
                                                             ("min", 5), ("sum", 7), ("prod", 8))})
AGG_RAISES_ON_EMPTY = ("max", "amax", "min", "amin", "ptp", "nanmax", "nanmin")
FFT_ATTR = {"real": 0, "imag": 1, "abs": 2, "angle": 3}
SPEC_ATTR = {"centroid": 0, "variance": 1, "skew": 2, "kurtosis": 3}
LR_ATTR = {"pvalue": 0, "rvalue": 1, "intercept": 2, "slope": 3, "stderr": 4, "intercept_stderr": 5}
ADF_ATTR = {"teststat": 0, "pvalue": 1, "usedlag": 2}
AUTOLAG = {"aic": 0, "bic": 1, None: 2, "t-stat": 3}     # statsmodels lower-cases the name


class tsfx_feature_desc(ctypes.Structure):
    _fields_ = [("calc", ctypes.c_int32), ("attr", ctypes.c_int32), ("i0", ctypes.c_int32),
                ("i1", ctypes.c_int32), ("i2", ctypes.c_int32), ("col", ctypes.c_int32),
                ("p0", ctypes.c_double), ("p1", ctypes.c_double)]


DESC_DTYPE = np.dtype([("calc", "<i4"), ("attr", "<i4"), ("i0", "<i4"), ("i1", "<i4"), ("i2", "<i4"),
                       ("col", "<i4"), ("p0", "<f8"), ("p1", "<f8")])
assert DESC_DTYPE.itemsize == ctypes.sizeof(tsfx_feature_desc) == 40


def param_string(param):
    """`k_v__k_v` with keys sorted and strings quoted (string_manipulation.py:47-74)."""
    def fmt(v):
        return '"' + str(v) + '"' if isinstance(v, str) else str(v)
    return "__".join(str(k) + "_" + fmt(param[k]) for k in sorted(param.keys()))


def _unsupported(name, why):
    raise NotImplementedError("%s: %s has no GPU implementation (and there is no CPU fallback)" % (name, why))


def _need(name, p, keys):
    extra = set(p) - set(keys)
    missing = set(keys) - set(p)
    if extra or missing:
        raise TypeError("%s() got parameters %s, expected %s" % (name, sorted(p), sorted(keys)))


def _int(name, key, v, lo=None, hi=None):
    if isinstance(v, (bool, np.bool_)) or int(v) != v:
        _unsupported(name, "%s=%r (integer expected)" % (key, v))
    v = int(v)
    if lo is not None and v < lo:
        raise ValueError("%s: %s=%d must be >= %d" % (name, key, v, lo))
    if hi is not None and v > hi:
        _unsupported(name, "%s=%d (> %d)" % (key, v, hi))
    return v


# Largest parameter values the kernels' layouts hold (tsfx_plan_create checks the same; DESIGN.md section 1)
MAX_LAG = 4096              # autocorrelation, agg_autocorrelation maxlag, partial_autocorrelation: lag products per warp
MAX_AR_K = 32               # ar_coefficient
MAX_CWT_PEAKS_N = 16        # number_cwt_peaks: rows of the Ricker tap table
MAX_FRIEDRICH_R = 256       # friedrich_coefficients, max_langevin_fixed_point: quantile bins
MAX_PERM_DIMENSION = 8      # permutation_entropy: order bits of a window fit 32 bits
MAX_LZ_BINS = 65535         # lempel_ziv_complexity: 16-bit symbols, and the all-ones key marks an empty slot


# ------------------------------------------------------------------------------------------------
# simple calculators: name -> (required keys, lambda(param) -> dict(attr,i0,i1,i2,p0,p1))
def _s_agg(name, f_agg, allowed):
    if not isinstance(f_agg, str) or f_agg not in allowed:
        _unsupported(name, "f_agg=%r" % (f_agg,))
    return AGG_NUMPY[f_agg]


def _lr_attr(name, attr):
    """linregress attribute code; the reference's getattr(LinregressResult, attr) raises AttributeError for any other"""
    if not isinstance(attr, str) or attr not in LR_ATTR:
        raise AttributeError("%s: 'LinregressResult' object has no attribute %r" % (name, attr))
    return LR_ATTR[attr]


_SIMPLE_NO_PARAM = {
    n: CALC["TSFX_" + n.upper()] for n in (
        "variance_larger_than_standard_deviation", "has_duplicate_max", "has_duplicate_min", "has_duplicate",
        "sum_values", "abs_energy", "mean_abs_change", "mean_change", "mean_second_derivative_central",
        "median", "mean", "length", "standard_deviation", "variation_coefficient", "variance", "skewness",
        "kurtosis", "root_mean_square", "absolute_sum_of_changes", "longest_strike_below_mean",
        "longest_strike_above_mean", "count_above_mean", "count_below_mean", "last_location_of_maximum",
        "first_location_of_maximum", "last_location_of_minimum", "first_location_of_minimum",
        "percentage_of_reoccurring_values_to_all_values",
        "percentage_of_reoccurring_datapoints_to_all_datapoints", "sum_of_reoccurring_values",
        "sum_of_reoccurring_data_points", "ratio_value_number_to_time_series_length", "sample_entropy",
        "maximum", "absolute_maximum", "minimum", "benford_correlation")
}


def _simple_with_params(name, p):
    """Returns the descriptor fields for one parameter dict of a "simple" calculator."""
    f = dict(attr=0, i0=0, i1=0, i2=0, p0=0.0, p1=0.0)
    if name in ("ratio_beyond_r_sigma", "large_standard_deviation"):
        _need(name, p, ["r"]); f["p0"] = float(p["r"])
    elif name == "cid_ce":
        _need(name, p, ["normalize"]); f["i0"] = 1 if p["normalize"] else 0
    elif name in ("quantile", ):
        _need(name, p, ["q"]); f["p0"] = float(p["q"])
        if not (0.0 <= f["p0"] <= 1.0):
            raise ValueError("Quantiles must be in the range [0, 1]")
    elif name in ("autocorrelation", "time_reversal_asymmetry_statistic", "c3"):
        _need(name, p, ["lag"]); f["i0"] = _int(name, "lag", p["lag"], 0, MAX_LAG if name == "autocorrelation" else None)
    elif name in ("number_cwt_peaks", "number_peaks"):
        _need(name, p, ["n"]); f["i0"] = _int(name, "n", p["n"], 1, MAX_CWT_PEAKS_N if name == "number_cwt_peaks" else None)
    elif name == "binned_entropy":
        _need(name, p, ["max_bins"]); f["i0"] = _int(name, "max_bins", p["max_bins"], 1)
    elif name == "change_quantiles":
        _need(name, p, ["ql", "qh", "isabs", "f_agg"])
        f["p0"], f["p1"] = float(p["ql"]), float(p["qh"])
        f["i0"] = 1 if p["isabs"] else 0
        f["attr"] = _s_agg(name, p["f_agg"], AGG_NUMPY)
    elif name == "mean_n_absolute_max":
        _need(name, p, ["number_of_maxima"]); f["i0"] = _int(name, "number_of_maxima", p["number_of_maxima"], 1)
    elif name == "approximate_entropy":
        _need(name, p, ["m", "r"])
        f["i0"] = _int(name, "m", p["m"], 1); f["p0"] = float(p["r"])
        if f["p0"] < 0:
            raise ValueError("Parameter r must be positive.")
        if f["i0"] != 2:
            _unsupported(name, "m=%d (only m=2)" % f["i0"])
    elif name in ("fourier_entropy", "lempel_ziv_complexity"):
        _need(name, p, ["bins"]); f["i0"] = _int(name, "bins", p["bins"], 1, MAX_LZ_BINS if name == "lempel_ziv_complexity" else None)
    elif name == "permutation_entropy":
        _need(name, p, ["tau", "dimension"])
        f["i0"] = _int(name, "tau", p["tau"], 1); f["i1"] = _int(name, "dimension", p["dimension"], 2, MAX_PERM_DIMENSION)
    elif name == "number_crossing_m":
        _need(name, p, ["m"]); f["p0"] = float(p["m"])
    elif name == "value_count":
        _need(name, p, ["value"]); f["p0"] = float(p["value"])
    elif name == "range_count":
        _need(name, p, ["min", "max"]); f["p0"], f["p1"] = float(p["min"]), float(p["max"])
    elif name in ("count_above", "count_below"):
        _need(name, p, ["t"]); f["p0"] = float(p["t"])
    elif name == "max_langevin_fixed_point":
        _need(name, p, ["m", "r"])
        f["i1"] = _int(name, "m", p["m"], 1); f["i2"] = _int(name, "r", p["r"], 1, MAX_FRIEDRICH_R)
        if f["i1"] != 3:
            _unsupported(name, "m=%d (only the cubic m=3)" % f["i1"])
    else:
        raise KeyError(name)
    return f


_SIMPLE_WITH_PARAM = ("ratio_beyond_r_sigma", "large_standard_deviation", "cid_ce", "quantile",
                      "autocorrelation", "time_reversal_asymmetry_statistic", "c3", "number_cwt_peaks",
                      "number_peaks", "binned_entropy", "change_quantiles", "mean_n_absolute_max",
                      "approximate_entropy", "fourier_entropy", "lempel_ziv_complexity",
                      "permutation_entropy", "number_crossing_m", "value_count", "range_count",
                      "count_above", "count_below", "max_langevin_fixed_point")


class Plan:
    """Ordered columns + descriptor table for ONE kind's settings."""

    def __init__(self, fc_parameters, has_datetime_index=False):
        self.suffixes = []          # "calculator[__params]" per column (kind prefix added by the caller)
        rows = []                   # dict(calc, attr, i0, i1, i2, p0, p1) per column
        self.cwt_scales = []        # distinct cwt scales -> table index
        self.skipped = []           # calculators skipped with a warning (DatetimeIndex required)
        self.needs_times = False    # linear_trend_timewise columns: the extract call needs the rows' timestamps
        for key, plist in fc_parameters.items():
            if callable(key):
                _unsupported(getattr(key, "__name__", repr(key)), "a user-supplied callable calculator")
            name = str(key)
            if name == "linear_trend_timewise" and not has_datetime_index:
                self.skipped.append(name)   # extraction.py:349-358: warn + continue
                continue
            for suffix, fields in self._expand(name, plist):
                self.suffixes.append(name + ("__" + suffix if suffix else ""))
                rows.append(fields)
        self.n_cols = len(rows)
        self.descs = np.zeros(self.n_cols, dtype=DESC_DTYPE)
        for c, f in enumerate(rows):
            self.descs[c] = (f["calc"], f["attr"], f["i0"], f["i1"], f["i2"], c, f["p0"], f["p1"])

    # ----------------------------------------------------------------------------------------
    def _table_index(self, scale):
        if scale not in self.cwt_scales:
            self.cwt_scales.append(scale)
        return self.cwt_scales.index(scale)

    def _expand(self, name, plist):
        base = dict(attr=0, i0=0, i1=0, i2=0, p0=0.0, p1=0.0)
        if name in _SIMPLE_NO_PARAM:
            if plist:
                raise TypeError("%s() takes no parameters" % name)
            yield "", dict(base, calc=_SIMPLE_NO_PARAM[name])
            return
        if name in _SIMPLE_WITH_PARAM:
            if not plist:
                raise TypeError("%s() needs a parameter list" % name)
            for p in plist:
                yield param_string(p), dict(_simple_with_params(name, p), calc=CALC["TSFX_" + name.upper()])
            return
        fn = getattr(self, "_c_" + name, None)
        if fn is None:
            if name == "matrix_profile":
                _unsupported(name, "the optional matrixprofile dependency")
            raise AttributeError("module 'tsfresh.feature_extraction.feature_calculators' has no attribute %r" % name)
        if plist is None:
            raise TypeError("%s() needs a parameter list" % name)
        seen = set()
        for suffix, fields in fn(plist, base):
            if suffix in seen:      # dict-returning combiners collapse duplicate keys
                continue
            seen.add(suffix)
            yield suffix, fields

    # ---- combiners (key formats: the f-strings of feature_calculators.py, line in the comment) ----
    def _c_symmetry_looking(self, plist, b):     # :319
        for p in plist:
            yield "r_%s" % (p["r"],), dict(b, calc=CALC["TSFX_SYMMETRY_LOOKING"], p0=float(p["r"]))

    def _c_agg_autocorrelation(self, plist, b):  # :432
        for p in plist:
            a = _s_agg("agg_autocorrelation", p["f_agg"], AGG_NUMPY)
            maxlag = _int("agg_autocorrelation", "maxlag", p["maxlag"], 0, MAX_LAG)
            if maxlag == 0 and p["f_agg"] in AGG_RAISES_ON_EMPTY:
                getattr(np, p["f_agg"])(np.zeros(0))    # numpy's ValueError: the reference's a[:0] is empty for every series
            yield ('f_agg_"%s"__maxlag_%s' % (p["f_agg"], p["maxlag"]),
                   dict(b, calc=CALC["TSFX_AGG_AUTOCORRELATION"], attr=a, i0=maxlag))

    def _c_partial_autocorrelation(self, plist, b):  # :495
        top = max(_int("partial_autocorrelation", "lag", p["lag"], 0, MAX_LAG) for p in plist)
        for p in plist:
            yield "lag_%s" % (p["lag"],), dict(b, calc=CALC["TSFX_PARTIAL_AUTOCORRELATION"], i0=int(p["lag"]), i1=top)

    def _c_augmented_dickey_fuller(self, plist, b):  # :534
        for p in plist:
            al = p.get("autolag", "AIC")
            if al is not None and not isinstance(al, str):
                _unsupported("augmented_dickey_fuller", "autolag=%r" % (al,))
            key = al.lower() if isinstance(al, str) else al
            suffix = 'attr_"%s"__autolag_"%s"' % (p["attr"], al)
            if key not in AUTOLAG:      # adfuller raises ValueError, which the reference turns into NaN (:520-526)
                yield suffix, dict(b, calc=CALC["TSFX_CONST_NAN"])
                continue
            yield suffix, dict(b, calc=CALC["TSFX_AUGMENTED_DICKEY_FULLER"], attr=ADF_ATTR.get(p["attr"], 3), i0=AUTOLAG[key])

    def _c_fft_coefficient(self, plist, b):  # :1088-1118
        assert min(p["coeff"] for p in plist) >= 0, "Coefficients must be positive or zero."
        assert {p["attr"] for p in plist} <= set(FFT_ATTR), 'Attribute must be "real", "imag", "angle" or "abs"'
        for p in plist:
            yield ('attr_"%s"__coeff_%s' % (p["attr"], p["coeff"]),
                   dict(b, calc=CALC["TSFX_FFT_COEFFICIENT"], attr=FFT_ATTR[p["attr"]],
                        i0=_int("fft_coefficient", "coeff", p["coeff"], 0)))

    def _c_fft_aggregated(self, plist, b):  # :1136-1230
        assert {p["aggtype"] for p in plist} <= set(SPEC_ATTR), \
            'Attribute must be "centroid", "variance", "skew", "kurtosis"'
        for p in plist:
            yield 'aggtype_"%s"' % (p["aggtype"],), dict(b, calc=CALC["TSFX_FFT_AGGREGATED"], attr=SPEC_ATTR[p["aggtype"]])

    def _c_index_mass_quantile(self, plist, b):  # :1300
        for p in plist:
            yield "q_%s" % (p["q"],), dict(b, calc=CALC["TSFX_INDEX_MASS_QUANTILE"], p0=float(p["q"]))

    def _c_linear_trend(self, plist, b):  # :1364
        for p in plist:
            yield 'attr_"%s"' % (p["attr"],), dict(b, calc=CALC["TSFX_LINEAR_TREND"], attr=_lr_attr("linear_trend", p["attr"]))

    def _c_cwt_coefficients(self, plist, b):  # :1396-1412
        for p in plist:
            widths = tuple(p["widths"])
            if p["w"] not in widths:
                raise ValueError("tuple.index(x): x not in tuple")
            yield ("coeff_%s__w_%s__widths_%s" % (p["coeff"], p["w"], widths),
                   dict(b, calc=CALC["TSFX_CWT_COEFFICIENTS"], i0=_int("cwt_coefficients", "coeff", p["coeff"], 0),
                        i1=self._table_index(p["w"])))

    def _c_spkt_welch_density(self, plist, b):  # :1436-1437
        for p in plist:
            yield "coeff_%s" % (p["coeff"],), dict(b, calc=CALC["TSFX_SPKT_WELCH_DENSITY"],
                                                   i0=_int("spkt_welch_density", "coeff", p["coeff"], 0))

    def _c_ar_coefficient(self, plist, b):  # :1485-1505
        for p in plist:
            k = _int("ar_coefficient", "k", p["k"], 1, MAX_AR_K)
            yield "coeff_%s__k_%s" % (p["coeff"], p["k"]), dict(
                b, calc=CALC["TSFX_AR_COEFFICIENT"], i0=_int("ar_coefficient", "coeff", p["coeff"], 0), i1=k)

    def _c_friedrich_coefficients(self, plist, b):  # :2114-2128
        for p in plist:
            assert p["coeff"] >= 0, "Coefficients must be positive or zero. Found %s" % (p["coeff"],)
            m = _int("friedrich_coefficients", "m", p["m"], 1)
            if m != 3:
                _unsupported("friedrich_coefficients", "m=%d (only the cubic m=3)" % m)
            yield "coeff_%s__m_%s__r_%s" % (p["coeff"], p["m"], p["r"]), dict(
                b, calc=CALC["TSFX_FRIEDRICH_COEFFICIENTS"], i0=int(p["coeff"]), i1=m,
                i2=_int("friedrich_coefficients", "r", p["r"], 1, MAX_FRIEDRICH_R))

    def _c_agg_linear_trend(self, plist, b):  # :2198-2220
        for p in plist:
            attr = _lr_attr("agg_linear_trend", p["attr"])
            fa = _s_agg("agg_linear_trend", p["f_agg"], ("max", "min", "mean", "var", "std", "median"))
            yield ('attr_"%s"__chunk_len_%s__f_agg_"%s"' % (p["attr"], p["chunk_len"], p["f_agg"]),
                   dict(b, calc=CALC["TSFX_AGG_LINEAR_TREND"], attr=attr,
                        i0=_int("agg_linear_trend", "chunk_len", p["chunk_len"], 1), i1=fa))

    def _c_energy_ratio_by_chunks(self, plist, b):  # :2251-2265
        for p in plist:
            ns = _int("energy_ratio_by_chunks", "num_segments", p["num_segments"])
            sf = _int("energy_ratio_by_chunks", "segment_focus", p["segment_focus"])
            assert sf < ns
            assert ns > 0
            yield "num_segments_%s__segment_focus_%s" % (p["num_segments"], p["segment_focus"]), dict(
                b, calc=CALC["TSFX_ENERGY_RATIO_BY_CHUNKS"], i0=ns, i1=sf)

    def _c_linear_trend_timewise(self, plist, b):  # :2302-2305 (only reached with a DatetimeIndex)
        self.needs_times = True
        for p in plist:
            yield 'attr_"%s"' % p["attr"], dict(b, calc=CALC["TSFX_LINEAR_TREND_TIMEWISE"],
                                                attr=_lr_attr("linear_trend_timewise", p["attr"]))

    def _c_query_similarity_count(self, plist, b):  # :2505-2519
        for p in plist:
            q = np.asarray(p.get("query", None)).astype(float)
            if q.size >= 3:
                _unsupported("query_similarity_count", "a real query (stumpy.core.mass)")
            yield param_string(p), dict(b, calc=CALC["TSFX_QUERY_SIMILARITY_COUNT"])

    # ----------------------------------------------------------------------------------------
    def cwt_tables(self):
        """Convolution tables for cwt_coefficients: for each distinct scale `a` the difference kernel
        D_a[j] = -sqrt(a) * (K_a[j] - K_a[j-1]) where K_a is PyWavelets' reversed, resampled integrated
        Mexican-hat at that scale (pywt.cwt, called at feature_calculators.py:1402), so that
        coefficient c of the trimmed transform is sum_k x[k] * D_a[c + half_a - k]."""
        tabs, off, half = [], [0], []
        for a in self.cwt_scales:
            ker = _mexh_kernel(a)
            K = len(ker)
            ext = np.concatenate([[0.0], ker, [0.0]])
            d = -math.sqrt(a) * (ext[1:] - ext[:-1])       # D[j] = K[j] - K[j-1], j = 0..K
            tabs.append(d)
            off.append(off[-1] + len(d))
            half.append(int(math.floor((K - 2) / 2.0)) + 1)
        tables = np.concatenate(tabs) if tabs else np.zeros(0)
        return (np.ascontiguousarray(tables, dtype=np.float64), np.asarray(off, dtype=np.int64),
                np.asarray(half, dtype=np.int32))


def _mexh_kernel(scale):
    """PyWavelets cwt kernel for wavelet "mexh" at `scale` (precision=10 integration grid)."""
    t = np.linspace(-8.0, 8.0, 1024)
    psi = (1.0 - t ** 2) * np.exp(-(t ** 2) / 2.0) * 2.0 / (math.sqrt(3.0) * math.sqrt(math.sqrt(math.pi)))
    step = t[1] - t[0]
    int_psi = np.cumsum(psi) * step
    j = np.arange(scale * (t[-1] - t[0]) + 1) / (scale * step)
    j = j.astype(int)
    if j[-1] >= int_psi.size:
        j = np.extract(j < int_psi.size, j)
    return int_psi[j][::-1]
