"""TEST INFRASTRUCTURE: float64 CPU restatement of the tsfresh calculator registry.

Every function cites the reference lines it restates (paths relative to
/root/reference/tsfresh/feature_extraction/feature_calculators.py unless noted).  The numerics are
delegated to the same numpy / scipy / pandas routines the reference calls (they are installed in this
image and on the GPU box); the statsmodels / PyWavelets routines come from oracle/thirdparty.py.

Pinned against the unmodified reference by tests/test_oracle_vs_reference.py (build container) and by
tests/golden/*.npz (everywhere).  Not part of the product path.

Layout: SIMPLE[name](x, **params) -> scalar ; COMBINER[name](x, param_list) -> list of scalars in
param_list order (the reference's "combiner" calculators return (key, value) pairs; keys are produced
by tsfresh_b200.plan and checked against the golden column list).
"""
import itertools
import math

import numpy as np
import pandas as pd
from scipy.signal import find_peaks_cwt, welch
from scipy.stats import linregress

from . import thirdparty as tp

NAN = float("nan")
SIMPLE = {}
COMBINER = {}


def simple(fn):
    SIMPLE[fn.__name__] = fn
    return fn


def combiner(fn):
    COMBINER[fn.__name__] = fn
    return fn


def _runs_of_true(mask):
    """lengths of maximal True runs (:102-128); [0] when there is none."""
    out = [sum(1 for _ in g) for v, g in itertools.groupby(mask) if v]
    return out or [0]


def _cyc(a, shift):
    """:56-99 cyclic shift to the right by `shift`."""
    k = shift % len(a)
    return np.concatenate([a[-k:], a[:-k]])


# ------------------------------------------------------------------ class M / O : moments, counts, order
@simple
def variance_larger_than_standard_deviation(x):  # :239-252
    v = np.var(x)
    return v > np.sqrt(v)


@simple
def ratio_beyond_r_sigma(x, r):  # :256-269
    return np.sum(np.abs(x - np.mean(x)) > r * np.std(x)) / x.size


@simple
def large_standard_deviation(x, r):  # :273-295
    return np.std(x) > r * (np.max(x) - np.min(x))


@combiner
def symmetry_looking(x, param):  # :299-321
    gap = np.abs(np.mean(x) - np.median(x))
    span = np.max(x) - np.min(x)
    return [gap < p["r"] * span for p in param]


@simple
def has_duplicate_max(x):  # :325-336
    return np.sum(x == np.max(x)) >= 2


@simple
def has_duplicate_min(x):  # :340-351
    return np.sum(x == np.min(x)) >= 2


@simple
def has_duplicate(x):  # :355-366
    return x.size != np.unique(x).size


@simple
def sum_values(x):  # :371-383
    return np.sum(x) if len(x) else 0


@simple
def abs_energy(x):  # :548-563
    return np.dot(x, x)


@simple
def cid_ce(x, normalize):  # :567-600
    if normalize:
        s = np.std(x)
        if s == 0:
            return 0.0
        x = (x - np.mean(x)) / s
    d = np.diff(x)
    return np.sqrt(np.dot(d, d))


@simple
def mean_abs_change(x):  # :604-620
    return np.mean(np.abs(np.diff(x)))


@simple
def mean_change(x):  # :624-640
    return (x[-1] - x[0]) / (len(x) - 1) if len(x) > 1 else NAN


@simple
def mean_second_derivative_central(x):  # :644-658
    return (x[-1] - x[-2] - x[1] + x[0]) / (2 * (len(x) - 2)) if len(x) > 2 else NAN


@simple
def median(x):  # :663-672
    return np.median(x)


@simple
def mean(x):  # :677-686
    return np.mean(x)


@simple
def length(x):  # :691-700
    return len(x)


@simple
def standard_deviation(x):  # :705-714
    return np.std(x)


@simple
def variation_coefficient(x):  # :718-730
    m = np.mean(x)
    return np.std(x) / m if m != 0 else NAN


@simple
def variance(x):  # :735-744
    return np.var(x)


@simple
def skewness(x):  # :749-761 (pandas bias-corrected G1)
    return pd.Series(x).skew(skipna=False)


@simple
def kurtosis(x):  # :766-778 (pandas bias-corrected G2)
    return pd.Series(x).kurtosis()


@simple
def root_mean_square(x):  # :783-792
    return np.sqrt(np.mean(np.square(x))) if len(x) else NAN


@simple
def absolute_sum_of_changes(x):  # :796-809
    return np.sum(np.abs(np.diff(x)))


@simple
def longest_strike_below_mean(x):  # :813-824
    return max(_runs_of_true(x < np.mean(x))) if x.size else 0


@simple
def longest_strike_above_mean(x):  # :828-839
    return max(_runs_of_true(x > np.mean(x))) if x.size else 0


@simple
def count_above_mean(x):  # :843-853
    return int(np.count_nonzero(x > np.mean(x)))


@simple
def count_below_mean(x):  # :857-867
    return int(np.count_nonzero(x < np.mean(x)))


@simple
def last_location_of_maximum(x):  # :871-882
    return 1.0 - np.argmax(x[::-1]) / len(x) if len(x) else NAN


@simple
def first_location_of_maximum(x):  # :886-898
    return np.argmax(x) / len(x) if len(x) else NAN


@simple
def last_location_of_minimum(x):  # :902-913
    return 1.0 - np.argmin(x[::-1]) / len(x) if len(x) else NAN


@simple
def first_location_of_minimum(x):  # :917-929
    return np.argmin(x) / len(x) if len(x) else NAN


# ------------------------------------------------------------------ class S : needs a sorted copy
@simple
def percentage_of_reoccurring_values_to_all_values(x):  # :933-956
    if len(x) == 0:
        return NAN
    _, c = np.unique(x, return_counts=True)
    return np.sum(c > 1) / float(c.shape[0]) if c.shape[0] else 0.0


@simple
def percentage_of_reoccurring_datapoints_to_all_datapoints(x):  # :961-988
    if len(x) == 0:
        return NAN
    vc = pd.Series(x).value_counts()
    tot = vc[vc > 1].sum()
    return 0.0 if np.isnan(tot) else tot / len(x)


@simple
def sum_of_reoccurring_values(x):  # :992-1016
    u, c = np.unique(x, return_counts=True)
    return np.sum((c > 1) * u)


@simple
def sum_of_reoccurring_data_points(x):  # :1020-1041
    u, c = np.unique(x, return_counts=True)
    c = np.where(c < 2, 0, c)
    return np.sum(c * u)


@simple
def ratio_value_number_to_time_series_length(x):  # :1045-1063
    return np.unique(x).size / x.size if x.size else NAN


@simple
def quantile(x, q):  # :1963-1976
    return np.quantile(x, q) if len(x) else NAN


@simple
def mean_n_absolute_max(x, number_of_maxima):  # :1643-1662
    top = np.sort(np.absolute(x))[-number_of_maxima:]
    return np.mean(top) if len(x) > number_of_maxima else NAN


@simple
def change_quantiles(x, ql, qh, isabs, f_agg):  # :1511-1553
    if ql >= qh:
        return 0.0
    d = np.diff(x)
    if isabs:
        d = np.abs(d)
    try:
        inside = pd.qcut(x, [ql, qh], labels=False) == 0
    except ValueError:
        return 0.0
    both = (inside & _cyc(inside, 1))[1:]
    if np.sum(both) == 0:
        return 0.0
    return getattr(np, f_agg)(d[np.where(both == 1)])


def friedrich_points(x, r):  # :131-170
    """the (signal mean, delta mean) of every non-empty quantile bin, or None where pd.qcut fails"""
    frame = pd.DataFrame({"signal": x[:-1], "delta": np.diff(x)})
    try:
        frame["q"] = pd.qcut(frame.signal, r)
    except (ValueError, IndexError):
        return None
    g = frame.groupby("q", observed=False)
    return pd.DataFrame({"xm": g.signal.mean(), "ym": g.delta.mean()}).dropna()


def _friedrich_fit(x, m, r):  # :131-173
    pts = friedrich_points(x, r)
    if pts is None:
        return [NAN] * (m + 1)
    try:
        return np.polyfit(pts.xm, pts.ym, deg=m)
    except (np.linalg.LinAlgError, ValueError):
        return [NAN] * (m + 1)


@combiner
def friedrich_coefficients(x, param):  # :2082-2130
    cache, res = {}, {}
    for p in param:
        key = (p["m"], p["r"])
        if key not in cache:
            cache[key] = _friedrich_fit(x, p["m"], p["r"])
        try:
            res[(p["coeff"], p["m"], p["r"])] = cache[key][p["coeff"]]
        except IndexError:
            res[(p["coeff"], p["m"], p["r"])] = NAN
    return list(res.values())          # dict result: duplicate keys collapse (:2126-2130)


@simple
def max_langevin_fixed_point(x, r, m):  # :2134-2167
    c = _friedrich_fit(x, m, r)
    try:
        return np.max(np.real(np.roots(c)))
    except (np.linalg.LinAlgError, ValueError):
        return NAN


# ------------------------------------------------------------------ autocorrelation family
@combiner
def agg_autocorrelation(x, param):  # :387-436
    n = len(x)
    top = max(p["maxlag"] for p in param)
    if np.abs(np.var(x)) < 10 ** -10 or n == 1:
        a = [0] * n
    else:
        a = tp.acf(x, adjusted=True, fft=n > 1250, nlags=top)[1:]
    return [getattr(np, p["f_agg"])(a[: int(p["maxlag"])]) for p in param]


@combiner
def partial_autocorrelation(x, param):  # :440-495
    want = max(p["lag"] for p in param)
    n = len(x)
    if n <= 1:
        c = [NAN] * (want + 1)
    else:
        use = n // 2 - 1 if want >= n // 2 else want
        if use > 0:
            c = list(tp.pacf(x, method="ld", nlags=use)) + [NAN] * max(0, want - use)
        else:
            c = [NAN] * (want + 1)
    return [c[p["lag"]] for p in param]


@combiner
def augmented_dickey_fuller(x, param):  # :499-544
    cache, out = {}, []
    for p in param:
        al = p.get("autolag", "AIC")
        if al not in cache:
            try:
                cache[al] = tp.adfuller(x, autolag=al)
            except (np.linalg.LinAlgError, ValueError, tp.MissingDataError):
                cache[al] = (NAN, NAN, NAN)
        idx = {"teststat": 0, "pvalue": 1, "usedlag": 2}.get(p["attr"])
        out.append(NAN if idx is None else cache[al][idx])
    return out


@simple
def autocorrelation(x, lag):  # :1919-1959
    if len(x) < lag:
        return NAN
    mu = np.mean(x)
    num = np.sum((x[: len(x) - lag] - mu) * (x[lag:] - mu))
    v = np.var(x)
    if np.isclose(v, 0):
        return NAN
    return num / ((len(x) - lag) * v)


@combiner
def ar_coefficient(x, param):  # :1459-1507
    fits, res = {}, {}
    for p in param:
        k, c = p["k"], p["coeff"]
        if k not in fits:
            try:
                fits[k] = tp.AutoReg(list(x), lags=k, trend="c").fit().params
            except (ZeroDivisionError, np.linalg.LinAlgError, ValueError):
                fits[k] = [NAN] * k
        if c <= k:
            try:
                res[(c, k)] = fits[k][c]
            except IndexError:
                res[(c, k)] = 0
        else:
            res[(c, k)] = NAN
    return list(res.values())          # the reference returns list(res.items()): duplicate keys collapse


@simple
def time_reversal_asymmetry_statistic(x, lag):  # :1557-1596
    n = len(x)
    if 2 * lag >= n:
        return 0.0
    a, b, c = x[: n - 2 * lag], x[lag: n - lag], x[2 * lag:]
    return np.mean(c * c * b - b * a * a)


@simple
def c3(x, lag):  # :1600-1639
    n = x.size
    if 2 * lag >= n:
        return 0.0
    return np.mean(x[2 * lag:] * x[lag: n - lag] * x[: n - 2 * lag])


# ------------------------------------------------------------------ spectral
@combiner
def fft_coefficient(x, param):  # :1067-1119
    f = np.fft.rfft(x)
    pick = {"real": lambda z: z.real, "imag": lambda z: z.imag, "abs": np.abs,
            "angle": lambda z: np.angle(z, deg=True)}
    return [pick[p["attr"]](f[p["coeff"]]) if p["coeff"] < len(f) else NAN for p in param]


@combiner
def fft_aggregated(x, param):  # :1123-1231
    y = np.abs(np.fft.rfft(x))
    k = np.arange(len(y), dtype=float)

    def mom(j):
        return y.dot(k ** j) / y.sum()

    def var():
        return mom(2) - mom(1) ** 2

    def skew():
        v = var()
        if v < 0.5:
            return NAN
        c = mom(1)
        return (mom(3) - 3 * c * v - c ** 3) / var() ** 1.5

    def kurt():
        v = var()
        if v < 0.5:
            return NAN
        c = mom(1)
        # the reference's expression ends in "- 3 * centroid" (:1213-1218); restated as is
        return (mom(4) - 4 * c * mom(3) + 6 * mom(2) * c ** 2 - 3 * c) / var() ** 2

    table = {"centroid": lambda: mom(1), "variance": var, "skew": skew, "kurtosis": kurt}
    with np.errstate(all="ignore"):
        return [table[p["aggtype"]]() for p in param]


@combiner
def spkt_welch_density(x, param):  # :1418-1455
    _, pxx = welch(x, nperseg=min(len(x), 256))
    return [pxx[p["coeff"]] if p["coeff"] < len(pxx) else NAN for p in param]


@simple
def binned_entropy(x, max_bins):  # :1666-1694
    if np.isnan(x).any():
        return NAN
    h, _ = np.histogram(x, bins=max_bins)
    p = h / x.size
    p[p == 0] = 1.0
    return -np.sum(p * np.log(p))


@simple
def fourier_entropy(x, bins):  # :1809-1821
    _, pxx = welch(x, nperseg=min(len(x), 256))
    return binned_entropy(pxx / np.max(pxx), bins)


@combiner
def cwt_coefficients(x, param):  # :1370-1414
    cache, out = {}, []
    for p in param:
        widths = tuple(p["widths"])
        if widths not in cache:
            cache[widths], _ = tp.cwt(x, widths, "mexh")
        mat = cache[widths]
        out.append(NAN if mat.shape[1] <= p["coeff"] else mat[widths.index(p["w"]), p["coeff"]])
    return out


def _ricker(points, a):  # :1307-1316
    v = np.arange(0, points) - (points - 1.0) / 2
    return 2 / (np.sqrt(3 * a) * (np.pi ** 0.25)) * (1 - v ** 2 / a ** 2) * np.exp(-(v ** 2) / (2 * a ** 2))


@simple
def number_cwt_peaks(x, n):  # :1320-1339
    return len(find_peaks_cwt(vector=x, widths=np.array(list(range(1, n + 1))), wavelet=_ricker))


# ------------------------------------------------------------------ order-dependent streams
@simple
def number_peaks(x, n):  # :1235-1271
    core = x[n:-n]
    ok = None
    for i in range(1, n + 1):
        left = core > _cyc(x, i)[n:-n]
        ok = left if ok is None else ok & left
        ok &= core > _cyc(x, -i)[n:-n]
    return np.sum(ok)


@combiner
def index_mass_quantile(x, param):  # :1275-1304
    a = np.abs(x)
    s = np.sum(a)
    if s == 0:
        return [NAN for _ in param]
    cm = np.cumsum(a) / s
    return [(np.argmax(cm >= p["q"]) + 1) / len(x) for p in param]


@combiner
def linear_trend(x, param):  # :1343-1366
    lr = linregress(range(len(x)), x)
    return [getattr(lr, p["attr"]) for p in param]


def linear_trend_timewise(x, times_ns, param):  # :2274-2306; times_ns: the series' DatetimeIndex as int64 nanoseconds
    ix = pd.DatetimeIndex(np.asarray(times_ns, dtype="datetime64[ns]"))
    times_hours = np.asarray((ix - ix[0]).total_seconds() / float(3600))
    lr = linregress(times_hours, np.asarray(x, dtype=np.float64))
    return [getattr(lr, p["attr"]) for p in param]


@combiner
def agg_linear_trend(x, param):  # :2171-2222 with _aggregate_on_chunks :176-193
    cache, out = {}, []
    for p in param:
        cl, fa = p["chunk_len"], p["f_agg"]
        if cl >= len(x):
            out.append(NAN)
            continue
        if (fa, cl) not in cache:
            agg = [getattr(x[i * cl:(i + 1) * cl], fa)() for i in range(int(np.ceil(len(x) / cl)))]
            cache[(fa, cl)] = linregress(range(len(agg)), agg)
        out.append(getattr(cache[(fa, cl)], p["attr"]))
    return out


@combiner
def energy_ratio_by_chunks(x, param):  # :2226-2268
    total = np.sum(x ** 2)
    out = []
    for p in param:
        assert p["segment_focus"] < p["num_segments"] and p["num_segments"] > 0
        if total == 0:
            out.append(NAN)
        else:
            out.append(np.sum(np.array_split(x, p["num_segments"])[p["segment_focus"]] ** 2.0) / total)
    return out


@simple
def number_crossing_m(x, m):  # :1980-1998
    return np.where(np.diff(x > m))[0].size


@simple
def maximum(x):  # :2003-2012
    return np.max(x)


@simple
def absolute_maximum(x):  # :2017-2026
    return np.max(np.absolute(x)) if len(x) else NAN


@simple
def minimum(x):  # :2031-2040
    return np.min(x)


@simple
def value_count(x, value):  # :2044-2061
    if np.isnan(value):
        return np.isnan(x).sum()
    return x[x == value].size


@simple
def range_count(x, min, max):  # :2065-2078
    return np.sum((x >= min) & (x < max))


@simple
def count_above(x, t):  # :2309-2321
    return np.sum(x >= t) / len(x)


@simple
def count_below(x, t):  # :2325-2337
    return np.sum(x <= t) / len(x)


@simple
def benford_correlation(x):  # :2341-2380
    digits = np.array([int(str(np.format_float_scientific(v))[:1]) for v in np.abs(np.nan_to_num(x))])
    law = np.array([np.log10(1 + 1 / d) for d in range(1, 10)])
    seen = np.array([(digits == d).mean() for d in range(1, 10)])
    with np.errstate(all="ignore"):
        return np.corrcoef(law, seen)[0, 1]


# ------------------------------------------------------------------ class Q / SEQ
def _windows(x, width, step=1):  # :196-219
    count = (len(x) - width) // step + 1
    idx = np.arange(width)[None, :] + (step * np.arange(count))[:, None]
    return np.asarray(x)[idx]


@simple
def sample_entropy(x):  # :1701-1754
    if np.isnan(x).any():
        return NAN
    tol = 0.2 * np.std(x)
    with np.errstate(all="ignore"):
        w2 = _windows(x, 2)
        B = np.sum([np.sum(np.abs(w - w2).max(axis=1) <= tol) - 1 for w in w2])
        w3 = _windows(x, 3)
        A = np.sum([np.sum(np.abs(w - w3).max(axis=1) <= tol) - 1 for w in w3])
        return -np.log(A / B)


APEN_BLOCK_ELEMENTS = 1 << 22      # float64 elements of one block of the pairwise distance matrix (32 MB)


def _apen_counts(w, r, block_cols):
    """counts[j] = #{i : max_k |w[i, k] - w[j, k]| <= r}, evaluated on [n x block_cols] slices of the distance matrix
    (None: the whole [n x n x mm] array at once, as the reference does).  The maximum of the absolute differences is
    exact in any order, so every block size gives the same integer counts."""
    n = len(w)
    if block_cols is None:
        return np.sum(np.max(np.abs(w[:, None] - w[None, :]), axis=2) <= r, axis=0)
    counts = np.empty(n, dtype=np.int64)
    for j0 in range(0, n, block_cols):
        j1 = min(n, j0 + block_cols)
        d = np.abs(w[:, 0, None] - w[None, j0:j1, 0])
        for k in range(1, w.shape[1]):
            np.maximum(d, np.abs(w[:, k, None] - w[None, j0:j1, k]), out=d)
        counts[j0:j1] = np.sum(d <= r, axis=0)
    return counts


def approximate_entropy_blocked(x, m, r, block_cols=0):
    """approximate_entropy with the match counts taken over column blocks of the distance matrix; block_cols=0 sizes
    the blocks to APEN_BLOCK_ELEMENTS, None forms the full N x N x m array (the reference's memory footprint)."""
    N = x.size
    r = r * np.std(x)
    if r < 0:
        raise ValueError("Parameter r must be positive.")
    if N <= m + 1:
        return 0

    def phi(mm):
        w = np.array([x[i:i + mm] for i in range(N - mm + 1)])
        cols = block_cols if block_cols is None or block_cols > 0 else max(1, APEN_BLOCK_ELEMENTS // len(w))
        C = _apen_counts(w, r, cols) / (N - mm + 1)
        return np.sum(np.log(C)) / (N - mm + 1.0)

    return np.abs(phi(m) - phi(m + 1))


@simple
def approximate_entropy(x, m, r):  # :1759-1805
    return approximate_entropy_blocked(x, m, r)


@simple
def lempel_ziv_complexity(x, bins):  # :1825-1862
    edges = np.linspace(np.min(x), np.max(x), bins + 1)[1:]
    seq = np.searchsorted(edges, x, side="left")
    seen, n, i, w = set(), len(seq), 0, 1
    while i + w <= n:
        piece = tuple(seq[i:i + w])
        if piece in seen:
            w += 1
        else:
            seen.add(piece)
            i += w
            w = 1
    return len(seen) / n


@simple
def permutation_entropy(x, tau, dimension):  # :1866-1915
    if len(x) < dimension:
        return NAN
    W = _windows(x, dimension, tau)
    if len(W) == 0:
        return NAN
    ranks = np.argsort(np.argsort(W))
    _, c = np.unique(ranks, axis=0, return_counts=True)
    p = c / len(ranks)
    return -np.sum(p * np.log(p))


@combiner
def query_similarity_count(x, param):  # :2475-2521 (default query=None -> NaN; stumpy never reached)
    out = []
    for p in param:
        q = np.asarray(p.get("query", None)).astype(float)
        if q.size >= 3:
            raise NotImplementedError("query_similarity_count with a real query needs stumpy (absent)")
        out.append(NAN)
    return out


FCTYPE = {**{k: "simple" for k in SIMPLE}, **{k: "combiner" for k in COMBINER}}


def evaluate(name, x, params):
    """All values of calculator `name` on float64 array `x` for the settings entry `params`
    (None or a list of dicts), in the column order of extraction.py:363-378."""
    x = np.asarray(x, dtype=np.float64)
    if name in COMBINER:
        return [float(v) for v in COMBINER[name](x, params)]
    fn = SIMPLE[name]
    if params:
        return [float(fn(x, **p)) for p in params]
    return [float(fn(x))]
