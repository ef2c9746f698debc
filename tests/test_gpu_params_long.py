"""User-chosen parameter values on long series: every kernel variant, every parameter limit, against the oracle.

tests/test_gpu_params.py runs parameter values away from the ComprehensiveFCParameters grid, but only on series of at most
256 samples (the compact kernels), where its larger values are past the end of the series and both sides return NaN.
tests/test_gpu_variants.py and tests/test_gpu_long_series.py reach every other variant, with the Comprehensive and
Efficient grids only.  This module crosses the two:

  * settings(group, n): one parameter set per kernel group, built from the longest series n of the call -- lags on both
    sides of 64 (where the lag products leave the tensor-core path) up to min(n - 2, 4096), FFT coefficients around n / 2,
    CWT coefficients n - 1 and n, window and chunk parameters on both sides of n / 2 and n, AR orders up to 32, every ADF
    autolag mode, Lempel-Ziv alphabets up to 65 535 symbols, nine change_quantiles corridors, Friedrich r up to 256 ...;
  * CASES: each set in one call per length class (CSR, with 1-5, 33, 255 and 257-sample series, a constant and a walk in
    the same call; dense at a length that is no multiple of 4, and at 32 768), the classes chosen per group so that every
    general variant runs, and for every group but ENTROPY past 21 000 samples up to 131 072;
  * heavy() / HEAVY_BOUNDS: plans whose working set moves the variant bounds of tests/test_gpu_variants.py:BOUNDS, compared
    on both sides of every moved bound -- a call just under the shared-to-global bound must run;
  * limits: the largest accepted value of every limited parameter matches the oracle, the first refused one raises at
    plan creation, before any launch, and the context extracts correctly afterwards;
  * ledger: every general variant of the seven groups was reached here, by a plan that is not a grid.

Comparisons are those of tests/test_gpu_variants.py: atol 0 on random and random-walk rows, NOISE_FLOOR on degenerate
ones; waivers in _waived, each decided from the data.  All oracle rows of the module come from one pool pass."""
import os
import sys

import numpy as np
import pytest

from tests.helpers import to_csr
from tests.test_gpu_variants import TIED, _report, check, oracle
from tsfresh_b200.plan import MAX_LAG, Plan

pytestmark = pytest.mark.gpu
L_MAX = 131072
GROUPS = ("basic", "sorted", "spectral", "la", "entropy", "seq", "peaks")
REPORTED = set()


# ---------------------------------------------------------------------------------------------- parameter sets
def _lags(n, limit=None):
    """both sides of lag 64, a third of the series, the largest lag inside it, one past its end; none above `limit`"""
    return sorted(l for l in {1, 63, 64, 65, n // 3, n - 2, n + 3, limit or 1} if not limit or l <= limit)


def _around(n):
    """both sides of n / 2 and of n"""
    return sorted({n // 2 - 1, n // 2, n // 2 + 1, n - 1, n, n + 1})


CORRIDORS = ((0.0, 1.0), (0.3, 0.3), (0.9, 0.2), (0.1, 0.11), (0.45, 0.55), (0.0, 0.2), (0.8, 1.0), (0.25, 0.75), (0.05, 0.95))


def settings(group, n, reduced=False):
    """the non-grid parameter set of one kernel group for a call whose longest series has n samples; `reduced` keeps the
    values whose oracle is affordable at 131 072 samples"""
    if group == "basic":
        around = [1, 7] + ([] if reduced else _around(n))
        return {
            "ratio_beyond_r_sigma": [{"r": r} for r in (0.0, 0.25, 3.3)],
            "large_standard_deviation": [{"r": r} for r in (0.01, 0.33)],
            "cid_ce": [{"normalize": True}, {"normalize": False}],
            "autocorrelation": [{"lag": l} for l in _lags(n, MAX_LAG)],
            "agg_autocorrelation": [{"f_agg": f, "maxlag": m} for f in ("mean", "median", "var", "std")
                                    for m in (1, 64, 150, min(n - 2, MAX_LAG))],
            "partial_autocorrelation": [{"lag": l} for l in (0, 1, 5, 45, 200)],
            "number_peaks": [{"n": v} for v in around],
            "binned_entropy": [{"max_bins": b} for b in (1, 7, 1000, 5000)],
            "index_mass_quantile": [{"q": q} for q in (0.0, 0.001, 0.5, 0.999, 1.0)],
            "value_count": [{"value": v} for v in (0.5, 2, float("nan"))],
            "range_count": [{"min": -0.5, "max": 0.5}, {"min": 1, "max": -1}, {"min": -1e30, "max": 1e30}],
            "number_crossing_m": [{"m": m} for m in (0.3, -2.5, 100)],
            "count_above": [{"t": t} for t in (-1, 0.5, 10)],
            "count_below": [{"t": t} for t in (-1, 0.5, 10)],
            "time_reversal_asymmetry_statistic": [{"lag": l} for l in _lags(n) + [n // 2]],
            "c3": [{"lag": l} for l in _lags(n) + [n // 2]],
            "energy_ratio_by_chunks": [{"num_segments": s, "segment_focus": f} for s in [3] + _around(n) for f in (0, s - 1)],
            "linear_trend": [{"attr": a} for a in ("slope", "pvalue")],
            "agg_linear_trend": [{"attr": a, "chunk_len": c, "f_agg": f} for a in ("pvalue", "slope", "stderr")
                                 for c in [3, 66] + _around(n) for f in ("max", "mean", "var")],
        }
    if group == "basic_light":       # no 4096-lag products, 200-lag pacf or 5 000 bins: several warps per CTA past 256 samples
        full = settings("basic", n, reduced)
        return dict(full, autocorrelation=[{"lag": l} for l in (1, 63, 64, 65, 100)],
                    agg_autocorrelation=[{"f_agg": f, "maxlag": m} for f in ("mean", "median", "var", "std") for m in (64, 100)],
                    partial_autocorrelation=[{"lag": l} for l in (0, 1, 5)],
                    binned_entropy=[{"max_bins": b} for b in (7, 100)])
    if group == "spectral_light":    # at most 500 fourier_entropy bins
        return dict(settings("spectral", n), fourier_entropy=[{"bins": b} for b in (1, 17, 500)])
    if group == "la_light":          # AR orders up to 16
        return dict(settings("la", n), ar_coefficient=[{"coeff": c, "k": k} for k in (1, 15, 16) for c in (0, k, k + 1)])
    if group == "sorted":
        return {
            "symmetry_looking": [{"r": r} for r in (0.0, 0.013, 0.5)],
            "has_duplicate": None, "median": None, "sum_of_reoccurring_values": None,
            "percentage_of_reoccurring_datapoints_to_all_datapoints": None,
            "quantile": [{"q": q} for q in (0.0, 0.01, 0.5, 0.999, 1.0)],
            "mean_n_absolute_max": [{"number_of_maxima": k} for k in [1, 50] + _around(n)],
            "change_quantiles": [{"ql": ql, "qh": qh, "isabs": b, "f_agg": f} for ql, qh in CORRIDORS
                                 for b in (False, True) for f in ("mean", "var")],
            "friedrich_coefficients": [{"coeff": c, "m": 3, "r": r} for r in (2, 30, 100, 256) for c in (0, 3, 4)],
            "max_langevin_fixed_point": [{"m": 3, "r": r} for r in (5, 256)],
        }
    if group == "spectral":
        return {
            "fft_coefficient": [{"coeff": k, "attr": a} for a in ("real", "imag", "abs", "angle")
                                for k in (0, 1, 100, n // 2 - 1, n // 2, n // 2 + 1)],
            "fft_aggregated": [{"aggtype": s} for s in ("centroid", "variance", "skew", "kurtosis")],
            "spkt_welch_density": [{"coeff": c} for c in (0, 128, 129)],
            "fourier_entropy": [{"bins": b} for b in (1, 17, 500, 5000)],
            "cwt_coefficients": [{"widths": w, "coeff": c, "w": s} for w in ((1, 3), (2, 7, 30), (50,)) for s in w
                                 for c in (0, n - 1, n)],
        }
    if group == "la":
        return {
            "ar_coefficient": [{"coeff": c, "k": k} for k in (1, 15, 16, 32) for c in (0, k, k + 1)],
            "augmented_dickey_fuller": [{"attr": a, "autolag": al} for al in (("BIC",) if reduced else ("AIC", "BIC", None))
                                        for a in ("teststat", "pvalue", "usedlag")],
        }
    if group == "entropy":
        return {"approximate_entropy": [{"m": 2, "r": r} for r in (0.0, 0.05, 1.0, 3.0)], "sample_entropy": None}
    if group == "seq":
        return {"lempel_ziv_complexity": [{"bins": b} for b in (1, 2, 127, 128, 1000, 65535)],
                "permutation_entropy": [{"tau": t, "dimension": d} for t in (1, 5, 50) for d in (3, 7, 8)]}
    if group == "seq_perm":        # no Lempel-Ziv tables: the general SEQ kernel's working set stays in shared memory
        return {"permutation_entropy": settings("seq", n)["permutation_entropy"]}
    if group == "peaks":
        return {"number_cwt_peaks": [{"n": v} for v in ((16,) if reduced else (1, 8, 16))]}
    raise KeyError(group)


# ---------------------------------------------------------------------------------------------- series
def _rng_series(n, seed, walk):
    x = np.random.default_rng(seed).standard_normal(n)
    return (x.cumsum() if walk else x).astype(np.float32)


def short_series(seed):
    """(series, degenerate) next to the long ones: 1-5, 33, 255 and 257 samples of N(0, 1), a constant, a walk"""
    out = [(_rng_series(n, seed + n, False), n <= 5) for n in (1, 2, 3, 4, 5, 33, 255, 257)]
    return out + [(np.full(40, 2.5, np.float32), TIED), (_rng_series(100, seed, True), False)]


def call_series(n, dense, seed, count=2):
    """(series, degenerate flags, rows that are random walks) of one call: `count` series of n samples, normal and walk
    in turn, with the short ones (CSR) or a constant row (dense)"""
    series = [_rng_series(n, seed + i, walk=i % 2 == 1) for i in range(count)]
    walks = {i for i in range(count) if i % 2 == 1}
    if dense:
        return series + [np.full(n, 2.5, np.float32)], [False] * count + [TIED], walks
    extra = short_series(seed)
    return series + [s for s, _ in extra], [False] * count + [d for _, d in extra], walks | {len(series) + len(extra) - 1}


# group -> [(case, longest series, dense, series of that length, reduced set, variant the call must run)]; the variants
# follow from the launchers' arithmetic for these plans and were confirmed on an H100 with Context.last_kernels().
# basic_light, spectral_light, la_light and seq_perm are lighter non-grid plans: the full sets need more shared memory
# per warp than the 8- and 4-warp geometries have at any length past the compact kernels' 256 samples.
def _c(n, variant, dense=False, count=2, reduced=False):
    return ("%s_%d" % ("dense" if dense else "csr", n), n, dense, count, reduced, variant)


LENGTHS = {
    "basic": [_c(300, "basic/w1/shared"), _c(700, "basic/w1/shared"), _c(5000, "basic/w1/shared"),
              _c(12000, "basic/w4/global"), _c(24001, "basic/w4/global"), _c(1301, "basic/w1/shared", True),
              _c(32768, "basic/w4/global", True), _c(L_MAX, "basic/w4/global", count=1, reduced=True)],
    "basic_light": [_c(258, "basic/w12/shared"), _c(700, "basic/w4/shared"), _c(1500, "basic/w2/shared")],
    "sorted": [_c(300, "sorted/w8/shared"), _c(700, "sorted/w4/shared"), _c(3000, "sorted/w2/shared"),
               _c(5000, "sorted/w1/shared"), _c(12000, "sorted/w1/shared"), _c(24001, "sorted/w4/global"),
               _c(1301, "sorted/w4/shared", True), _c(32768, "sorted/w4/global", True), _c(L_MAX, "sorted/w4/global", count=1)],
    "spectral": [_c(700, "spectral/w2/shared"), _c(5000, "spectral/w1/shared"), _c(12000, "spectral/w4/global"),
                 _c(24001, "spectral/w4/global"), _c(1301, "spectral/w1/shared", True), _c(2048, "spectral/pow2/w2/shared", True),
                 _c(8192, "spectral/pow2/w1/shared", True), _c(32768, "spectral/pow2/w4/global", True),
                 _c(L_MAX, "spectral/w4/global", count=1)],
    "spectral_light": [_c(300, "spectral/w8/shared"), _c(700, "spectral/w4/shared"), _c(512, "spectral/pow2/w8/shared", True),
                       _c(1024, "spectral/pow2/w4/shared", True)],
    "la": [_c(300, "la/w4/shared"), _c(700, "la/w2/shared"), _c(5000, "la/w1/shared"), _c(12000, "la/w4/global"),
           _c(24001, "la/w4/global"), _c(1301, "la/w2/shared", True), _c(32768, "la/w4/global", True),
           _c(L_MAX, "la/w4/global", count=1, reduced=True)],
    "la_light": [_c(300, "la/w8/shared")],
    "entropy": [_c(300, "entropy/rank-g4"), _c(700, "entropy/rank-g16"), _c(1500, "entropy/tiles/w2/shared"),
                _c(5000, "entropy/tiles/w1/shared"), _c(12000, "entropy/tiles/w4/global", count=1),
                _c(1301, "entropy/tiles/w2/shared", True)],
    "seq": [_c(700, "seq/general/w4/global"), _c(5000, "seq/general/w4/global"), _c(12000, "seq/general/w4/global"),
            _c(24001, "seq/general/w4/global"), _c(1301, "seq/general/w4/global", True),
            _c(32768, "seq/general/w4/global", True), _c(L_MAX, "seq/general/w4/global", count=1)],
    "seq_perm": [_c(700, "seq/general/w8/shared"), _c(1500, "seq/general/w4/shared")],
    "peaks": [_c(300, "peaks/general/hybrid/w4/global"), _c(700, "peaks/general/w4/global"),
              _c(5000, "peaks/general/w4/global"), _c(12000, "peaks/general/w4/global"), _c(24001, "peaks/general/w4/global", count=1),
              _c(1301, "peaks/general/w4/global", True), _c(32768, "peaks/general/w4/global", True, count=1),
              _c(L_MAX, "peaks/general/w4/global", count=1, reduced=True)],
}


def _cases():
    out = {}
    for group, rows in LENGTHS.items():
        for name, n, dense, count, reduced, variant in rows:
            series, degenerate, walks = call_series(n, dense, 1000 * len(out) + n, count)
            out[group + "/" + name] = dict(group=group, settings=settings(group, n, reduced), series=series,
                                           degenerate=degenerate, walks=walks, dense=dense, variant=variant)
    return out


CASES = _cases()


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pool():
    import multiprocessing as mp

    from tests.helpers import cores
    threads = ("OMP_NUM_THREADS", "MKL_NUM_THREADS", "OPENBLAS_NUM_THREADS")
    before = {k: os.environ.get(k) for k in threads}
    os.environ.update({k: "1" for k in threads})      # inherited by the workers: one BLAS thread each, set before numpy loads
    try:
        with mp.get_context("spawn").Pool(cores()) as p:
            yield p
    finally:
        for k, v in before.items():
            os.environ.pop(k) if v is None else os.environ.__setitem__(k, v)


def extract(ctx, plan_settings, series, dense=False):
    """(result, kernel variants) of one extract call"""
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(plan_settings))
    try:
        got = dp.extract_dense(np.stack(series)) if dense else dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
    REPORTED.update(kernels)
    return got, kernels


def variant_of(kernels, group):
    prefix = group.split("_")[0] + "/"
    hit = [k for k in kernels if k.startswith(prefix)]
    assert len(hit) == 1, kernels
    return hit[0]


def _waived(bad, series, walks, want, suffixes):
    """mismatches left out, the cells no float64 implementation pins down (the waivers of tests/test_gpu_long_series.py):
      * permutation_entropy on a row with tied windows: the reference's argsort is unstable there;
      * ar_coefficient on a constant series of more than 100 samples: the reference's pinv of the rank-one design returns
        rounding noise at these lengths (the dense calls' constant row; the 40-sample constant of the CSR calls agrees);
      * ar_coefficient on a random walk within 1e-5 of the row's largest coefficient: the lag columns are nearly
        collinear, so coefficients close to 0 carry both solvers' rounding."""
    ar = [c for c, s in enumerate(suffixes) if s.startswith("ar_coefficient")]
    out = []
    for b in bad:
        r, suf, g, w = b
        x = series[r]
        if suf.startswith("permutation_entropy"):
            tau, dim = (int(suf.split(k + "_")[1].split("__")[0]) for k in ("tau", "dimension"))
            if len(x) >= (dim - 1) * tau + 1:
                win = np.sort(np.lib.stride_tricks.sliding_window_view(x, (dim - 1) * tau + 1)[:, ::tau], axis=1)
                if np.any(win[:, 1:] == win[:, :-1]):
                    continue
        if suf.startswith("ar_coefficient") and len(x) > 100 and np.all(x == x[0]):
            continue
        if suf.startswith("ar_coefficient") and r in walks and abs(g - w) <= 1e-5 * np.nanmax(np.abs(want[r][ar])):
            continue
        out.append(b)
    return out


# ---------------------------------------------------------------------------------------------- heavy plans
def heavy(group, n):
    """plans whose working set moves the variant bounds away from those of the Comprehensive plan"""
    if group == "basic":       # lag 4096, a 200-lag pacf, 5 000 bins and 3 010 columns (a 120 KB descriptor table)
        return {"autocorrelation": [{"lag": l} for l in list(range(1, 2801)) + [4096]],
                "partial_autocorrelation": [{"lag": l} for l in range(0, 201)],
                "binned_entropy": [{"max_bins": b} for b in (10, 5000)],
                "agg_linear_trend": [{"attr": "slope", "chunk_len": c, "f_agg": "var"} for c in (5, 50, 500)],
                "c3": [{"lag": l} for l in (1, 2, 3)]}
    if group == "seq":         # eight lempel_ziv_complexity columns: eight lanes of key tables and symbols
        return {"lempel_ziv_complexity": [{"bins": b} for b in (2, 3, 5, 10, 100, 1000, 10000, 65535)]}
    return settings(group, n)  # SORTED: r = 256 and nine corridors; SPECTRAL: 5 000 fourier_entropy bins


# bounds of the heavy plans, (longest series, variant) on both sides: read from the launchers' arithmetic (launch_* in
# tsfresh_b200/csrc/k_*.cu) and confirmed on an H100 with Context.last_kernels().  Compare tests/test_gpu_variants.py:
# BOUNDS -- BASIC leaves shared memory at 1 536 samples instead of 11 116 (47 KB of lag products and a 120 KB descriptor
# table), SORTED drops to four warps at 500 instead of 1 024 (r = 256), SPECTRAL never runs more than two warps
# (20 KB of histogram) and leaves shared memory at 7 548 instead of 8 248.
HEAVY_BOUNDS = {
    "basic": [(1536, "basic/w1/shared"), (1537, "basic/w4/global")],
    "sorted": [(500, "sorted/w8/shared"), (501, "sorted/w4/shared"), (2048, "sorted/w4/shared"), (2049, "sorted/w2/shared"),
               (4096, "sorted/w2/shared"), (4097, "sorted/w1/shared"), (23156, "sorted/w1/shared"), (23157, "sorted/w4/global")],
    "spectral": [(1076, "spectral/w2/shared"), (1077, "spectral/w1/shared"), (7548, "spectral/w1/shared"),
                 (7549, "spectral/w4/global")],
    # alphabets past 127 symbols keep series of at most 256 samples out of the compact kernel
    "seq": [(84, "seq/general/w8/shared"), (85, "seq/general/w4/shared"), (168, "seq/general/w4/shared"),
            (169, "seq/general/w4/global"), (256, "seq/general/w4/global"), (257, "seq/general/w4/global")],
}


def _all_tasks():
    """(key, settings, series) of every oracle row of CASES, costliest first (the entropies are quadratic)"""
    tasks = [((name, i), c["settings"], s) for name, c in CASES.items() for i, s in enumerate(c["series"])]
    cost = lambda t: float(len(t[2])) ** (2 if CASES[t[0][0]]["group"] == "entropy" else 1) * len(Plan(t[1]).suffixes)
    return sorted(tasks, key=cost, reverse=True)


@pytest.fixture(scope="module")
def want(pool):
    """oracle rows of every case of CASES, one pool pass"""
    from tests.test_gpu_variants import _oracle_one
    tasks = _all_tasks()
    rows = dict(zip((k for k, _, _ in tasks), pool.map(_oracle_one, [(st, s) for _, st, s in tasks], chunksize=1)))
    return {name: np.asarray([rows[(name, i)] for i in range(len(c["series"]))]) for name, c in CASES.items()}


def _compare(got, want_rows, plan_settings, series, degenerate, walks):
    suffixes = Plan(plan_settings).suffixes
    return _waived(check(got, want_rows, suffixes, degenerate), series, walks, want_rows, suffixes)


@pytest.mark.parametrize("name", list(CASES))
def test_params_long(ctx, want, name):
    c = CASES[name]
    got, kernels = extract(ctx, c["settings"], c["series"], c["dense"])
    assert variant_of(kernels, c["group"]) == c["variant"], kernels
    bad = _compare(got, want[name], c["settings"], c["series"], c["degenerate"], c["walks"])
    assert not bad, _report(bad)


@pytest.mark.parametrize("group,length,variant", [(g, L, v) for g, cases in HEAVY_BOUNDS.items() for L, v in cases])
def test_heavy_plan_bound(ctx, pool, group, length, variant):
    plan_settings = heavy(group, length)
    series, degenerate, walks = call_series(length, False, 31 * length)
    keep = [i for i, s in enumerate(series) if len(s) <= length]         # `length` is the longest series of the call
    series, degenerate, walks = [series[i] for i in keep], [degenerate[i] for i in keep], {keep.index(i) for i in walks if i in keep}
    got, kernels = extract(ctx, plan_settings, series)
    assert variant_of(kernels, group) == variant, kernels
    bad = _compare(got, oracle(pool, plan_settings, series), plan_settings, series, degenerate, walks)
    assert not bad, _report(bad)


# ---------------------------------------------------------------------------------------------- limits
def _distinct(n, seed):
    """n distinct float32 samples in random order: every Lempel-Ziv alphabet up to n symbols is fully used"""
    return np.random.default_rng(seed).permutation(n).astype(np.float32)


LIMIT_SETTINGS = {      # the largest accepted value of every limited parameter
    "autocorrelation": [{"lag": 4096}], "agg_autocorrelation": [{"f_agg": "var", "maxlag": 4096}],
    "ar_coefficient": [{"coeff": c, "k": 32} for c in (0, 32)], "number_cwt_peaks": [{"n": 16}],
    "friedrich_coefficients": [{"coeff": c, "m": 3, "r": 256} for c in range(4)],
    "max_langevin_fixed_point": [{"m": 3, "r": 256}], "permutation_entropy": [{"tau": 1, "dimension": 8}],
    "lempel_ziv_complexity": [{"bins": 65535}],
}
# the first refused value: (settings refused by the plan compiler, descriptor field that holds the value)
REFUSED = {
    "autocorrelation": ({"autocorrelation": [{"lag": 4097}]}, "i0"),
    "agg_autocorrelation": ({"agg_autocorrelation": [{"f_agg": "mean", "maxlag": 4097}]}, "i0"),
    "partial_autocorrelation": ({"partial_autocorrelation": [{"lag": 4097}]}, "i1"),
    "ar_coefficient": ({"ar_coefficient": [{"coeff": 0, "k": 33}]}, "i1"),
    "number_cwt_peaks": ({"number_cwt_peaks": [{"n": 17}]}, "i0"),
    "friedrich_coefficients": ({"friedrich_coefficients": [{"coeff": 0, "m": 3, "r": 257}]}, "i2"),
    "max_langevin_fixed_point": ({"max_langevin_fixed_point": [{"m": 3, "r": 257}]}, "i2"),
    "permutation_entropy": ({"permutation_entropy": [{"tau": 1, "dimension": 9}]}, "i1"),
    "lempel_ziv_complexity": ({"lempel_ziv_complexity": [{"bins": 65536}]}, "i0"),
}


def test_largest_accepted_values(ctx, pool):
    series, degenerate, walks = call_series(5000, False, 77)
    got, kernels = extract(ctx, LIMIT_SETTINGS, series)
    assert "basic/w1/shared" in kernels, kernels
    bad = _compare(got, oracle(pool, LIMIT_SETTINGS, series), LIMIT_SETTINGS, series, degenerate, walks)
    assert not bad, _report(bad)


def _legal(value):
    """the refused settings with the parameter lowered to a value every calculator accepts"""
    return {k: [dict(p, **{q: 2 for q in p if q in ("lag", "maxlag", "k", "n", "r", "dimension", "bins")}) for p in v]
            for k, v in value.items()}


@pytest.mark.parametrize("name", list(REFUSED))
def test_first_refused_value(ctx, name):
    """refused by the plan compiler, and by tsfx_plan_create when the descriptor reaches it anyway: before any launch,
    and the context extracts correctly afterwards"""
    from oracle.extract import compare, oracle_rows
    from tsfresh_b200._lib import DevicePlan
    refused, field = REFUSED[name]
    with pytest.raises(NotImplementedError):
        Plan(refused)
    x = _rng_series(300, 5, False)
    legal = _legal(refused)
    got, _ = extract(ctx, legal, [x])
    launches = ctx.launch_count()
    assert launches > 0
    plan = Plan(legal)
    plan.descs[field] = _refused_value(refused)
    with pytest.raises(NotImplementedError):
        DevicePlan(ctx, plan)
    assert ctx.launch_count() == launches
    again, _ = extract(ctx, legal, [x])
    np.testing.assert_array_equal(again, got)
    bad = compare(got, oracle_rows([x.astype(np.float64)], legal), Plan(legal).suffixes)
    assert not bad, _report(bad)


def _refused_value(refused):
    (plist,) = refused.values()
    return max(v for k, v in plist[0].items() if k in ("lag", "maxlag", "k", "n", "r", "dimension", "bins"))


LZ_SERIES = {"300": (300, "seq/general/w8/shared"), "20000": (20000, "seq/general/w4/global"),
             "100003": (100003, "seq/general/w4/global")}       # compact table, 32-bit keys, 64-bit keys


@pytest.mark.parametrize("which", list(LZ_SERIES))
def test_lempel_ziv_largest_alphabet(ctx, pool, which):
    """65 535 bins on series of distinct samples: the largest symbol, 65 534, in every key layout.  One bin more and the
    key of the series' maximum at the root would be the 32-bit table's empty-slot marker, any more and the 16-bit symbols
    would wrap: test_first_refused_value has the refusal."""
    n, variant = LZ_SERIES[which]
    plan_settings = {"lempel_ziv_complexity": [{"bins": b} for b in (65535, 65534, 40000)]}
    series = [_distinct(n, n), _rng_series(n, n + 1, False), _distinct(300, 3)]
    got, kernels = extract(ctx, plan_settings, series)
    assert kernels == [variant], kernels
    bad = _compare(got, oracle(pool, plan_settings, series), plan_settings, series, [False] * 3, set())
    assert not bad, _report(bad)


def _basic_columns(count):
    st = {"autocorrelation": [{"lag": l} for l in range(min(count, 4097))]}
    rest = count - 4097
    if rest > 0:
        st["c3"] = [{"lag": l} for l in range(1, rest // 2 + 1)]
        st["time_reversal_asymmetry_statistic"] = [{"lag": l} for l in range(1, rest - rest // 2 + 1)]
    return st


def test_widest_basic_plan(ctx, pool):
    """5 632 BASIC columns, the most one plan may hold (the kernel's descriptor table takes 40 bytes of shared memory per
    column in every placement), match the oracle; one more is refused at plan creation, 7 000 too, before any launch"""
    from tsfresh_b200._lib import DevicePlan
    plan_settings = _basic_columns(5632)
    assert Plan(plan_settings).n_cols == 5632
    series, degenerate, walks = call_series(5000, False, 91, count=1)
    got, kernels = extract(ctx, plan_settings, series)
    assert kernels == ["basic/w4/global"], kernels
    launches = ctx.launch_count()
    bad = _compare(got, oracle(pool, plan_settings, series), plan_settings, series, degenerate, walks)
    assert not bad, _report(bad)
    for count in (5633, 7000):
        with pytest.raises(NotImplementedError, match="columns of the BASIC kernel group"):
            DevicePlan(ctx, Plan(_basic_columns(count)))
        assert ctx.launch_count() == launches
    again, _ = extract(ctx, plan_settings, series)
    np.testing.assert_array_equal(again, got)


# ---------------------------------------------------------------------------------------------- ledger
# compact kernels for series of at most 256 samples (tests/test_gpu_params.py runs non-grid plans through them), the
# reduction-only kernels, and the one-warp global geometries no call selects (tests/test_gpu_variants.py:NOT_REACHED)
NOT_GENERAL = {"moments/dense", "moments/general", "la/small", "entropy/rank-g1", "seq/small",
               "peaks/small"}
N_CASES = len(CASES) + sum(len(v) for v in HEAVY_BOUNDS.values()) + 1 + len(REFUSED) + len(LZ_SERIES) + 1


def test_variant_ledger(request):
    """runs last: every general variant of the seven groups ran in this module, under a plan that is not a grid"""
    from tests.test_gpu_variants import NOT_REACHED
    from tsfresh_b200._lib import kernel_variants
    mine = [i for i in request.session.items if i.module is sys.modules[__name__] and i.name != "test_variant_ledger"]
    if len(mine) < N_CASES:
        pytest.skip("only %d of the %d cases of this module ran" % (len(mine), N_CASES))
    if request.session.testsfailed:
        pytest.skip("some cases failed")
    general = set(kernel_variants()) - NOT_GENERAL - set(NOT_REACHED)
    assert {v.split("/")[0] for v in general} == set(GROUPS)
    assert REPORTED == general, "never reported: %s; not expected: %s" % (sorted(general - REPORTED), sorted(REPORTED - general))
