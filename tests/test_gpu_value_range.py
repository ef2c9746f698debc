"""GPU parity on series with a level and a spread: level + spread * z, cast to float32.

Every other parity test feeds zero-centred data of unit scale, where cancellation against the level cannot show.  Here
the base shapes z (N(0, 1), a 0.3-step random walk, a linear trend plus noise, a sine plus noise, noise rounded to
halves) are shifted to levels of up to 1e4 and scaled by 1e-6 .. 1e6, and ComprehensiveFCParameters is compared with the
oracle (rtol 1e-5, atol 0) in the calls that select the compact variants (<= 256 samples), the general ones
(1 153 .. 1 300 samples, CSR and dense) and, for EfficientFCParameters, the paths past 21 000 samples.  Constant series
at a level are compared in a call of their own with the noise floor scaled by the level: their mean is not exactly
representable, so the reference's variance is rounding noise (DESIGN.md §2).

friedrich_coefficients is compared with the exact fit of the oracle's bin means (tests/helpers.py:polyfit3_accepts):
past a level/spread of ~1e3 np.polyfit itself loses digits, so the oracle is no reference for it there.
max_langevin_fixed_point is compared with the oracle, and with the exact fit's root where the oracle's is off
(friedrich_failures).  Waivers are the existing ones (DESIGN.md §2), decided from the data (_waived)."""
import numpy as np
import pytest

from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from tests.helpers import polyfit3_accepts, pool_map, to_csr
from tsfresh_b200.plan import Plan
from tsfresh_b200.settings import ComprehensiveFCParameters, EfficientFCParameters

pytestmark = pytest.mark.gpu

SHAPES = ("normal", "walk", "trend", "sine", "tied")
SCALES = [(0.0, 1.0), (300.0, 1.0), (1e3, 1.0), (-1e3, 1.0), (1e4, 1.0), (1e4, 30.0), (0.0, 1e-6), (0.0, 1e6)]
SETTINGS = {"comprehensive": ComprehensiveFCParameters, "efficient": EfficientFCParameters}


def base(shape, n, rng):
    t = np.arange(n) / max(n - 1, 1)
    e = rng.standard_normal(n)
    if shape == "normal":
        return e
    if shape == "walk":
        return 0.3 * e.cumsum()
    if shape == "trend":
        return 4.0 * t - 2.0 + 0.3 * e
    if shape == "sine":
        return np.sin(2 * np.pi * 7.3 * t) + 0.3 * e
    if shape == "tied":
        return np.round(2 * e) / 2
    raise ValueError(shape)


def shifted(level, spread, z):
    return (level + spread * z).astype(np.float32)


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def _oracle_row(args):
    name, x = args
    return oracle_rows([np.asarray(x, np.float32).astype(np.float64)], SETTINGS[name]())[0]


def oracle(name, series):
    """oracle rows, one task per series, longest first"""
    order = sorted(range(len(series)), key=lambda i: -len(series[i]))
    rows = pool_map(_oracle_row, [(name, series[i]) for i in order])
    out = [None] * len(series)
    for i, r in zip(order, rows):
        out[i] = r
    return np.asarray(out, np.float64)


def run(ctx, settings, series, dense=False):
    from tsfresh_b200._lib import DevicePlan
    plan = Plan(settings)
    dp = DevicePlan(ctx, plan)
    try:
        got = dp.extract_dense(np.stack(series)) if dense else dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
    return got, kernels, plan


# ---------------------------------------------------------------------------------------------- Friedrich rule
def _max_real_root(c):
    try:
        return np.max(np.real(np.roots(c)))
    except ValueError:                      # no roots: the oracle's NaN
        return np.nan


def _close(a, b):
    return bool(np.isclose(a, b, rtol=1e-5, atol=0) or (np.isnan(a) and np.isnan(b)))


def friedrich_failures(x, got, want, suffixes):
    """Mismatches of the friedrich_coefficients / max_langevin_fixed_point columns of one row:
      * NaN exactly where the oracle has NaN (duplicate qcut edges, no bins), never NaN where it has a number;
      * the coefficients of each r within the perturbation bound of the exact fit, and where that bound is below 1e-7
        within rtol 1e-5 of the oracle, coefficient by coefficient (a coefficient that is exactly 0 has no relative
        accuracy on either side and is left to the bound);
      * max_langevin_fixed_point within rtol 1e-5 of the oracle, or, where the oracle's root is itself more than 1e-5
        from the largest real root of the exact fit, of that root.  A largest root outside the bin means is sensitive
        to the coefficients, and np.polyfit's lose digits at high levels: on a walk at 1e4 (bin means 9 992 .. 9 999,
        r = 5) the oracle gave 10 113.136, the exact fit 10 112.921 (its cubic is -5e-13 there, 4e-2 at the oracle's)."""
    from oracle.calculators import friedrich_points
    x = np.asarray(x, np.float32).astype(np.float64)
    bad = []
    fits, roots = {}, {}
    for j, s in enumerate(suffixes):
        r = int(s.rsplit("__r_", 1)[1])
        if s.startswith("friedrich_coefficients"):
            fits.setdefault(r, [None] * 4)[int(s.split("__coeff_")[1].split("__")[0])] = j
        else:
            roots[r] = j
    exact = {}
    for r, cols in fits.items():
        g, w = got[cols], want[cols]
        if np.isnan(w).all() or np.isnan(g).any():
            if not (np.isnan(w).all() and np.isnan(g).all()):
                bad.append(("friedrich r=%d" % r, list(g), list(w)))
            continue
        pts = friedrich_points(x, r)
        ok, err, bound, ex = polyfit3_accepts(g, pts.xm.to_numpy(np.float64), pts.ym.to_numpy(np.float64))
        exact[r] = [float(v) for v in ex]
        if not ok:
            bad.append(("friedrich r=%d error %.3g bound %.3g" % (r, err, bound), list(g), list(w)))
        elif bound < 1e-7 and not all(_close(a, b) for a, b, e in zip(g, w, ex) if e != 0):
            bad.append(("friedrich r=%d vs oracle (bound %.3g)" % (r, bound), list(g), list(w)))
    for r, j in roots.items():
        if _close(got[j], want[j]):
            continue
        true = _max_real_root(exact[r]) if r in exact else np.nan
        if r not in exact or _close(want[j], true) or not _close(got[j], true):
            bad.append(("max_langevin_fixed_point r=%d (exact fit %r)" % (r, true), got[j], want[j]))
    return bad


def _friedrich_task(args):
    x, got, want, suffixes = args
    return friedrich_failures(x, got, want, suffixes)


def _waived(x, suffix):
    """The existing waivers (DESIGN.md §2), decided from the data: permutation_entropy where a window of its dimension
    holds tied samples (the reference's unstable argsort; float32 rounding ties a 0.3-step walk at level 1e3), and
    number_cwt_peaks on a constant series (one plateau, like the integer plateaus: its CWT rows are mirror-symmetric and
    which of two mirror entries is the larger is rounding)"""
    if suffix.startswith("permutation_entropy"):
        d = int(suffix.split("__dimension_")[1].split("__")[0])
        w = np.sort(np.lib.stride_tricks.sliding_window_view(x, d), axis=1) if len(x) >= d else np.zeros((0, d))
        return bool((np.diff(w, axis=1) == 0).any())
    return suffix.startswith("number_cwt_peaks") and len(x) > 0 and x.min() == x.max()


def check(series, got, want, suffixes, atol=0.0, tied=None):
    """compare() on every column but the Friedrich ones (atol NOISE_FLOOR on the `tied` rows, whose exact zeros the
    reference returns as rounding noise, as in the other tests), the Friedrich rule on those"""
    fr = np.array([s.startswith(("friedrich_coefficients", "max_langevin_fixed_point")) for s in suffixes])
    rest = [j for j in range(len(suffixes)) if not fr[j]]
    tied = np.zeros(len(series), bool) if tied is None else np.asarray(tied, bool)
    bad = []
    for mask, a in ((~tied, atol), (tied, max(atol, NOISE_FLOOR))):
        idx = np.flatnonzero(mask)
        if len(idx):
            bad += [(int(idx[b[0]]),) + b[1:]
                    for b in compare(got[np.ix_(idx, rest)], want[np.ix_(idx, rest)], [suffixes[j] for j in rest], atol=a)
                    if not _waived(series[idx[b[0]]], b[1])]
    if fr.any():
        fsuf = [s for s, f in zip(suffixes, fr) if f]
        per_row = pool_map(_friedrich_task, [(x, g[fr], w[fr], fsuf) for x, g, w in zip(series, got, want)])
        bad += [(i,) + b for i, rb in enumerate(per_row) for b in rb]
    return bad


def _report(bad, tags):
    return "\n".join("row %d (%s) %s: gpu=%r oracle=%r" % ((b[0], tags[b[0]]) + tuple(b[1:])) for b in bad[:40]) + \
        "\n(%d mismatches)" % len(bad)


# ---------------------------------------------------------------------------------------------- Comprehensive sweep
def sweep(lengths, seed):
    """every (shape, level, spread) once per length in `lengths`, with its tag"""
    rng = np.random.default_rng(seed)
    series, tags = [], []
    for shape in SHAPES:
        for level, spread in SCALES:
            for n in lengths:
                series.append(shifted(level, spread, base(shape, n, rng)))
                tags.append("%s level %g spread %g n %d" % (shape, level, spread, n))
    return series, tags


def test_comprehensive_compact(ctx):
    series, tags = sweep((256, 97), 1)
    got, kernels, plan = run(ctx, ComprehensiveFCParameters(), series)
    for v in ("la/small", "seq/small", "peaks/small", "entropy/rank-g1", "basic/w12/shared", "sorted/w8/shared"):
        assert v in kernels, kernels
    bad = check(series, got, oracle("comprehensive", series), plan.suffixes, tied=[t.startswith("tied") for t in tags])
    assert not bad, _report(bad, tags)


@pytest.mark.parametrize("dense", [False, True])
def test_comprehensive_general(ctx, dense):
    series, tags = sweep((1200,) if dense else (1300, 1153), 2 + dense)
    got, kernels, plan = run(ctx, ComprehensiveFCParameters(), series, dense=dense)
    for v in ("la/w2/shared", "seq/general/w4/global", "entropy/tiles/w2/shared", "spectral/w2/shared"):
        assert v in kernels, kernels
    bad = check(series, got, oracle("comprehensive", series), plan.suffixes, tied=[t.startswith("tied") for t in tags])
    assert not bad, _report(bad, tags)


def test_efficient_long_at_a_level(ctx):
    """Bluestein FFT (25 013 samples), 64-bit Lempel-Ziv keys and the sliding noise window of number_cwt_peaks"""
    rng = np.random.default_rng(4)
    series = [shifted(1e3, 1.0, base(s, n, rng)) for s, n in (("walk", 25013), ("normal", 24000), ("sine", 25000))]
    tags = ["walk 25013", "normal 24000", "sine 25000"]
    got, kernels, plan = run(ctx, EfficientFCParameters(), series)
    assert "spectral/w4/global" in kernels and "seq/general/w4/global" in kernels, kernels
    bad = check(series, got, oracle("efficient", series), plan.suffixes)
    assert not bad, _report(bad, tags)


def test_constant_at_a_level(ctx):
    """np.full(n, level) in float32: the reference's variance of a constant whose mean is not representable is rounding
    noise, so these rows are compared with the noise floor scaled by the level"""
    for level in (300.15, -1e3 / 3, 1e4 + 0.1, 65535.0):
        series = [np.full(n, level, np.float32) for n in (2, 5, 100, 256)]
        got, _, plan = run(ctx, ComprehensiveFCParameters(), series)
        bad = check(series, got, oracle("comprehensive", series), plan.suffixes, atol=NOISE_FLOOR * max(1.0, abs(level)))
        # time_reversal_asymmetry_statistic is cubic in the samples: mean(x[i+2l]^2 x[i+l]) - mean(x[i+l] x[i]^2) of a
        # constant c is 0 up to the rounding of two sums of size c^3 (-4.9e-5 at c = 10000.1, 5e-17 of c^3)
        bad = [b for b in bad if not (b[1].startswith("time_reversal_asymmetry_statistic")
                                      and abs(b[2] - b[3]) <= NOISE_FLOOR * max(1.0, abs(level)) ** 3)]
        assert not bad, _report(bad, ["constant %g n %d" % (level, len(s)) for s in series])


# ---------------------------------------------------------------------------------------------- Friedrich
FRIEDRICH_R = (2, 3, 4, 5, 10, 30, 100)
FRIEDRICH = {"friedrich_coefficients": [{"coeff": c, "m": 3, "r": r} for r in FRIEDRICH_R for c in range(4)],
             "max_langevin_fixed_point": [{"m": 3, "r": r} for r in FRIEDRICH_R]}


def _friedrich_oracle(x):
    return oracle_rows([np.asarray(x, np.float32).astype(np.float64)], FRIEDRICH)[0]


def test_friedrich_levels(ctx):
    rng = np.random.default_rng(5)
    series, tags = [], []
    for level in (0.0, 30.0, 100.0, 300.0, 1e3, 3e3, 1e4, -1e3):
        for shape in ("walk", "trend", "normal", "tied"):
            for n in (5, 31, 256, 1000):
                for _ in range(3):
                    series.append(shifted(level, 1.0, base(shape, n, rng)))
                    tags.append("%s level %g n %d" % (shape, level, n))
    got, _, plan = run(ctx, FRIEDRICH, series)
    want = np.asarray(pool_map(_friedrich_oracle, series))
    assert np.isnan(want).any() and not np.isnan(want).all()
    bad = check(series, got, want, plan.suffixes)
    assert not bad, _report(bad, tags)
