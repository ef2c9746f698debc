"""EfficientFCParameters on series longer than 21 000 samples, up to TSFX_L_MAX = 131 072, against the oracle.

Past 21 000 samples the launchers switch to the long-series layouts (DESIGN.md §3): 64-bit Lempel-Ziv keys in SEQ, 32-bit
ridge-line columns and a sliding noise window in PEAKS, a third round of ADF autolag models in LA (from 71 260 samples,
maxlag > 62) and Bluestein's FFT for lengths that are not powers of two in SPECTRAL.  Every case puts 1-5-sample,
constant and tied series in the same call as the long ones, and asserts the variant each group ran.  The ENTROPY group
keeps the 21 000-sample cap, every length error is raised before any group runs, and a plan of BASIC and SORTED
calculators only has no length limit.  number_cwt_peaks also runs on long series with pairs of infinite samples.

Comparisons are those of tests/test_gpu_variants.py: atol 0 on random and random-walk rows, NOISE_FLOOR on degenerate
ones, with the waivers of _waived.  The oracle rows of the whole module come from one pool pass: on an H100 host the
module takes 3.5 to 5 minutes, most of it in the oracle (about 30 s per 131 072-sample series on one core)."""
import numpy as np
import pandas as pd
import pytest

from tests.helpers import to_csr
from tests.test_gpu_variants import TIED, _report, check, oracle, short_and_degenerate
from tsfresh_b200.plan import Plan
from tsfresh_b200.settings import ComprehensiveFCParameters, EfficientFCParameters

pytestmark = pytest.mark.gpu

L_MAX = 131072
CSR_LENGTHS = (21001, 32000, 32001, 71259, 71260, 100003, 131072)
DENSE_LENGTHS = (65536, 131072)
FRAME_LENGTHS = (50000, 131072)          # extract_features on a long frame: one id per length
ROLL_ROWS, ROLL_SHIFT = 40002, 40000     # roll_time_series: two windows of 40 001 samples
AR_COLS = [c for c, s in enumerate(Plan(EfficientFCParameters()).suffixes) if s.startswith("ar_coefficient")]
GLOBAL = {"basic/w4/global", "la/w4/global", "seq/general/w4/global", "peaks/general/w4/global"}


def _long(length, seed, walk):
    x = np.random.default_rng(seed).standard_normal(length)
    return (x.cumsum() if walk else x).astype(np.float32)


def _waived(bad, series, walk_rows, want):
    """mismatches left out of the comparison, the cells no float64 implementation pins down:
      * permutation_entropy on a row with tied windows (a float32 random walk this long has a few equal neighbours):
        the reference's argsort is unstable there, as in tests/test_gpu_variants.py;
      * ar_coefficient on a constant series: the reference's pinv of the rank-one design returns rounding noise at these
        lengths (tests/test_gpu_la.py picks its constants for that reason);
      * ar_coefficient on a random walk within 1e-5 of the row's largest coefficient: the lag columns are nearly
        collinear, so coefficients close to 0 carry both solvers' rounding."""
    out = []
    for b in bad:
        r, suf, g, w = b
        x = series[r]
        if suf.startswith("permutation_entropy") and len(x) >= 8:
            win = np.sort(np.lib.stride_tricks.sliding_window_view(x, 8), axis=1)
            if np.any(win[:, 1:] == win[:, :-1]):
                continue
        if suf.startswith("ar_coefficient") and len(x) > 100:
            if np.all(x == x[0]):
                continue
            if r in walk_rows and abs(g - w) <= 1e-5 * np.nanmax(np.abs(want[r][AR_COLS])):
                continue
        out.append(b)
    return out


def _cases():
    """name -> (series, degenerate flags, dense, random-walk rows).  One long series per CSR call, random-normal and random-walk in turn
    (the oracle takes about 30 s per 131 072-sample series); the dense 131 072 call reuses the CSR call's series."""
    cases = {}
    for i, length in enumerate(CSR_LENGTHS):
        extra = short_and_degenerate("basic", seed=length)
        cases["csr_%d" % length] = ([_long(length, length, walk=i % 2 == 1)] + [s for s, _ in extra],
                                    [False] + [d for _, d in extra], False, {0} if i % 2 else set())
    walk = _long(DENSE_LENGTHS[0], 5, walk=True)
    tied = (np.round(np.random.default_rng(6).standard_normal(DENSE_LENGTHS[0]) * 2) / 2).astype(np.float32)
    cases["dense_%d" % DENSE_LENGTHS[0]] = ([walk, np.full(len(walk), 2.5, np.float32), tied], [False, True, TIED], True, {0})
    x = cases["csr_%d" % L_MAX][0][0]
    cases["dense_%d" % L_MAX] = ([x, np.full(L_MAX, 2.5, np.float32)], [False, True], True, set())
    return cases


CASES = _cases()
FRAME = [_long(FRAME_LENGTHS[0], 11, walk=False), CASES["csr_%d" % L_MAX][0][0]]
ROLL = _long(ROLL_ROWS, 13, walk=True)
ROLL_WINDOWS = [ROLL[e - ROLL_SHIFT:e + 1] for e in range(ROLL_SHIFT, ROLL_ROWS)]


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def want():
    """oracle rows of every series of the module (one pool pass, longest series first, each array once)"""
    import multiprocessing as mp

    from tests.helpers import cores
    groups = [(name, c[0]) for name, c in CASES.items()] + [("frame", FRAME), ("roll", ROLL_WINDOWS)]
    unique = {}
    for _, ss in groups:
        for s in ss:
            unique.setdefault(id(s), s)
    with mp.get_context("spawn").Pool(cores()) as pool:
        rows = dict(zip(unique, oracle(pool, EfficientFCParameters(), list(unique.values()))))
    return {name: np.asarray([rows[id(s)] for s in ss]) for name, ss in groups}


def _extract(ctx, settings, series, dense):
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(settings))
    try:
        got = dp.extract_dense(np.stack(series)) if dense else dp.extract_csr(*to_csr(series))
        return got, ctx.last_kernels()
    finally:
        dp.close()


@pytest.mark.parametrize("name", list(CASES))
def test_efficient_long(ctx, want, name):
    series, degenerate, dense, walk_rows = CASES[name]
    settings = EfficientFCParameters()
    got, kernels = _extract(ctx, settings, series, dense)
    length = len(series[0])
    spectral = "spectral/pow2/w4/global" if dense else "spectral/w4/global"
    # at 21 001 samples SORTED's working set still fits one warp's 227 KB of shared memory, as at 21 000
    sorted_ = "sorted/w1/shared" if length == 21001 else "sorted/w4/global"
    assert set(kernels) == GLOBAL | {spectral, sorted_}, kernels
    suffixes = Plan(settings).suffixes
    bad = _waived(check(got, want[name], suffixes, degenerate), series, walk_rows, want[name])
    assert not bad, _report(bad)
    if length == L_MAX:
        # past the 15-bit node ids of the narrow Lempel-Ziv keys
        phrases = want[name][0, suffixes.index("lempel_ziv_complexity__bins_100")] * length
        assert round(phrases) > 32767, phrases


def test_cwt_peaks_past_int16_columns():
    """the 131 072-sample case has ridge lines ending past column 32 767 (the int16 range of the narrow tables)"""
    from scipy.signal import find_peaks_cwt
    x = CASES["csr_%d" % L_MAX][0][0].astype(np.float64)
    peaks = find_peaks_cwt(x, np.arange(1, 6))
    assert len(peaks) and max(peaks) > 32767


def test_too_long_before_any_group(ctx):
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(EfficientFCParameters()))
    try:
        with pytest.raises(ValueError, match=r"series length 131073 exceeds the shared-memory staging of kernel group "
                                             r"\w+ \(limit 131072 samples\)"):
            dp.extract_csr(*to_csr([np.zeros(10, np.float32), np.zeros(L_MAX + 1, np.float32)]))
        assert ctx.last_kernels() == [] and ctx.launch_count() == 0
    finally:
        dp.close()


def test_entropy_keeps_21000(ctx):
    from tsfresh_b200._lib import DevicePlan
    settings = EfficientFCParameters()
    settings["approximate_entropy"] = ComprehensiveFCParameters()["approximate_entropy"]
    dp = DevicePlan(ctx, Plan(settings))
    try:
        dp.extract_csr(*to_csr([np.ones(21000, np.float32)]))
        with pytest.raises(ValueError, match=r"series length 21001 exceeds the shared-memory staging of kernel group "
                                             r"entropy \(limit 21000 samples\)"):
            dp.extract_csr(*to_csr([np.ones(21001, np.float32)]))
        assert ctx.last_kernels() == [] and ctx.launch_count() == 0
    finally:
        dp.close()


def test_extract_features_long_frame(want):
    """the pipelined long-frame path (tsfx_extract_long) with ids of 50 000 and 131 072 rows"""
    from tsfresh_b200.extraction import extract_features
    df = pd.DataFrame({"id": np.repeat([7, 3], [len(s) for s in FRAME]),
                       "time": np.concatenate([np.arange(len(s)) for s in FRAME]),
                       "value": np.concatenate(FRAME)})
    settings = EfficientFCParameters()
    res = extract_features(df, default_fc_parameters=settings, column_id="id", column_sort="time")
    assert list(res.index) == [3, 7]
    assert list(res.columns) == ["value__" + s for s in Plan(settings).suffixes]
    got = res.to_numpy()[[1, 0]]
    bad = check(got, want["frame"], Plan(settings).suffixes, [False] * len(FRAME))
    assert not bad, _report(bad)


def test_roll_time_series_long_windows(want):
    from tsfresh_b200.extraction import extract_features
    from tsfresh_b200.rolling import roll_time_series
    df = pd.DataFrame({"id": np.zeros(ROLL_ROWS, np.int64), "time": np.arange(ROLL_ROWS), "value": ROLL})
    rolled = roll_time_series(df, column_id="id", column_sort="time", max_timeshift=ROLL_SHIFT, min_timeshift=ROLL_SHIFT)
    settings = EfficientFCParameters()
    res = extract_features(rolled, default_fc_parameters=settings)
    assert list(res.index) == [(0, e) for e in range(ROLL_SHIFT, ROLL_ROWS)]
    bad = _waived(check(res.to_numpy(), want["roll"], Plan(settings).suffixes, [False] * len(ROLL_WINDOWS)),
                  ROLL_WINDOWS, set(range(len(ROLL_WINDOWS))), want["roll"])
    assert not bad, _report(bad)


def test_cwt_peaks_with_infinite_samples(ctx):
    """pairs of +-inf samples put inf and NaN into the CWT rows: the sliding noise window must keep NaN in order (as
    scipy's sort does) and stay inside its own slots -- four long series of one CTA, their windows side by side in shared
    memory, against the oracle"""
    from oracle.extract import oracle_rows
    settings = {"number_cwt_peaks": ComprehensiveFCParameters()["number_cwt_peaks"]}
    rng = np.random.default_rng(21)
    series = []
    for k, vals in enumerate(([np.inf], None, [np.inf, -np.inf], None)):
        x = rng.standard_normal(30000 + 7 * k)
        if vals:
            for j, at in enumerate(rng.choice(len(x) - 1, 40, replace=False)):
                x[at] = x[at + 1] = vals[j % len(vals)]
        series.append(x.astype(np.float32))
    got, kernels = _extract(ctx, settings, series, False)
    assert kernels == ["peaks/general/w4/global"], kernels
    want = oracle_rows([s.astype(np.float64) for s in series], settings)
    np.testing.assert_array_equal(got, want)


def test_basic_sorted_plans_have_no_length_limit(ctx):
    """a plan of BASIC and SORTED calculators only (MinimalFCParameters) is not capped at 131 072 samples"""
    from oracle.extract import compare, oracle_rows
    from tsfresh_b200.settings import MinimalFCParameters
    settings = MinimalFCParameters()
    rng = np.random.default_rng(22)
    series = [rng.standard_normal(200003).astype(np.float32), rng.standard_normal(17).astype(np.float32)]
    got, kernels = _extract(ctx, settings, series, False)
    assert {k.split("/")[0] for k in kernels} <= {"basic", "sorted", "moments"}, kernels
    want = oracle_rows([s.astype(np.float64) for s in series], settings)
    bad = compare(got, want, Plan(settings).suffixes)
    assert not bad, _report(bad)
