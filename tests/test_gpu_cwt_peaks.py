"""number_cwt_peaks on the GPU, exactly, on both sides of the length bound that selects the compact shared-memory kernel
(k_peaks_small, series <= 256 samples) over the general one, with series rich in local maxima, plateaus and ties."""
import numpy as np
import pytest

from tests.helpers import gpu_vs_oracle, to_csr

pytestmark = pytest.mark.gpu

LENGTHS = (5, 32, 33, 255, 256, 257, 1024)
# one plan per width set: the kernel is chosen from the longest series and the largest n of the call, so n = 16 at
# 255 / 256 samples runs the general kernel and at <= 33 samples the compact one
N_SETS = ((1,), (5,), (16,), (1, 5))


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def peaky_series(length, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(length)
    out = [
        np.where(t % 2 == 0, -1.0, 1.0) * (1.0 + 0.01 * rng.standard_normal(length)),     # alternation
        np.repeat(rng.standard_normal(length // 2 + 1), 2)[:length],                        # plateaus of two
        np.round(rng.standard_normal(length) * 2) / 2,                                      # many ties
        np.full(length, 3.0),                                                               # constant
        np.zeros(length),
        rng.standard_normal(length).cumsum(),                                               # random walk
        rng.standard_normal(length),                                                        # N(0, 1)
        rng.standard_normal(length) * 1e4 + 1e6,
        np.sin(t * 0.7) + 0.5 * np.sin(t * 3.1),
    ]
    return [np.asarray(s, dtype=np.float32) for s in out]


def exact_tie_series(length):
    """CWT rows with exactly tied neighbours: whether a sample is a strict maximum is decided by the rounding of the
    convolution sums, so numpy's convolution (the oracle) and the kernels' fma chains can disagree on the count"""
    t = np.arange(length)
    rng = np.random.default_rng(length)
    return [np.where(t % 2 == 0, -1.0, 1.0).astype(np.float32),                                   # strict alternation
            np.repeat(rng.integers(-2, 3, length // 3 + 1), 3)[:length].astype(np.float32)]     # integer plateaus


def _report(bad):
    return "\n".join("row %d %s: gpu=%r oracle=%r" % b for b in bad[:40]) + "\n(%d mismatches)" % len(bad)


@pytest.mark.parametrize("ns", N_SETS, ids=lambda ns: "n" + "_".join(map(str, ns)))
@pytest.mark.parametrize("length", LENGTHS)
def test_number_cwt_peaks_exact(ctx, ns, length):
    series = peaky_series(length, 1000 + length) + peaky_series(length, 2000 + length)
    settings = {"number_cwt_peaks": [{"n": n} for n in ns]}
    bad, plan, got, want = gpu_vs_oracle(ctx, settings, series, rtol=0.0)
    assert not bad, _report(bad)
    assert np.array_equal(got, np.round(got))


def test_number_cwt_peaks_ragged(ctx):
    """one call with lengths on both sides of the bound: the longest series selects the general kernel for all"""
    series = [s for L in LENGTHS for s in peaky_series(L, 3000 + L)[::2]]
    bad, *_ = gpu_vs_oracle(ctx, {"number_cwt_peaks": [{"n": 1}, {"n": 5}]}, series, rtol=0.0)
    assert not bad, _report(bad)


@pytest.mark.parametrize("ns", ((1, 5), (16,)), ids=lambda ns: "n" + "_".join(map(str, ns)))
def test_number_cwt_peaks_kernels_agree(ctx, ns):
    """both kernels form every CWT row with the same fma order, so they count the same peaks even where the count
    hangs on rounding: series of <= 256 samples alone (compact kernel where it fits) and next to a 257-sample
    series (general kernel)"""
    from tsfresh_b200._lib import DevicePlan
    from tsfresh_b200.plan import Plan
    short = [s for L in (5, 32, 33, 64, 100, 255, 256) for s in exact_tie_series(L) + peaky_series(L, 4000 + L)]
    long_ = peaky_series(257, 5000)[:1]
    dp = DevicePlan(ctx, Plan({"number_cwt_peaks": [{"n": n} for n in ns]}))
    try:
        alone = dp.extract_csr(*to_csr(short))
        mixed = dp.extract_csr(*to_csr(short + long_))
    finally:
        dp.close()
    assert np.array_equal(alone, mixed[: len(short)]), np.argwhere(alone != mixed[: len(short)])[:20]
