"""ar_coefficient and augmented_dickey_fuller against the oracle around the compact LA kernel's bounds.

Calls whose longest series has at most 256 samples (and whose largest AR order is at most 15) run the compact kernel
`la/small`; longer calls, and larger AR orders, run the general one.  Every call below mixes many lengths in one CSR
batch, so the short series go through the variant the longest one selects:

  * 1-40 samples, where the ADF maxlag cap n/2 - 2, the k = 10 feasibility rows >= k + 1 and the nobs - q limits change;
  * 100, 255 and 256 samples (la/small), and 257 (the general kernel);
  * normal, random-walk, trending and constant series.

Comparisons use oracle.extract.compare with atol 0 on the random rows and NOISE_FLOOR on the degenerate ones
(constant, at most 5 samples).  Exactly collinear series (linear ramps, exact alternation) are left out, as in the
other suites (DESIGN.md §2).  A constant series is a rank-one AR design: both kernels return numpy pinv's minimum-norm
solution, which the reference reproduces only while its singular-value cutoff drops the rounding noise -- at 256
samples of 1.75 with k = 3 it does not, so the constant rows use 2.5 (as the other suites do)."""
import numpy as np
import pytest

from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from tests.helpers import to_csr
from tsfresh_b200.plan import Plan
from tsfresh_b200.settings import ComprehensiveFCParameters

pytestmark = pytest.mark.gpu

ATTRS = ("teststat", "pvalue", "usedlag")


def comprehensive_la():
    full = ComprehensiveFCParameters()
    return {k: full[k] for k in ("ar_coefficient", "augmented_dickey_fuller")}


def bic_none_la():
    return {"augmented_dickey_fuller": [{"attr": a, "autolag": al} for al in ("BIC", None) for a in ATTRS],
            "ar_coefficient": [{"coeff": c, "k": k} for k in (1, 3, 15) for c in (0, 1, k)]}


def series_set(lengths, seed):
    """(series, degenerate) of every kind at every length"""
    rng = np.random.default_rng(seed)
    out = []
    for n in lengths:
        t = np.arange(n)
        out.append((rng.standard_normal(n), n <= 5))
        out.append((rng.standard_normal(n).cumsum(), n <= 5))
        out.append((3.0 + 0.05 * t + rng.standard_normal(n), n <= 5))
        out.append((np.full(n, 2.5), True))
    return [(np.asarray(s, dtype=np.float32), d) for s, d in out]


def run(ctx, settings, series):
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(settings))
    try:
        got = dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
    return got, kernels


def check(got, want, suffixes, degenerate):
    degenerate = np.asarray(degenerate, dtype=bool)
    bad = []
    for mask, atol in ((~degenerate, 0.0), (degenerate, NOISE_FLOOR)):
        idx = np.flatnonzero(mask)
        if len(idx):
            bad += [(int(idx[b[0]]),) + b[1:] for b in compare(got[idx], want[idx], suffixes, atol=atol)]
    return bad


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


CASES = [
    ("comprehensive", comprehensive_la, list(range(1, 41)) + [100, 255, 256], "la/small"),
    ("comprehensive", comprehensive_la, list(range(1, 41)) + [100, 255, 256, 257], "la/w8/shared"),
    ("bic_none", bic_none_la, list(range(1, 41)) + [100, 255, 256], "la/small"),
    ("bic_none", bic_none_la, list(range(1, 41)) + [100, 255, 256, 257], "la/w8/shared"),
]


@pytest.mark.parametrize("name,make,lengths,variant", CASES, ids=["%s-%d-%s" % (c[0], max(c[2]), c[3]) for c in CASES])
def test_la_vs_oracle(ctx, name, make, lengths, variant):
    settings = make()
    pairs = series_set(lengths, seed=max(lengths))
    series = [s for s, _ in pairs]
    got, kernels = run(ctx, settings, series)
    assert [k for k in kernels if k.startswith("la/")] == [variant], kernels
    want = np.asarray(oracle_rows([s.astype(np.float64) for s in series], settings), dtype=np.float64)
    suffixes = Plan(settings).suffixes
    bad = check(got, want, suffixes, [d for _, d in pairs])
    assert not bad, "\n".join("row %d (n = %d) %s: gpu=%r oracle=%r" % ((b[0], len(series[b[0]])) + b[1:])
                              for b in bad[:40]) + "\n(%d mismatches)" % len(bad)


def test_large_ar_order_runs_the_general_kernel(ctx):
    """AR orders above 15 do not fit the compact kernel's reduce-scatter: short calls take the general kernel"""
    settings = {"ar_coefficient": [{"coeff": c, "k": 20} for c in (0, 1, 20)]}
    pairs = series_set([30, 41, 64, 200], seed=5)
    series = [s for s, _ in pairs]
    got, kernels = run(ctx, settings, series)
    assert [k for k in kernels if k.startswith("la/")] == ["la/w8/shared"], kernels
    want = np.asarray(oracle_rows([s.astype(np.float64) for s in series], settings), dtype=np.float64)
    bad = check(got, want, Plan(settings).suffixes, [d for _, d in pairs])
    assert not bad, bad[:10]
