"""change_quantiles against the oracle with many corridors per plan.

The SORTED kernel serves four corridors (ql, qh) per sweep over the consecutive pairs, with float32 thresholds rounded
outwards from each corridor's float64 quantiles.  These plans have 64 distinct corridors (16 sweeps, the last batch
full and others mixed), among them shared bounds, ql == qh and reversed corridors (both write 0).  The series:

  * 1, 2 and 3 samples (no pair, one pair, two pairs), and lengths on both sides of 256 and of 1 024;
  * normal, random-walk, few-valued (many ties, and quantiles that fall on a tied value), constant, and normal series
    with +-inf samples (quantile bounds of +-inf at ql = 0 / qh = 1, changes of +-inf and NaN);
  * one CSR call with every series of at most 1 024 samples (sorted/w8/shared) and one with 1 025 and 2 000 added
    (sorted/w4/shared).

Floats are compared at rtol 1e-5 (oracle.extract.compare); which cells are 0 -- an empty corridor -- must agree exactly."""
import numpy as np
import pytest

from oracle.extract import compare, oracle_rows
from tests.helpers import to_csr
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu

LEVELS = (0.0, 0.1, 0.11, 0.3, 0.45, 0.55, 0.9, 1.0)
SETTINGS = {"change_quantiles": [{"ql": ql, "qh": qh, "isabs": b, "f_agg": f}
                                 for ql in LEVELS for qh in LEVELS for b in (False, True) for f in ("mean", "var")]}


def series_set(lengths, seed):
    rng = np.random.default_rng(seed)
    out = []
    for n in lengths:
        out.append(rng.standard_normal(n))
        out.append(rng.standard_normal(n).cumsum())
        out.append(rng.integers(0, 4, n).astype(np.float64))
        out.append(np.full(n, 1.75))
        if n >= 20:
            x = rng.standard_normal(n)
            x[rng.integers(0, n, max(1, n // 50))] = np.inf
            x[rng.integers(0, n, max(1, n // 60))] = -np.inf
            out.append(x)
    return [np.asarray(s, dtype=np.float32) for s in out]


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


SHORT = [1, 2, 3, 5, 31, 32, 33, 100, 255, 256, 257, 1000, 1023, 1024]
CASES = [(SHORT, "sorted/w8/shared"), (SHORT + [1025, 2000], "sorted/w4/shared")]


@pytest.mark.parametrize("lengths,variant", CASES, ids=[c[1] for c in CASES])
def test_change_quantiles_vs_oracle(ctx, lengths, variant):
    from tsfresh_b200._lib import DevicePlan
    plan = Plan(SETTINGS)
    assert len({(d["ql"], d["qh"]) for d in SETTINGS["change_quantiles"]}) == 64
    series = series_set(lengths, seed=len(lengths))
    dp = DevicePlan(ctx, plan)
    try:
        got = dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
    assert kernels == [variant], kernels
    want = np.asarray(oracle_rows([s.astype(np.float64) for s in series], SETTINGS), dtype=np.float64)
    # With an infinite extreme, Q(0) or Q(1) interpolates inf - inf: NaN in the kernel, +-inf in numpy, so corridors
    # bounded by level 0 or 1 differ on those rows whatever the kernel does with the pairs.  Only the other corridors
    # of the +-inf rows are compared (there the infinite samples lie outside every corridor).
    edge = np.array([s.endswith("__ql_0.0") or "__qh_1.0__" in s for s in plan.suffixes])
    skip = np.array([np.isinf(s).any() for s in series])[:, None] & edge[None, :]
    got, want = np.where(skip, 0.0, got), np.where(skip, 0.0, want)
    bad = compare(got, want, plan.suffixes)
    assert not bad, "\n".join("row %d (n = %d) %s: gpu=%r oracle=%r" % ((b[0], len(series[b[0]])) + b[1:])
                              for b in bad[:40]) + "\n(%d mismatches)" % len(bad)
    assert np.array_equal(got == 0.0, want == 0.0)
