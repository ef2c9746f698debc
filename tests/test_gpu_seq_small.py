"""The short-series SEQ kernel (k_seq_small: series of at most 256 samples, alphabets of at most 127 symbols) against
the oracle where its counting changes: 1, 2, D - 1, D and D + 1 samples for every dimension D, and 255 and 256 samples;
normal, tied and constant series; tau 1 to 3 with dimensions 2 to 8, and every Lempel-Ziv alphabet from 1 to 127
symbols, in one plan.

The reference ranks a window with np.argsort, whose order among tied values depends on numpy's sort; the kernel ranks
ties stably (the earlier sample is the smaller).  On tied and constant series the permutation_entropy columns are
therefore compared with the reference's formula evaluated with stable ranks."""
import re

import numpy as np
import pytest

from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from tests.helpers import to_csr
from tsfresh_b200.plan import Plan

pytestmark = pytest.mark.gpu

SETTINGS = {"lempel_ziv_complexity": [{"bins": b} for b in (1, 2, 3, 5, 10, 100, 127)],
            "permutation_entropy": [{"tau": t, "dimension": d} for t in (1, 2, 3) for d in range(2, 9)]}
LENGTHS = sorted({1, 2, 255, 256} | {m for d in range(2, 9) for m in (d - 1, d, d + 1)})


def stable_permutation_entropy(x, tau, dimension):
    if len(x) < dimension:
        return np.nan
    W = np.array([x[st:st + dimension] for st in range(0, len(x) - dimension + 1, tau)])
    if len(W) == 0:
        return np.nan
    ranks = np.argsort(np.argsort(W, axis=1, kind="stable"), axis=1, kind="stable")
    _, c = np.unique(ranks, axis=0, return_counts=True)
    p = c / len(ranks)
    return -np.sum(p * np.log(p))


def series_set():
    rng = np.random.default_rng(11)
    normal = [rng.standard_normal(n).astype(np.float32) for n in LENGTHS]
    tied = [rng.integers(0, 3, n).astype(np.float32) for n in LENGTHS]
    constant = [np.full(n, 1.5, np.float32) for n in LENGTHS]
    return normal, tied + constant


def test_seq_small_against_the_oracle():
    from tsfresh_b200._lib import Context, DevicePlan
    normal, degenerate = series_set()
    series = normal + degenerate
    plan = Plan(SETTINGS)
    ctx = Context(0)
    dp = DevicePlan(ctx, plan)
    try:
        got = dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
        ctx.close()
    assert "seq/small" in kernels, kernels
    want = oracle_rows([s.astype(np.float64) for s in series], SETTINGS)
    for r, s in enumerate(degenerate, start=len(normal)):
        for c, suffix in enumerate(plan.suffixes):
            if suffix.startswith("permutation_entropy"):
                tau = int(re.search(r"tau_(\d+)", suffix).group(1))
                dim = int(re.search(r"dimension_(\d+)", suffix).group(1))
                want[r, c] = stable_permutation_entropy(s.astype(np.float64), tau, dim)
    n = len(normal)
    bad = compare(got[:n], want[:n], plan.suffixes)
    bad += [(b[0] + n,) + b[1:] for b in compare(got[n:], want[n:], plan.suffixes, atol=NOISE_FLOOR)]
    assert not bad, "\n".join("row %d %s: gpu=%r oracle=%r" % b for b in bad[:40]) + "\n(%d mismatches)" % len(bad)
