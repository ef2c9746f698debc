"""GPU parity AT THE BASELINE SHAPES (BASELINE.json configs[1..4]) on >= 2 000 series per shape: the C-ABI result
against the oracle evaluated in a process pool on the same seeded float32 inputs.

  config 2  EfficientFCParameters       2 048 series x 256
  config 3  ComprehensiveFCParameters   2 048 series x 256 (N(0,1)) + 512 random walks x 256
  config 4  ComprehensiveFCParameters     512 series x 1024  (the oracle needs ~1 s per series at this length)
  config 5  roll_time_series(32, 255, 255) over 17 parents x 4096 -> 2 057 windows x 256, Comprehensive

Every mismatch fails the test.  The cells that only pass because of the absolute noise floor of oracle.extract.compare
are written to $TSFX_AUDIT_DIR/atol_cells_<shape>.json, when that variable names a directory, so the list of columns
that need a floor can be audited."""
import json
import multiprocessing as mp
import os

import numpy as np
import pytest

from oracle.extract import compare, oracle_rows
from tests.helpers import cores, synthetic_series, to_csr
from tsfresh_b200.plan import Plan
from tsfresh_b200.settings import ComprehensiveFCParameters, EfficientFCParameters

pytestmark = pytest.mark.gpu
SETTINGS = {"efficient": EfficientFCParameters, "comprehensive": ComprehensiveFCParameters}


def _oracle_chunk(args):
    name, chunk = args
    for k in ("OMP_NUM_THREADS", "MKL_NUM_THREADS", "OPENBLAS_NUM_THREADS"):
        os.environ[k] = "1"
    return oracle_rows([np.asarray(s, dtype=np.float32).astype(np.float64) for s in chunk], SETTINGS[name]())


def oracle_parallel(series, name):
    n = cores()
    per = max(1, (len(series) + 4 * n - 1) // (4 * n))
    chunks = [(name, series[i:i + per]) for i in range(0, len(series), per)]
    with mp.get_context("spawn").Pool(n) as pool:
        parts = pool.map(_oracle_chunk, chunks)
    return np.concatenate(parts, axis=0)


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


def _check(ctx, tag, name, series, via="csr"):
    from tsfresh_b200._lib import DevicePlan
    plan = Plan(SETTINGS[name]())
    dp = DevicePlan(ctx, plan)
    try:
        if via == "dense":
            got = dp.extract_dense(np.stack(series))
        else:
            got = dp.extract_csr(*to_csr(series))
    finally:
        dp.close()
    want = oracle_parallel(series, name)
    bad = compare(got, want, plan.suffixes)
    strict = compare(got, want, plan.suffixes, atol=0.0)
    floor_cells = sorted({b[1] for b in strict} - {b[1] for b in bad})
    audit = os.environ.get("TSFX_AUDIT_DIR")
    if audit:
        worst = {}
        for r, suf, g, w in strict:
            if suf in floor_cells:
                worst[suf] = max(worst.get(suf, 0.0), abs(g - w))
        try:
            os.makedirs(audit, exist_ok=True)
            json.dump({"shape": tag, "series": len(series), "columns_passing_only_with_the_noise_floor": worst},
                      open(os.path.join(audit, "atol_cells_%s.json" % tag), "w"), indent=1)
        except OSError:
            pass
    assert not bad, "%d mismatching cells, first: %r" % (len(bad), bad[:20])
    return got


def test_config2_efficient_2048x256(ctx):
    _check(ctx, "config2", "efficient", list(synthetic_series(4301, 2048, 256)), via="dense")


def test_config3_comprehensive_2048x256(ctx):
    _check(ctx, "config3", "comprehensive", list(synthetic_series(4302, 2048, 256)), via="dense")


def test_config3_comprehensive_random_walks_512x256(ctx):
    _check(ctx, "config3_walk", "comprehensive", list(synthetic_series(4303, 512, 256, "walk")))


def test_config4_comprehensive_512x1024(ctx):
    _check(ctx, "config4", "comprehensive", list(synthetic_series(4304, 512, 1024)), via="dense")


def test_config5_rolled_windows_17x4096(ctx):
    """roll_time_series(rolling_direction=32, max_timeshift=255, min_timeshift=255): 121 windows of 256 rows per
    parent, evaluated as (begin, len) views on the parents' buffer; the oracle gets the materialised windows."""
    from tsfresh_b200 import _lib
    from tsfresh_b200._lib import DevicePlan
    parents = synthetic_series(4305, 17, 4096, "walk")
    values, begin, lens = to_csr(list(parents))
    wb, wl, wp, we = _lib.roll_windows(begin, lens, 32, 255, 255)
    assert len(wb) == 17 * 121 and (wl == 256).all()
    plan = Plan(ComprehensiveFCParameters())
    dp = DevicePlan(ctx, plan)
    try:
        got = dp.extract_csr(values, wb, wl)
    finally:
        dp.close()
    windows = [values[b:b + l] for b, l in zip(wb, wl)]
    want = oracle_parallel(windows, "comprehensive")
    bad = compare(got, want, plan.suffixes)
    assert not bad, "%d mismatching cells, first: %r" % (len(bad), bad[:20])
