"""Every kernel variant the launchers select, at its length boundaries, against the oracle.

Each kernel group launches one of several variants, chosen from the longest series of the call, the plan, and how much
shared memory a warp's working set needs (`launch_*` in tsfresh_b200/csrc/k_*.cu, `plan_geometry` in tsfx_kernels.h).
Context.last_kernels() reports which variant every group ran, so each case below asserts that it reached the variant it
targets; the bounds in BOUNDS are the lengths at which the choice changes for the Comprehensive calculators (DESIGN.md §3).

  * boundary sweep: one plan per kernel group, the series that selects the variant next to short and degenerate series
    (1-5, 8, 31-33 and 255 samples, constant, tied), CSR and dense input;
  * long series: ComprehensiveFCParameters at 11 300, 12 000 and 21 000 samples; 21 001 is TSFX_E_TOO_LONG;
  * forced variants: the launch knobs (read once per process) in subprocesses -- global-region instantiations, among
    them the entropy tile kernel's, and four streams;
  * warp reuse: a grid of one CTA (wave) per SM, so every warp processes many series in turn, must give the same bits as
    batches in which no warp processes two series; permuting the rows permutes the result;
  * ledger: every variant the launchers can choose under the default and the tested settings was reported here.

Comparisons use oracle.extract.compare with atol 0 on random and random-walk rows and NOISE_FLOOR on the degenerate rows
(DESIGN.md §2).  Waivers are the existing ones: exactly collinear series are left out of LA, SORTED and SPECTRAL, tied
windows out of permutation_entropy, exact +-1 alternation and integer plateaus out of number_cwt_peaks."""
import json
import multiprocessing as mp
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.extract import NOISE_FLOOR, compare, oracle_rows
from tests.helpers import to_csr
from tests.test_gpu_shapes import _cores
from tsfresh_b200.plan import Plan
from tsfresh_b200.settings import ComprehensiveFCParameters, MinimalFCParameters

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CALCS = {
    "sorted": ["symmetry_looking", "has_duplicate", "median", "percentage_of_reoccurring_values_to_all_values",
               "percentage_of_reoccurring_datapoints_to_all_datapoints", "sum_of_reoccurring_values",
               "sum_of_reoccurring_data_points", "ratio_value_number_to_time_series_length", "quantile",
               "mean_n_absolute_max", "change_quantiles", "friedrich_coefficients", "max_langevin_fixed_point"],
    "spectral": ["fft_coefficient", "fft_aggregated", "spkt_welch_density", "fourier_entropy", "cwt_coefficients"],
    "la": ["ar_coefficient", "augmented_dickey_fuller"],
    "entropy": ["sample_entropy", "approximate_entropy"],
    "seq": ["lempel_ziv_complexity", "permutation_entropy"],
    "peaks": ["number_cwt_peaks"],
}


def group_settings(group):
    """the Comprehensive calculators of one kernel group (BASIC: every calculator no other group takes; moments: the
    MinimalFCParameters without the median, which the reduction-only kernel evaluates)"""
    full = ComprehensiveFCParameters()
    if group == "basic":
        others = {c for v in _CALCS.values() for c in v}
        return {k: full[k] for k in full if k not in others}
    if group == "seq_perm":
        return {"permutation_entropy": full["permutation_entropy"]}
    if group == "moments":
        mini = MinimalFCParameters()
        return {k: mini[k] for k in mini if k != "median"}
    return {k: full[k] for k in full if k in _CALCS[group]}


# group -> [(longest series of the call, variant it selects)] on both sides of every bound, read from the launchers'
# arithmetic and confirmed on an H100 with Context.last_kernels()
BOUNDS = {
    "basic": [(480, "basic/w12/shared"), (481, "basic/w4/shared"), (1024, "basic/w4/shared"), (1025, "basic/w2/shared"),
              (2272, "basic/w2/shared"), (2273, "basic/w1/shared"), (11116, "basic/w1/shared"), (11117, "basic/w4/global")],
    "sorted": [(1024, "sorted/w8/shared"), (1025, "sorted/w4/shared"), (2048, "sorted/w4/shared"), (2049, "sorted/w2/shared"),
               (4168, "sorted/w2/shared"), (4169, "sorted/w1/shared"), (21000, "sorted/w1/shared")],
    "spectral": [(404, "spectral/w8/shared"), (405, "spectral/w4/shared"), (860, "spectral/w4/shared"),
                 (861, "spectral/w2/shared"), (1776, "spectral/w2/shared"), (1777, "spectral/w1/shared"),
                 (8248, "spectral/w1/shared"), (8249, "spectral/w4/global")],
    "la": [(316, "la/w8/shared"), (317, "la/w4/shared"), (784, "la/w4/shared"), (785, "la/w2/shared"), (1896, "la/w2/shared"),
           (1897, "la/w1/shared"), (10156, "la/w1/shared"), (10157, "la/w4/global")],
    "entropy": [(256, "entropy/rank-g1"), (257, "entropy/rank-g4"), (512, "entropy/rank-g4"), (513, "entropy/rank-g16"),
                (1152, "entropy/rank-g16"), (1153, "entropy/tiles/w2/shared"), (1616, "entropy/tiles/w2/shared"),
                (1617, "entropy/tiles/w1/shared"), (11600, "entropy/tiles/w1/shared"), (11601, "entropy/tiles/w4/global")],
    "seq": [(256, "seq/small"), (257, "seq/general/w4/global"), (1024, "seq/general/w4/global")],
    # permutation_entropy alone: no Lempel-Ziv tables, so the general kernel's working set fits the 16 KB below which
    # it runs from shared memory
    "seq_perm": [(256, "seq/small"), (257, "seq/general/w8/shared"), (1024, "seq/general/w8/shared"),
                 (1025, "seq/general/w4/shared"), (2048, "seq/general/w4/shared"), (2049, "seq/general/w4/global")],
    "peaks": [(256, "peaks/small"), (257, "peaks/general/hybrid/w4/global"), (348, "peaks/general/hybrid/w4/global"),
              (349, "peaks/general/w4/global")],
}
DENSE = {      # dense input: group -> [(length, variant)]; power-of-two lengths need no twiddle-word table
    "spectral": [(4, "spectral/pow2/w8/shared"), (8, "spectral/pow2/w8/shared"), (16, "spectral/pow2/w8/shared"),
                 (32, "spectral/pow2/w8/shared"), (64, "spectral/pow2/w8/shared"), (128, "spectral/pow2/w8/shared"),
                 (252, "spectral/w8/shared"), (256, "spectral/pow2/w8/shared"), (260, "spectral/w8/shared"),
                 (512, "spectral/pow2/w8/shared"), (1024, "spectral/pow2/w4/shared"), (2048, "spectral/pow2/w2/shared"),
                 (4096, "spectral/pow2/w2/shared"), (8192, "spectral/pow2/w1/shared")],
    "moments": [(4, "moments/dense"), (8, "moments/dense"), (252, "moments/dense"), (256, "moments/dense"),
                (255, "moments/general"), (260, "moments/general")],
}

REPORTED = set()           # variant names reported in this module (the ledger at the end)


@pytest.fixture(scope="module")
def ctx():
    from tsfresh_b200._lib import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pool():
    with mp.get_context("spawn").Pool(_cores()) as p:
        yield p


def _oracle_one(args):
    settings, x = args
    for k in ("OMP_NUM_THREADS", "MKL_NUM_THREADS", "OPENBLAS_NUM_THREADS"):
        os.environ[k] = "1"
    return oracle_rows([np.asarray(x, dtype=np.float32).astype(np.float64)], settings)[0]


def oracle(pool, settings, series):
    """oracle rows of `series`, one task per series, longest first"""
    order = sorted(range(len(series)), key=lambda i: -len(series[i]))
    rows = pool.map(_oracle_one, [(settings, series[i]) for i in order], chunksize=1)
    out = [None] * len(series)
    for i, r in zip(order, rows):
        out[i] = r
    return np.asarray(out, dtype=np.float64)


TIED = "tied"          # degenerate row with tied windows: permutation_entropy is not compared there


def short_and_degenerate(group, seed=0):
    """(series, degenerate) next to the variant-selecting series: 1-5, 8, 31-33 and 255 samples of N(0, 1), a constant
    and a tied series (not for the SEQ group: permutation_entropy is compared on tie-free series only), and for ENTROPY
    the two exactly collinear series"""
    rng = np.random.default_rng(seed)
    out = [(rng.standard_normal(n), n <= 5) for n in (1, 2, 3, 4, 5, 8, 31, 32, 33, 255)]
    if not group.startswith("seq"):
        out += [(np.full(40, 2.5), TIED), (np.round(rng.standard_normal(60) * 2) / 2, TIED)]
    if group == "entropy":
        out += [(np.array([-1.0, 1.0] * 20), True), (np.arange(50, dtype=np.float64), True)]
    return [(np.asarray(s, dtype=np.float32), d) for s, d in out]


def main_series(length, seed):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(length).astype(np.float32), rng.standard_normal(length).cumsum().astype(np.float32)]


def check(got, want, suffixes, degenerate):
    """atol 0 on the random rows, NOISE_FLOOR on the degenerate ones (True or TIED)"""
    tied = np.array([d is TIED for d in degenerate], dtype=bool)
    degenerate = np.array([bool(d) for d in degenerate], dtype=bool)
    bad = []
    for mask, atol in ((~degenerate, 0.0), (degenerate, NOISE_FLOOR)):
        idx = np.flatnonzero(mask)
        if len(idx):
            bad += [(int(idx[b[0]]),) + b[1:] for b in compare(got[idx], want[idx], suffixes, atol=atol)
                    if not (tied[idx[b[0]]] and b[1].startswith("permutation_entropy"))]
    return bad


def _report(bad):
    return "\n".join("row %d %s: gpu=%r oracle=%r" % b for b in bad[:40]) + "\n(%d mismatches)" % len(bad)


def run(ctx, settings, series, dense=False):
    """(result, kernel variants) of one extract call"""
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(settings))
    try:
        got = dp.extract_dense(np.stack(series)) if dense else dp.extract_csr(*to_csr(series))
        kernels = ctx.last_kernels()
    finally:
        dp.close()
    REPORTED.update(kernels)
    return got, kernels


def _variant_of(kernels, group):
    prefix = group.split("_")[0] + "/"
    hit = [k for k in kernels if k.startswith(prefix)]
    assert len(hit) == 1, kernels
    return hit[0]


# ---------------------------------------------------------------------------------------------- boundary sweep
@pytest.mark.parametrize("group,length,variant", [(g, L, v) for g, cases in BOUNDS.items() for L, v in cases])
def test_bound_csr(ctx, pool, group, length, variant):
    settings = group_settings(group)
    extra = short_and_degenerate(group, seed=length)
    series = main_series(length, 7 * length + 1) + [s for s, _ in extra]
    degenerate = [False, False] + [d for _, d in extra]
    got, kernels = run(ctx, settings, series)
    assert _variant_of(kernels, group) == variant, kernels
    want = oracle(pool, settings, series)
    suffixes = Plan(settings).suffixes
    bad = check(got, want, suffixes, degenerate)
    assert not bad, _report(bad)


@pytest.mark.parametrize("group,length,variant", [(g, L, v) for g, cases in DENSE.items() for L, v in cases])
def test_bound_dense(ctx, pool, group, length, variant):
    settings = group_settings(group)
    rng = np.random.default_rng(length)
    series = [rng.standard_normal(length).astype(np.float32) for _ in range(3)]
    series += [rng.standard_normal(length).cumsum().astype(np.float32) for _ in range(3)]
    got, kernels = run(ctx, settings, series, dense=True)
    assert _variant_of(kernels, group) == variant, kernels
    want = oracle(pool, settings, series)
    bad = check(got, want, Plan(settings).suffixes, [length <= 5] * len(series))
    assert not bad, _report(bad)


def test_moments_csr_unaligned_and_long(ctx, pool):
    """the CSR reduction kernel: series starting at every offset mod 4 (scalar head before the 128-bit loads), lengths
    that are not multiples of 4, series longer than the register-resident 256 samples"""
    settings = group_settings("moments")
    rng = np.random.default_rng(3)
    lens = [1, 2, 3, 4, 5, 7, 8, 9, 252, 253, 255, 256, 257, 260, 511, 1000, 1024, 3001]
    series = [rng.standard_normal(n).astype(np.float32) for n in lens]
    series += [rng.standard_normal(n).cumsum().astype(np.float32) for n in (255, 256, 257, 1000)]
    pad = np.zeros(3, np.float32)
    for head in range(4):                   # begin = head (mod 4) for the first series, every offset for the rest
        vals, begin, ln = to_csr(series)
        values = np.concatenate([pad[:head], vals])
        from tsfresh_b200._lib import DevicePlan
        dp = DevicePlan(ctx, Plan(settings))
        try:
            got = dp.extract_csr(values, begin + head, ln)
            kernels = ctx.last_kernels()
        finally:
            dp.close()
        REPORTED.update(kernels)
        assert kernels == ["moments/general"], kernels
        if head == 0:
            want = oracle(pool, settings, series)
        bad = check(got, want, Plan(settings).suffixes, [len(s) <= 5 for s in series])
        assert not bad, (head, _report(bad))


# ---------------------------------------------------------------------------------------------- long series
LONG = ((11300, 2), (12000, 2), (21000, 1))       # (length, series): inside the former BASIC window, all-global, the limit


def test_long_series_comprehensive(ctx, pool):
    """one or two series per call; the oracle rows of all three calls come from one pool pass"""
    settings = ComprehensiveFCParameters()
    calls = []
    for length, count in LONG:
        series = main_series(length, length)[:count]
        got, kernels = run(ctx, settings, series)
        calls.append((length, series, got, kernels))
    want = oracle(pool, settings, [s for _, series, _, _ in calls for s in series])
    suffixes = Plan(settings).suffixes
    r = 0
    failures = []
    for length, series, got, kernels in calls:
        bad = check(got, want[r:r + len(series)], suffixes, [False] * len(series))
        r += len(series)
        if bad:
            failures.append("%d samples (%s):\n%s" % (length, ", ".join(kernels), _report(bad)))
    assert not failures, "\n".join(failures)
    by_len = {length: set(kernels) for length, _, _, kernels in calls}
    assert {"basic/w4/global", "spectral/w4/global", "la/w4/global", "entropy/tiles/w4/global"} <= by_len[12000], by_len
    assert "basic/w4/global" in by_len[11300], by_len


def test_longer_than_21000_is_too_long(ctx):
    from tsfresh_b200._lib import DevicePlan
    dp = DevicePlan(ctx, Plan(ComprehensiveFCParameters()))
    try:
        with pytest.raises(ValueError, match="series length 21001 exceeds"):
            dp.extract_csr(*to_csr([np.zeros(21001, np.float32)]))
    finally:
        dp.close()


# ---------------------------------------------------------------------------------------------- forced variants
def _forced_cases():
    """(name, settings, series, dense, degenerate rows): Comprehensive at 256 and 1000 samples and the ENTROPY group at
    1200 samples (the tile kernel) next to the short and degenerate series, the SPECTRAL group on dense power-of-two rows"""
    cases = []
    for name, settings, group, length in (("comprehensive_256", ComprehensiveFCParameters(), "basic", 256),
                                          ("comprehensive_1000", ComprehensiveFCParameters(), "basic", 1000),
                                          ("entropy_1200", group_settings("entropy"), "entropy", 1200)):
        extra = short_and_degenerate(group, seed=length + 1)
        cases.append((name, settings, main_series(length, length + 2) + [s for s, _ in extra], False,
                      [False, False] + [d for _, d in extra]))
    rng = np.random.default_rng(4)
    cases.append(("spectral_dense_256", group_settings("spectral"),
                  [rng.standard_normal(256).astype(np.float32) for _ in range(4)], True, [False] * 4))
    return cases


def _run_cases(cases):
    from tsfresh_b200._lib import Context
    c = Context(0)
    try:
        return {name: run(c, settings, series, dense) for name, settings, series, dense, _ in cases}
    finally:
        c.close()


def _reuse_inputs():
    """20 000 series of <= 256 samples and 3 000 of <= 1024, in runs of falling length (a warp's next series is shorter
    than its last one), with normal, walk, tied and constant series mixed"""
    rng = np.random.default_rng(2024)
    out = {}
    for name, count, top in (("short", 20000, 256), ("long", 3000, 1024)):
        lens = rng.integers(1, top + 1, count)
        lens[rng.integers(0, count, 8)] = top
        for i in range(0, count, 500):
            lens[i:i + 500] = np.sort(lens[i:i + 500])[::-1]
        kinds = rng.integers(0, 4, count)
        series = []
        for n, k in zip(lens, kinds):
            x = rng.standard_normal(n)
            x = x.cumsum() if k == 1 else np.round(x * 2) / 2 if k == 2 else np.full(n, x[0]) if k == 3 else x
            series.append(x.astype(np.float32))
        out[name] = series
    out["dense"] = list(rng.standard_normal((20000, 256)).astype(np.float32))
    return out


def _reuse_cases():
    inp = _reuse_inputs()
    comp, mom = ComprehensiveFCParameters(), group_settings("moments")
    return [("comprehensive_short", comp, inp["short"], False, None), ("comprehensive_long", comp, inp["long"], False, None),
            ("moments_short", mom, inp["short"], False, None), ("moments_dense", mom, inp["dense"], True, None)]


def _worker(what, path):
    results = _run_cases(_forced_cases() if what == "forced" else _reuse_cases())
    np.savez(path + ".npz", **{k: v[0] for k, v in results.items()})
    json.dump({k: v[1] for k, v in results.items()}, open(path + ".json", "w"))


def _in_subprocess(tmp_path, what, tag, env):
    """runs _worker in a fresh process (the launch knobs are read once per process) -> ({case: result}, {case: kernels})"""
    path = str(tmp_path / tag)
    full = {k: v for k, v in os.environ.items() if not k.startswith("TSFX_")}
    full.update(env)
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_variants", what, path], cwd=ROOT, env=full,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "%s worker (%s) failed:\n%s\n%s" % (what, env, r.stdout[-4000:], r.stderr[-4000:])
    arrays = np.load(path + ".npz")
    kernels = json.load(open(path + ".json"))
    for v in kernels.values():
        REPORTED.update(v)
    return {k: arrays[k] for k in arrays.files}, kernels


FORCED = {       # configuration -> (environment, variants it must reach)
    "default": ({}, {"entropy/tiles/w2/shared"}),
    "global": ({"TSFX_GLOBAL_ABOVE": "1"},
               {"basic/w4/global", "sorted/w4/global", "spectral/w4/global", "la/w4/global", "spectral/pow2/w4/global",
                "entropy/tiles/w4/global"}),
    "streams": ({"TSFX_STREAMS": "4"}, set()),
}


def test_forced_variants(pool, tmp_path):
    """Every configuration matches the oracle, and gives the default's bits: they change only where the working set
    lives, the warps per CTA or the stream a group runs on."""
    cases = _forced_cases()
    want = {name: oracle(pool, settings, series) for name, settings, series, _, _ in cases}
    res = {cfg: _in_subprocess(tmp_path, "forced", cfg, env) for cfg, (env, _) in FORCED.items()}
    failures = []
    for cfg, (env, must) in FORCED.items():
        got, kernels = res[cfg]
        reached = {k for v in kernels.values() for k in v}
        if not must <= reached:
            failures.append("%s: did not reach %s (ran %s)" % (cfg, sorted(must - reached), sorted(reached)))
        ref = res["default"][0]
        for name, settings, series, dense, degenerate in cases:
            suffixes = Plan(settings).suffixes
            bad = check(got[name], want[name], suffixes, degenerate)
            if bad:
                failures.append("%s / %s vs oracle:\n%s" % (cfg, name, _report(bad)))
            a, b = got[name], ref[name]
            diff = ~((a == b) | (np.isnan(a) & np.isnan(b)))
            if diff.any():
                r, c = np.argwhere(diff)[0]
                failures.append("%s / %s: %d cells differ from default, first row %d %s: %r vs %r" % (
                    cfg, name, diff.sum(), r, suffixes[c], a[r, c], b[r, c]))
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------- warp reuse
def _same_bits(a, b):
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def test_warp_reuse_and_batch_invariance(ctx, tmp_path):
    """TSFX_GRID_WAVES=1 (one wave of CTAs per SM for the shared-memory kernels) and TSFX_GLOBAL_CTAS=1 (one CTA per SM
    in the global region) make every warp process many series in turn, shorter after longer; the result must equal,
    bit for bit, batches of at most 1 000 series -- each with a series of the maximal length appended, so that the
    same variants run -- in which no warp processes two series.  The batches are (begin, len) views of the same value
    buffer, so every series keeps its address: k_moments takes 128-bit loads only from 16-byte aligned series, and the
    other path sums in another order."""
    from tsfresh_b200._lib import DevicePlan
    got, kernels = _in_subprocess(tmp_path, "reuse", "reuse", {"TSFX_GRID_WAVES": "1", "TSFX_GLOBAL_CTAS": "1"})
    failures = []
    for name, settings, series, dense, _ in _reuse_cases():
        values, begin, lens = to_csr(series)
        anchor = int(np.argmax(lens))
        dp = DevicePlan(ctx, Plan(settings))
        try:
            parts = []
            for i in range(0, len(series), 1000):
                if dense:
                    parts.append(dp.extract_dense(np.stack(series[i:i + 1000])))
                else:
                    idx = list(range(i, min(i + 1000, len(series)))) + [anchor]
                    parts.append(dp.extract_csr(values, begin[idx], lens[idx])[:-1])
                    assert sorted(ctx.last_kernels()) == sorted(kernels[name]), (name, ctx.last_kernels(), kernels[name])
            ref = np.concatenate(parts)
        finally:
            dp.close()
        if not _same_bits(got[name], ref):
            diff = ~((got[name] == ref) | (np.isnan(got[name]) & np.isnan(ref)))
            r, c = np.argwhere(diff)[0]
            failures.append("%s: %d cells differ, first row %d (length %d) column %s: %r vs %r" % (
                name, diff.sum(), r, len(series[r]), Plan(settings).suffixes[c], got[name][r, c], ref[r, c]))
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("name", ["comprehensive_short", "comprehensive_long", "moments_dense"])
def test_row_permutation(ctx, name):
    from tsfresh_b200._lib import DevicePlan
    _, settings, series, dense, _ = next(c for c in _reuse_cases() if c[0] == name)
    perm = np.random.default_rng(1).permutation(len(series))
    dp = DevicePlan(ctx, Plan(settings))
    try:
        if dense:
            a, b = dp.extract_dense(np.stack(series)), dp.extract_dense(np.stack(series)[perm])
        else:
            a, b = dp.extract_csr(*to_csr(series)), dp.extract_csr(*to_csr([series[i] for i in perm]))
        REPORTED.update(ctx.last_kernels())
    finally:
        dp.close()
    assert _same_bits(a[perm], b)


# ---------------------------------------------------------------------------------------------- ledger
# variants no test here can reach: never chosen at the sizes run_groups gives the global working region (256 MB up to
# 1 024 samples, 1 GB beyond: four warps' working sets always fit)
NOT_REACHED = {g + "/w1/global": "the global working region always holds four warps"
               for g in ("basic", "sorted", "spectral", "spectral/pow2", "la", "entropy/tiles", "seq/general",
                         "peaks/general", "peaks/general/hybrid")}


def test_variant_ledger(request):
    """runs last: the variants reported by this module are exactly those the launchers can choose"""
    from tsfresh_b200._lib import kernel_variants
    mine = [i for i in request.session.items if i.module is sys.modules[__name__] and i.name != "test_variant_ledger"]
    if len(mine) < N_CASES:
        pytest.skip("only %d of the %d cases of this module ran" % (len(mine), N_CASES))
    if request.session.testsfailed:
        pytest.skip("some cases failed")
    known = set(kernel_variants())
    assert REPORTED <= known, sorted(REPORTED - known)
    assert set(NOT_REACHED) <= known, sorted(set(NOT_REACHED) - known)
    assert REPORTED == known - set(NOT_REACHED), ("never reported: %s; reported although listed as unreachable: %s" % (
        sorted(known - set(NOT_REACHED) - REPORTED), sorted(REPORTED & set(NOT_REACHED))))


N_CASES = sum(len(v) for v in BOUNDS.values()) + sum(len(v) for v in DENSE.values()) + 1 + 2 + 1 + 1 + 3   # + the tests below the sweep


if __name__ == "__main__":
    _worker(sys.argv[1], sys.argv[2])
