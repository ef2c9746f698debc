#!/usr/bin/env python
"""Splits the BASIC group's time by calculator family: one plan per family, holding the ComprehensiveFCParameters
entries of just that family's calculators, timed against a plan of every BASIC calculator of Comprehensive with the
per-group CUDA events (TSFX_FLAG_TIMING, ctx.timings()["basic"]).  Every plan runs the same k_basic on
device-resident random-normal series (1 M x 256 by default, the headline shape); a family plan walks only its own
descriptors, so its time approximates a kernel of that family alone, its own series load and moments included.

    python profiles/scripts/time_basic_families.py [--rounds 3] [--reps 5] [--series 1000000] [--len 256]

Needs a CUDA device and the tree's library (python -m tsfresh_b200.build).  The plans alternate in each round; the
script prints one JSON line: the card's name and power limit, the kernel each plan ran (a plan of class-M reductions
alone would run k_moments instead, so every plan must report a basic/... variant), the BASIC times of every plan in
ms, their medians and spreads (max - min), and the sum of the family medians against the full plan's.  With
--calculators it also times one plan per calculator (its Comprehensive entries next to count_above_mean, so that no
plan falls to k_moments) against count_above_mean alone, and reports what each calculator adds to that base."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# the BASIC calculators of ComprehensiveFCParameters, by the family that would own them in a split kernel
FAMILIES = {
    "stats": ("variance_larger_than_standard_deviation", "has_duplicate_max", "has_duplicate_min", "sum_values",
              "abs_energy", "mean_abs_change", "mean_change", "mean_second_derivative_central", "mean", "length",
              "standard_deviation", "variation_coefficient", "variance", "skewness", "kurtosis", "root_mean_square",
              "absolute_sum_of_changes", "longest_strike_below_mean", "longest_strike_above_mean",
              "count_above_mean", "count_below_mean", "last_location_of_maximum", "first_location_of_maximum",
              "last_location_of_minimum", "first_location_of_minimum", "maximum", "absolute_maximum", "minimum",
              "cid_ce", "large_standard_deviation", "autocorrelation", "query_similarity_count",
              "agg_autocorrelation", "partial_autocorrelation"),
    "scans": ("value_count", "range_count", "count_above", "count_below", "number_crossing_m", "number_peaks",
              "ratio_beyond_r_sigma", "index_mass_quantile", "energy_ratio_by_chunks", "binned_entropy",
              "benford_correlation", "time_reversal_asymmetry_statistic", "c3"),
    "trends": ("linear_trend", "linear_trend_timewise", "agg_linear_trend"),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--len", type=int, default=256)
    ap.add_argument("--calculators", action="store_true")
    a = ap.parse_args()

    sys.path.insert(0, HERE)
    import torch
    from tsfresh_b200._lib import Context, DevicePlan
    from tsfresh_b200.plan import Plan
    from tsfresh_b200.settings import ComprehensiveFCParameters

    full = ComprehensiveFCParameters()
    every = [c for f in FAMILIES.values() for c in f]
    settings = {name: {k: full[k] for k in calcs if k in full} for name, calcs in FAMILIES.items()}
    settings["all"] = {k: full[k] for k in every if k in full}
    if a.calculators:
        settings["base"] = {"count_above_mean": None}
        for k in every:
            if k in full and k != "count_above_mean":
                settings[k] = {"count_above_mean": None, k: full[k]}

    gen = torch.Generator(device="cuda").manual_seed(44)
    x = torch.randn(a.series, a.len, device="cuda", generator=gen, dtype=torch.float32)
    ctx = Context(0)
    runs = {}
    try:
        for name, s in settings.items():
            plan = Plan(s)
            if name in plan.skipped:                    # linear_trend_timewise: no columns without a DatetimeIndex
                continue
            runs[name] = (DevicePlan(ctx, plan), torch.empty(a.series, plan.n_cols, device="cuda", dtype=torch.float64),
                          plan.n_cols)
        kernels, ms = {}, {name: [] for name in runs}
        for name, (dp, out, _) in runs.items():                                       # warm-up
            dp.extract_dense_device(x.data_ptr(), a.series, a.len, out.data_ptr(), timing=True)
            ctx.sync()
            kernels[name] = ctx.last_kernels()
            if not any(k.startswith("basic/") for k in kernels[name]):
                raise SystemExit("plan %s did not run k_basic: %r" % (name, kernels[name]))
        for _ in range(a.rounds):
            for name, (dp, out, _) in runs.items():
                for _ in range(a.reps):
                    dp.extract_dense_device(x.data_ptr(), a.series, a.len, out.data_ptr(), timing=True)
                    ctx.sync()
                    ms[name].append(round(ctx.timings()["basic"], 3))
    finally:
        for dp, _, _ in runs.values():
            dp.close()
        ctx.close()
    med = {k: round(statistics.median(v), 2) for k, v in ms.items()}
    fam = sum(med[k] for k in FAMILIES)
    print(json.dumps({"gpu": card(), "shape": [a.series, a.len], "kernels": kernels,
                      "columns": {k: r[2] for k, r in runs.items()}, "basic_ms": ms, "median_ms": med,
                      "spread_ms": {k: round(max(v) - min(v), 2) for k, v in ms.items()},
                      "families_sum_ms": round(fam, 2), "all_ms": med["all"],
                      "saving_ms": round(med["all"] - fam, 2),
                      "calculator_ms": {k: round(med[k] - med["base"], 2) for k in med
                                        if a.calculators and k not in FAMILIES and k not in ("all", "base")}}))


if __name__ == "__main__":
    main()
