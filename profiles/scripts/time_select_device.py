#!/usr/bin/env python
"""Needs a CUDA device: what select_features_device saves a user whose feature matrix is already on the GPU, on the
ComprehensiveFCParameters matrix of 1 000 000 x 256 seeded random-normal float32 series (the bench.py workload),
extracted and imputed on the device by extract_features_device.

Two targets, both derived from one feature column plus seeded noise: a binary one (the noisy feature above its
median) and a regression one (the noisy feature).  For each, two ways to the relevant columns, each timed with a host
clock around the call and a device synchronise, after a warm-up (the median of the repetitions is reported):
  device   select_features_device(X, y, columns): the matrix is read in place on the GPU
  frame    X.cpu() -> pd.DataFrame -> select_features: the path a device user had before (skipped with --no-frame)
Before anything is timed, calculate_relevance_table_device and calculate_relevance_table on the DataFrame must give
equal tables (p-values as float64 bits); that DataFrame call is the frame path's warm-up.  Prints progress to stderr and
one JSON line with the card's name and power limit read in the same run.

    python profiles/scripts/time_select_device.py [--n 1000000] [--reps 3] [--frame-reps 1] [--no-frame] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--length", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frame-reps", type=int, default=1, help="the frame path moves the matrix through host memory")
    ap.add_argument("--feature", default="value__standard_deviation", help="the column the targets are derived from")
    ap.add_argument("--no-frame", action="store_true")
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import pandas as pd
    import torch
    from tsfresh_b200 import (calculate_relevance_table, calculate_relevance_table_device, extract_features_device,
                              impute, select_features, select_features_device)
    from tsfresh_b200.settings import ComprehensiveFCParameters

    if not torch.cuda.is_available():
        raise SystemExit("time_select_device.py needs a CUDA device")

    def progress(msg):
        print(msg, file=sys.stderr, flush=True)

    N, L = a.n, a.length
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn((N, L), device="cuda", generator=gen, dtype=torch.float32)
    X, columns = extract_features_device(x, kinds=["value"], default_fc_parameters=ComprehensiveFCParameters(),
                                         impute_function=impute)
    del x
    progress("matrix %s extracted" % (tuple(X.shape),))
    f = X[:, columns.index(a.feature)].cpu().numpy()
    noisy = f + np.random.default_rng(8).standard_normal(N) * f.std()
    targets = {"binary": (noisy > np.median(noisy)).astype(np.int64), "regression": noisy}

    def timed(fn, reps, warm_up=True):
        first = fn() if warm_up else None             # warm-up: context, scratch, torch's cached blocks
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            last = fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
            progress("  %.1f ms" % ts[-1])
        return float(np.median(ts)), [round(t, 1) for t in ts], first if warm_up else last

    def frame_select(y):
        df = pd.DataFrame(X.cpu().numpy(), columns=columns)
        return list(select_features(df, y).columns)

    res = {"workload": "ComprehensiveFCParameters %d x %d float32 -> device matrix, imputed" % (N, L), "gpu": card(),
           "n_features": len(columns), "matrix_bytes": N * len(columns) * 8, "reps": a.reps,
           "frame_reps": a.frame_reps}
    for name, y in targets.items():
        progress("%s: the two tables" % name)
        y_dev = torch.from_numpy(y).to(X.device)
        got = calculate_relevance_table_device(X, y_dev, columns)
        want = calculate_relevance_table(pd.DataFrame(X.cpu().numpy(), columns=columns), pd.Series(y))
        pd.testing.assert_frame_equal(got, want)
        p = lambda t: np.nan_to_num(t.p_value.to_numpy(dtype=float), nan=-1.0).view(np.int64)   # noqa: E731
        assert (p(got) == p(want)).all(), "p-values differ"
        del want
        kept = list(got[got.relevant].feature)
        res[name + "_relevant"] = len(kept)
        progress("%s: equal tables, %d relevant features; select_features_device" % (name, len(kept)))
        res[name + "_device_ms"], res[name + "_device_all"], (_, first) = timed(
            lambda: select_features_device(X, y_dev, columns), a.reps)
        assert first == kept
        if not a.no_frame:                            # the DataFrame path of the check above was its warm-up
            progress("%s: X.cpu() -> DataFrame -> select_features" % name)
            res[name + "_frame_ms"], res[name + "_frame_all"], last = timed(lambda: frame_select(y), a.frame_reps,
                                                                                warm_up=False)
            assert last == kept
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
