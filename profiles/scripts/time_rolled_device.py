#!/usr/bin/env python
"""Needs a CUDA device: extract_features_rolled_device against extract_features(roll_time_series(frame)) on the same
rows -- BASELINE.json configs[4] on one GPU: --ids series x --length rows (default 10 000 x 4 096 = 41 M rows), windows
of --window rows every --stride rows (rolling_direction = stride, max_timeshift = window - 1, min_timeshift 0: 128
windows per series, 1.28 M in all), ComprehensiveFCParameters.

  rolled_device  extract_features_rolled_device on CUDA tensors (int64 ids and sort keys, float32 values), result on
                 the device
  frame          extract_features(roll_time_series(frame, column_id="id", column_sort="time", ...)) on the same rows
                 from host memory, result on the host

Each is timed with a host clock around the call followed by torch.cuda.synchronize(), after one warm-up call, over
--reps repetitions (median reported; the frame's with --frame-reps).  The two results are compared bit for bit (values
with NaN as NaN, window names, column names).  Prints one JSON line with the card's name and power limit read in the same
run.

    python profiles/scripts/time_rolled_device.py [--ids 10000] [--length 4096] [--window 256] [--stride 32] [--reps 3]
                                                  [--frame-reps 1] [--out FILE]"""
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
    ap.add_argument("--ids", type=int, default=10_000)
    ap.add_argument("--length", type=int, default=4_096)
    ap.add_argument("--window", type=int, default=256)
    ap.add_argument("--stride", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frame-reps", type=int, default=1)
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import pandas as pd
    import torch
    from tsfresh_b200 import ComprehensiveFCParameters, extract_features, extract_features_rolled_device, roll_time_series

    if not torch.cuda.is_available():
        raise SystemExit("time_rolled_device.py needs a CUDA device")
    N, L = a.ids, a.length
    R = N * L
    settings = ComprehensiveFCParameters()
    roll = dict(rolling_direction=a.stride, max_timeshift=a.window - 1, min_timeshift=0)
    gen = torch.Generator(device="cuda").manual_seed(5)
    row = torch.arange(R, device="cuda", dtype=torch.int64)        # (id, time) order
    ids = row // L * 7 - 3000
    sort = row % L
    values = torch.randn(R, device="cuda", generator=gen, dtype=torch.float32)
    del row

    def timed(fn, reps):
        fn()                                          # warm-up: working regions, plans, twiddle table
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
            del out
        return float(np.median(ts)), [round(t, 1) for t in ts]

    res = {"workload": "ComprehensiveFCParameters, rolled windows of %d rows every %d rows over %d ids x %d rows (%d rows)"
                       % (a.window, a.stride, N, L, R), "gpu": card(), "reps": a.reps, "frame_reps": a.frame_reps}
    run = lambda: extract_features_rolled_device(ids, values, sort, default_fc_parameters=settings, **roll)  # noqa: E731
    res["rolled_device_ms"], res["rolled_device_all"] = timed(run, a.reps)
    X, wid, wkey, columns = run()
    res["n_windows"], res["n_features"] = int(X.shape[0]), len(columns)
    Xh, idh, keyh = X.cpu().numpy(), wid.cpu().numpy(), wkey.cpu().numpy()
    del X, wid, wkey
    torch.cuda.empty_cache()
    df = pd.DataFrame({"id": ids.cpu().numpy(), "time": sort.cpu().numpy(), "value": values.cpu().numpy()})
    frame = lambda: extract_features(roll_time_series(df, column_id="id", column_sort="time", **roll),  # noqa: E731
                                     default_fc_parameters=settings)
    res["frame_ms"], res["frame_all"] = timed(frame, a.frame_reps)
    want = frame()
    names = want.index.tolist()
    same = list(want.columns) == columns and len(names) == len(idh) and \
        names == list(zip(idh.tolist(), keyh.tolist()))
    del names
    W = want.to_numpy()
    for r0 in range(0, len(W), 65_536):                # NaN as NaN, bit for bit, in row blocks
        g, w = Xh[r0:r0 + 65_536], W[r0:r0 + 65_536]
        same = same and np.array_equal(np.where(np.isnan(g), np.nan, g).view(np.int64),
                                       np.where(np.isnan(w), np.nan, w).view(np.int64))
    res["equal_bits"] = bool(same)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
