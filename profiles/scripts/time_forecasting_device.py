#!/usr/bin/env python
"""Needs a CUDA device: extract_features_forecasting_device against extract_features(make_forecasting_frame(...)[0]) --
one series of --length samples (default 1 048 576), max_timeshift --max-timeshift (default 255), rolling_direction
--direction (default 1), ComprehensiveFCParameters.

  forecasting_device         extract_features_forecasting_device on a float32 CUDA tensor (index None), result and y on
                             the device, over the whole series
  forecasting_device_prefix  the same call on the first --prefix samples only
  frame                      extract_features(make_forecasting_frame(x[:prefix], ...)[0], column_id="id",
                             column_sort="time", column_kind="kind", column_value="value") from host memory, result on
                             the host (default prefix 8 192: the host path needs minutes per 100 000 windows)

Each is timed with a host clock around the call followed by torch.cuda.synchronize(), after one warm-up call, over
--reps repetitions (median reported; the frame's with --frame-reps).  On the prefix the two paths' matrices (bit for
bit, NaN as NaN), window names and targets (y against make_forecasting_frame's y) are compared.  Prints one JSON line
with the card's name and power limit read in the same run.

    python profiles/scripts/time_forecasting_device.py [--length 1048576] [--max-timeshift 255] [--direction 1]
                                                       [--reps 3] [--prefix 8192] [--frame-reps 1] [--out FILE]"""
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
    ap.add_argument("--length", type=int, default=1 << 20)
    ap.add_argument("--max-timeshift", type=int, default=255)
    ap.add_argument("--direction", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--prefix", type=int, default=8192)
    ap.add_argument("--frame-reps", type=int, default=1)
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import torch
    from tsfresh_b200 import ComprehensiveFCParameters, extract_features, extract_features_forecasting_device, \
        make_forecasting_frame

    if not torch.cuda.is_available():
        raise SystemExit("time_forecasting_device.py needs a CUDA device")
    settings = ComprehensiveFCParameters()
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(a.length, device="cuda", generator=gen, dtype=torch.float32).cumsum(0)

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

    res = {"workload": "ComprehensiveFCParameters, forecasting windows of one series of %d samples, max_timeshift %d, "
                       "rolling_direction %d" % (a.length, a.max_timeshift, a.direction), "gpu": card(), "reps": a.reps,
           "frame_reps": a.frame_reps, "prefix": a.prefix}

    def device(n):
        return extract_features_forecasting_device(x[:n], "x", a.max_timeshift, a.direction,
                                                   default_fc_parameters=settings)

    res["forecasting_device_ms"], res["forecasting_device_all"] = timed(lambda: device(a.length), a.reps)
    X, keys, y, columns = device(a.length)
    res["n_windows"], res["n_features"] = int(X.shape[0]), len(columns)
    del X, keys, y
    torch.cuda.empty_cache()
    res["forecasting_device_prefix_ms"], res["forecasting_device_prefix_all"] = timed(lambda: device(a.prefix), a.reps)
    X, keys, y, columns = device(a.prefix)
    Xh, kh, yh = X.cpu().numpy(), keys.cpu().numpy(), y.cpu().numpy()
    xs = x[:a.prefix].cpu().numpy()

    def frame():
        df_shift, _ = make_forecasting_frame(xs, "x", a.max_timeshift, a.direction)
        return extract_features(df_shift, column_id="id", column_sort="time", column_kind="kind", column_value="value",
                                default_fc_parameters=settings)

    res["frame_ms"], res["frame_all"] = timed(frame, a.frame_reps)
    want = frame()
    _, y_host = make_forecasting_frame(xs, "x", a.max_timeshift, a.direction)
    W = want.to_numpy()
    same = list(want.columns) == columns and want.index.tolist() == [("id", k) for k in kh.tolist()]
    same = same and np.array_equal(np.where(np.isnan(Xh), np.nan, Xh).view(np.int64),
                                   np.where(np.isnan(W), np.nan, W).view(np.int64))
    by_name = dict(zip(kh.tolist(), yh.tolist()))
    res["equal_bits"] = bool(same)
    res["equal_y"] = all(by_name[k[1]] == v for k, v in y_host.items()) and len(y_host) >= len(kh) - 1
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
