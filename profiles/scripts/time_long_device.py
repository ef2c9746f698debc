#!/usr/bin/env python
"""Needs a CUDA device: extract_features_long_device against extract_features on the same pandas frame, for a stacked
long frame of --ids ids x --kinds kinds x --length rows per series (default 100 000 x 4 x 256 = 102.4 M rows), rows
shuffled, EfficientFCParameters for every kind.

  long_device   extract_features_long_device on CUDA tensors (int64 ids and sort keys, int32 kind codes, float32
                values), result on the device
  frame         extract_features(frame, column_id, column_sort, column_kind, column_value) on the same rows from host
                memory, result on the host

Each is timed with CUDA events on torch's current stream around the call (the frame call synchronises before it
returns) after one warm-up call, over --reps repetitions (median reported; the frame's with --frame-reps).  The two
results are compared bit for bit.  Prints one JSON line with the card's name and power limit read in the same run.

    python profiles/scripts/time_long_device.py [--ids 100000] [--kinds 4] [--length 256] [--reps 5] [--frame-reps 2]
                                                [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

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
    ap.add_argument("--ids", type=int, default=100_000)
    ap.add_argument("--kinds", type=int, default=4)
    ap.add_argument("--length", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frame-reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import pandas as pd
    import torch
    from tsfresh_b200 import EfficientFCParameters, extract_features, extract_features_long_device

    if not torch.cuda.is_available():
        raise SystemExit("time_long_device.py needs a CUDA device")
    N, K, L = a.ids, a.kinds, a.length
    R = N * K * L
    settings = EfficientFCParameters()
    gen = torch.Generator(device="cuda").manual_seed(11)
    perm = torch.randperm(R, device="cuda", generator=gen)
    row = torch.arange(R, device="cuda", dtype=torch.int64)[perm]           # (kind, id, time) order, shuffled
    kind = (row // (N * L)).to(torch.int32)
    ids = (row // L) % N * 3 - 1000
    sort = row % L
    values = torch.randn(R, device="cuda", generator=gen, dtype=torch.float32)
    del perm, row
    kinds = list(range(K))

    def timed(fn, reps):
        fn()                                          # warm-up: working regions, plans, twiddle table
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
            del out
        return float(np.median(ts)), [round(t, 1) for t in ts]

    res = {"workload": "EfficientFCParameters, %d ids x %d kinds x %d rows, shuffled long rows (%d)" % (N, K, L, R),
           "gpu": card(), "reps": a.reps, "frame_reps": a.frame_reps}
    run = lambda: extract_features_long_device(ids, values, sort, kind, kinds=kinds, default_fc_parameters=settings)  # noqa: E731
    res["long_device_ms"], res["long_device_all"] = timed(run, a.reps)
    X, row_ids, columns = run()
    res["n_features"] = len(columns)
    Xh, idh = X.cpu().numpy(), row_ids.cpu().numpy()
    del X, row_ids
    torch.cuda.empty_cache()
    df = pd.DataFrame({"id": ids.cpu().numpy(), "time": sort.cpu().numpy(), "kind": kind.cpu().numpy(),
                       "value": values.cpu().numpy()})
    frame = lambda: extract_features(df, column_id="id", column_sort="time", column_kind="kind", column_value="value",  # noqa: E731
                                     default_fc_parameters=settings)
    res["frame_ms"], res["frame_all"] = timed(frame, a.frame_reps)
    want = frame()
    nan_same = lambda u: np.where(np.isnan(u), np.nan, u).view(np.int64)   # noqa: E731
    res["equal_bits"] = bool(list(want.columns) == columns and np.array_equal(want.index.to_numpy(), idh)
                             and np.array_equal(nan_same(want.to_numpy()), nan_same(Xh)))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
