#!/usr/bin/env python
"""Needs a CUDA device: extract_features_sub_device against extract_features(add_sub_time_series_index(frame)) on the
same rows -- --ids recordings x --kinds kinds x --length rows (default 64 x 2 x 1 048 576 = 134 M rows), cut into
packages of --sub-length rows (default 256: 262 144 union packages, 524 288 (kind, package) series),
ComprehensiveFCParameters.

  sub_device     extract_features_sub_device on CUDA tensors (int64 ids and sort keys, int32 kind codes, float32
                 values), result on the device, over all --ids recordings
  sub_device_subset  the same call on the first --frame-ids recordings only
  frame          extract_features(add_sub_time_series_index(frame, sub_length, column_id="id", column_sort="time",
                 column_kind="kind"), column_id="id", ...) on the rows of the first --frame-ids recordings (default 2:
                 the host path needs minutes and tens of GB of host memory per few recordings), from host memory,
                 result on the host

Each is timed with a host clock around the call followed by torch.cuda.synchronize(), after one warm-up call, over
--reps repetitions (median reported; the frame's with --frame-reps).  The subset results of the two paths are compared
bit for bit (values with NaN as NaN, package names, column names).  Prints one JSON line with the card's name and power
limit read in the same run.

    python profiles/scripts/time_subseries_device.py [--ids 64] [--kinds 2] [--length 1048576] [--sub-length 256]
                                                     [--reps 3] [--frame-ids 2] [--frame-reps 1] [--out FILE]"""
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
    ap.add_argument("--ids", type=int, default=64)
    ap.add_argument("--kinds", type=int, default=2)
    ap.add_argument("--length", type=int, default=1 << 20)
    ap.add_argument("--sub-length", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frame-ids", type=int, default=2)
    ap.add_argument("--frame-reps", type=int, default=1)
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import pandas as pd
    import torch
    from tsfresh_b200 import ComprehensiveFCParameters, add_sub_time_series_index, extract_features, \
        extract_features_sub_device

    if not torch.cuda.is_available():
        raise SystemExit("time_subseries_device.py needs a CUDA device")
    N, K, L = a.ids, a.kinds, a.length
    R = N * K * L
    settings = ComprehensiveFCParameters()
    kinds = ["k%d" % k for k in range(K)]
    gen = torch.Generator(device="cuda").manual_seed(5)
    row = torch.arange(R, device="cuda", dtype=torch.int64)        # (id, kind, time) order
    ids = row // (K * L) * 7 - 200
    kind = (row // L % K).to(torch.int32)
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

    res = {"workload": "ComprehensiveFCParameters, packages of %d rows of %d ids x %d kinds x %d rows (%d rows)"
                       % (a.sub_length, N, K, L, R), "gpu": card(), "reps": a.reps, "frame_reps": a.frame_reps,
           "frame_ids": a.frame_ids}

    def device(n_ids):
        r = n_ids * K * L
        return extract_features_sub_device(ids[:r], values[:r], sort[:r], kind[:r], kinds=kinds, sub_length=a.sub_length,
                                           default_fc_parameters=settings)

    res["sub_device_ms"], res["sub_device_all"] = timed(lambda: device(N), a.reps)
    X, pnum, pid, columns = device(N)
    res["n_packages"], res["n_rows"], res["n_features"] = int(X.shape[0]) * K, int(X.shape[0]), len(columns)
    del X, pnum, pid
    torch.cuda.empty_cache()
    res["sub_device_subset_ms"], res["sub_device_subset_all"] = timed(lambda: device(a.frame_ids), a.reps)
    X, pnum, pid, columns = device(a.frame_ids)
    Xh, ph, ih = X.cpu().numpy(), pnum.cpu().numpy(), pid.cpu().numpy()
    del X, pnum, pid
    torch.cuda.empty_cache()
    r = a.frame_ids * K * L
    df = pd.DataFrame({"id": ids[:r].cpu().numpy(), "time": sort[:r].cpu().numpy(),
                       "kind": np.asarray(kinds, dtype=object)[kind[:r].cpu().numpy()], "value": values[:r].cpu().numpy()})
    frame = lambda: extract_features(add_sub_time_series_index(df, a.sub_length, column_id="id", column_sort="time",  # noqa: E731
                                                               column_kind="kind"),
                                     column_id="id", column_sort="time", column_kind="kind",
                                     default_fc_parameters=settings)
    res["frame_ms"], res["frame_all"] = timed(frame, a.frame_reps)
    want = frame()
    same = list(want.columns) == columns and want.index.tolist() == list(zip(ph.tolist(), ih.tolist()))
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
