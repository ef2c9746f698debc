#!/usr/bin/env python
"""Needs a CUDA device: what extract_features_device costs over the raw device-pointer call it wraps, on
ComprehensiveFCParameters over 1 000 000 x 256 random-normal float32 series (the bench.py workload).

Four ways to the same [N x n_features] float64 matrix, each timed with a host clock around the call and a device
synchronise, over --reps repetitions after one warm-up (the median is reported):
  api_dense     extract_features_device(values [N, L]) into a preallocated `out`
  api_csr       extract_features_device(values [N*L], begin, length) into the same `out`
  raw_dense     DevicePlan.extract_dense_device on the same pointers (no checked pass, no stream rebinding)
  frame         extract_features(long DataFrame) from host memory, result on the host (skipped with --no-frame)
The two API rows also check that their result equals raw_dense bit for bit.  Prints one JSON line with the card's name
and power limit read in the same run.

    python profiles/scripts/time_device_api.py [--n 1000000] [--reps 5] [--no-frame] [--out FILE]"""
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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-frame", action="store_true")
    ap.add_argument("--out", default=None, help="append the JSON line to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import torch
    from tsfresh_b200 import extract_features, extract_features_device
    from tsfresh_b200.extraction import _device_plan, get_context
    from tsfresh_b200.plan import Plan
    from tsfresh_b200.settings import ComprehensiveFCParameters

    if not torch.cuda.is_available():
        raise SystemExit("time_device_api.py needs a CUDA device")
    N, L = a.n, a.length
    settings = ComprehensiveFCParameters()
    plan = Plan(settings)
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn((N, L), device="cuda", generator=gen, dtype=torch.float32)
    flat = x.reshape(-1)
    begin = torch.arange(N, device="cuda", dtype=torch.int64) * L
    length = torch.full((N,), L, device="cuda", dtype=torch.int32)
    out = torch.empty((N, plan.n_cols), device="cuda", dtype=torch.float64)
    ref = torch.empty_like(out)
    ctx = get_context(0)
    dp = _device_plan(ctx, plan)

    def timed(fn):
        fn()                                          # warm-up: working regions, twiddle table, plans
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), [round(t, 2) for t in ts]

    def raw():
        with ctx.lock:
            dp.extract_dense_device(x.data_ptr(), N, L, ref.data_ptr())
            ctx.sync()

    res = {"workload": "ComprehensiveFCParameters %d x %d float32, device-resident" % (N, L), "gpu": card(),
           "n_features": plan.n_cols, "reps": a.reps}
    res["raw_dense_ms"], res["raw_dense_all"] = timed(raw)
    res["api_dense_ms"], res["api_dense_all"] = timed(lambda: extract_features_device(x, default_fc_parameters=settings, out=out))
    same = lambda u, v: bool(torch.equal(torch.nan_to_num(u, nan=-7.0), torch.nan_to_num(v, nan=-7.0)))   # noqa: E731
    res["api_dense_equals_raw"] = same(out, ref)
    out.fill_(0.0)
    res["api_csr_ms"], res["api_csr_all"] = timed(
        lambda: extract_features_device(flat, begin, length, default_fc_parameters=settings, out=out))
    res["api_csr_equals_raw"] = same(out, ref)
    # the checked pass alone reads the values once (dense: N*L floats; CSR: also begin and length)
    res["input_bytes"] = N * L * 4
    del out, ref
    torch.cuda.empty_cache()
    if not a.no_frame:
        import pandas as pd
        xh = x.cpu().numpy()
        df = pd.DataFrame({"id": np.repeat(np.arange(N, dtype=np.int64), L), "time": np.tile(np.arange(L, dtype=np.int64), N),
                           "value": xh.reshape(-1)})
        del xh
        res["frame_ms"], res["frame_all"] = timed(
            lambda: extract_features(df, column_id="id", column_sort="time", default_fc_parameters=settings))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
