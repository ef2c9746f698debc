#!/usr/bin/env python
"""Needs a CUDA device: what a call of extract_features_device, of a DeviceExtractor and the replay of a CUDA graph that
captured the DeviceExtractor call cost, on random-walk float32 series of 256 samples already on the device.

For every shape (1 024, 8 192 and 1 048 576 series by default) and ComprehensiveFCParameters / EfficientFCParameters,
the three variants fill the same preallocated `out` and are alternated within every repetition:
  eager      extract_features_device(x, out=out)
  extractor  ex(x, out=out) with ex = DeviceExtractor(N, length=L)
  graph      g.replay() of a torch.cuda.graph that captured ex(x_static, out=out_static)
Per call two numbers, medians over --reps repetitions after one warm-up:
  host_ms    perf_counter around the call alone (what the calling thread spends before it can enqueue more work)
  step_ms    CUDA events recorded before and after the call, read after a device synchronise (the work on the stream)
Each variant's result is also compared with the eager one bit for bit.  Prints one JSON line per (shape, settings)
with the card's name and power limit read in the same run.

    python profiles/scripts/time_device_extractor.py [--n 1024 8192 1048576] [--reps 20] [--out FILE]"""
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
    ap.add_argument("--n", type=int, nargs="+", default=[1024, 8192, 1 << 20])
    ap.add_argument("--length", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="append the JSON lines to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import torch
    from tsfresh_b200 import DeviceExtractor, extract_features_device
    from tsfresh_b200.settings import ComprehensiveFCParameters, EfficientFCParameters

    if not torch.cuda.is_available():
        raise SystemExit("time_device_extractor.py needs a CUDA device")
    gpu = card()
    L = a.length
    same = lambda u, v: bool(torch.equal(torch.nan_to_num(u, nan=-7.0), torch.nan_to_num(v, nan=-7.0)))   # noqa: E731
    for N in a.n:
        gen = torch.Generator(device="cuda").manual_seed(N)
        x = torch.randn((N, L), device="cuda", generator=gen, dtype=torch.float32).cumsum(1)
        for name, settings in (("comprehensive", ComprehensiveFCParameters()), ("efficient", EfficientFCParameters())):
            ex = DeviceExtractor(N, length=L, default_fc_parameters=settings)
            W = len(ex.columns)
            outs = {v: torch.empty((N, W), device="cuda", dtype=torch.float64) for v in ("eager", "extractor", "graph")}
            x_static = x.clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                ex(x_static, out=outs["graph"])
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ex(x_static, out=outs["graph"])
            calls = {"eager": lambda: extract_features_device(x, default_fc_parameters=settings, out=outs["eager"]),
                     "extractor": lambda: ex(x, out=outs["extractor"]),
                     "graph": g.replay}
            host = {v: [] for v in calls}
            step = {v: [] for v in calls}
            for rep in range(a.reps + 1):
                for v, fn in calls.items():
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    t0 = time.perf_counter()
                    fn()
                    t1 = time.perf_counter()
                    e1.record()
                    torch.cuda.synchronize()
                    if rep:                          # repetition 0 is the warm-up
                        host[v].append((t1 - t0) * 1e3)
                        step[v].append(e0.elapsed_time(e1))
            ex.check()
            res = {"workload": "%s %d x %d float32 random walks, device-resident" % (name, N, L), "gpu": gpu,
                   "n_features": W, "reps": a.reps}
            for v in calls:
                res[v + "_host_ms"] = round(float(np.median(host[v])), 4)
                res[v + "_step_ms"] = round(float(np.median(step[v])), 4)
            res["extractor_equals_eager"] = same(outs["extractor"], outs["eager"])
            res["graph_equals_eager"] = same(outs["graph"], outs["eager"])
            line = json.dumps(res)
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
            del ex, g, outs, x_static, calls
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
