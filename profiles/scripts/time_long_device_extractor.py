#!/usr/bin/env python
"""Needs a CUDA device: what a call of extract_features_long_device, of a DeviceLongExtractor and the replay of a CUDA
graph that captured the DeviceLongExtractor call cost, on shuffled long-format rows already on the device.

For every shape (1 024 and 100 000 ids by default) x 256 rows per (id, kind) series x 1 and 4 kinds, and
ComprehensiveFCParameters / EfficientFCParameters, the three variants are alternated within every repetition:
  eager      extract_features_long_device(ids, values, sort, kind, kinds=...)
  extractor  ex(ids, values, sort, kind, out=out) with ex = DeviceLongExtractor(rows, ids, 256, kinds=...)
  graph      g.replay() of a torch.cuda.graph that captured the extractor call on the same tensors
Per call two numbers, medians over --reps repetitions after one warm-up:
  host_ms    perf_counter around the call alone (what the calling thread spends before it can enqueue more work)
  step_ms    CUDA events recorded before and after the call, read after a device synchronise (the work on the stream)
The extractor's and the graph's first n_ids rows and their row ids are also compared with the eager result bit for bit.
Prints one JSON line per (shape, kinds, settings) with the card's name and power limit read in the same run.

    python profiles/scripts/time_long_device_extractor.py [--ids 1024 100000] [--kinds 1 4] [--reps 10] [--out FILE]"""
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
    ap.add_argument("--ids", type=int, nargs="+", default=[1024, 100_000])
    ap.add_argument("--kinds", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--length", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="append the JSON lines to this file as well")
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    import numpy as np
    import torch
    from tsfresh_b200 import DeviceLongExtractor, extract_features_long_device
    from tsfresh_b200.settings import ComprehensiveFCParameters, EfficientFCParameters

    if not torch.cuda.is_available():
        raise SystemExit("time_long_device_extractor.py needs a CUDA device")
    gpu = card()
    L = a.length
    same = lambda u, v: bool(torch.equal(torch.nan_to_num(u, nan=-7.0), torch.nan_to_num(v, nan=-7.0)))   # noqa: E731
    for N in a.ids:
        for K in a.kinds:
            n = N * K * L
            gen = torch.Generator(device="cuda").manual_seed(N * 8 + K)
            row = torch.arange(n, device="cuda")
            values = torch.randn((N * K, L), device="cuda", generator=gen).cumsum(1).reshape(-1)
            perm = torch.randperm(n, device="cuda", generator=gen)
            ids, sort, kind, values = (row // L % N)[perm], (row % L)[perm], (row // (L * N))[perm], values[perm]
            kinds = ["k%d" % k for k in range(K)] if K > 1 else None
            if K == 1:
                kind = None
            for name, settings in (("comprehensive", ComprehensiveFCParameters()), ("efficient", EfficientFCParameters())):
                ex = DeviceLongExtractor(n, N, L, kinds=kinds, default_fc_parameters=settings)
                W = len(ex.columns)
                outs = {v: torch.empty((N, W), device="cuda", dtype=torch.float64) for v in ("extractor", "graph")}
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    ex(ids, values, sort, kind, out=outs["graph"])
                torch.cuda.current_stream().wait_stream(side)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    graph_res = ex(ids, values, sort, kind, out=outs["graph"])
                res = {}
                calls = {"eager": lambda: extract_features_long_device(ids, values, sort, kind, kinds=kinds,
                                                                       default_fc_parameters=settings),
                         "extractor": lambda: ex(ids, values, sort, kind, out=outs["extractor"]),
                         "graph": lambda: (g.replay(), graph_res)[1]}
                host = {v: [] for v in calls}
                step = {v: [] for v in calls}
                for rep in range(a.reps + 1):
                    for v, fn in calls.items():
                        torch.cuda.synchronize()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        t0 = time.perf_counter()
                        res[v] = fn()
                        t1 = time.perf_counter()
                        e1.record()
                        torch.cuda.synchronize()
                        if rep:                      # repetition 0 is the warm-up
                            host[v].append((t1 - t0) * 1e3)
                            step[v].append(e0.elapsed_time(e1))
                ex.check()
                X, row_ids, _ = res["eager"]
                line = {"workload": "%s %d ids x %d kinds x %d rows, shuffled float32 random walks, device-resident"
                                    % (name, N, K, L), "gpu": gpu, "rows": n, "n_features": W, "reps": a.reps}
                for v in calls:
                    line[v + "_host_ms"] = round(float(np.median(host[v])), 4)
                    line[v + "_step_ms"] = round(float(np.median(step[v])), 4)
                for v in ("extractor", "graph"):
                    Xv, idv, nv = res[v]
                    m = int(nv)
                    line[v + "_equals_eager"] = (m == X.shape[0] and tuple(X.shape) == (N, W) and same(Xv[:m], X)
                                                 and torch.equal(idv[:m], row_ids))
                line = json.dumps(line)
                print(line, flush=True)
                if a.out:
                    with open(a.out, "a") as f:
                        f.write(line + "\n")
                del ex, g, outs, calls, res, graph_res, X, row_ids
                torch.cuda.empty_cache()
            del ids, sort, kind, values, row, perm
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
