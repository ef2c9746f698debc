#!/usr/bin/env python
"""Needs a CUDA device: times the ENTROPY group where it runs the tile kernel (series longer than 1 152 samples, which
bench.py never reaches).  An ENTROPY-only plan (the Comprehensive sample_entropy / approximate_entropy columns) over dense device-resident
series, per-group CUDA events (TSFX_FLAG_TIMING).  Prints one JSON line: the variant that ran, the ENTROPY time of every
repetition in ms, and a checksum of the result so two builds can be compared output for output.

    python profiles/scripts/time_entropy_tiles.py [--root TREE] [--series 100000] [--len 2048] [--reps 5] [--out FILE]

--root imports tsfresh_b200 from another checkout (to alternate two builds in one session)."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=HERE)
    ap.add_argument("--series", type=int, default=100000)
    ap.add_argument("--len", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also save the result matrix here (.npy)")
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    import torch
    from tsfresh_b200._lib import Context, DevicePlan
    from tsfresh_b200.plan import Plan
    from tsfresh_b200.settings import ComprehensiveFCParameters

    full = ComprehensiveFCParameters()
    settings = {k: full[k] for k in ("sample_entropy", "approximate_entropy")}
    plan = Plan(settings)
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(a.series, a.len, device="cuda", generator=gen, dtype=torch.float32)
    out = torch.empty(a.series, plan.n_cols, device="cuda", dtype=torch.float64)
    ctx = Context(0)
    dp = DevicePlan(ctx, plan)
    try:
        dp.extract_dense_device(x.data_ptr(), a.series, a.len, out.data_ptr(), timing=True)      # warm-up
        ctx.sync()
        ms = []
        for _ in range(a.reps):
            dp.extract_dense_device(x.data_ptr(), a.series, a.len, out.data_ptr(), timing=True)
            ms.append(ctx.timings()["entropy"])
        kernels = ctx.last_kernels()
    finally:
        dp.close()
        ctx.close()
    res = out.cpu().numpy()
    if a.out:
        np.save(a.out, res)
    print(json.dumps({"root": os.path.abspath(a.root), "shape": [a.series, a.len], "kernels": kernels,
                      "entropy_ms": [round(v, 3) for v in ms], "sha256": hashlib.sha256(res.tobytes()).hexdigest()}))


if __name__ == "__main__":
    main()
