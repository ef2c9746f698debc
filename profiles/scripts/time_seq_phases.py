#!/usr/bin/env python
"""Splits the SEQ group's time by phase: builds of k_seq.cu whose short-series kernel (k_seq_small) leaves one phase
out (-DTSFX_SEQ_SKIP=k, see k_seq.cu), timed against the complete kernel with the per-group CUDA events
(TSFX_FLAG_TIMING).  The plan is the SEQ calculators of ComprehensiveFCParameters (five lempel_ziv_complexity and
five permutation_entropy columns) over device-resident random-normal series (1 M x 256 by default, the headline
shape, where every series runs k_seq_small); a SEQ-only plan runs the same kernel on the same descriptors, since
timed calls run the groups back to back on one stream.

    python profiles/scripts/time_seq_phases.py build DIR          # no GPU: one library per phase under DIR
    python profiles/scripts/time_seq_phases.py time DIR [--rounds 2] [--reps 5] [--series 1000000] [--len 256]

`build` needs the tree's own library built first (python -m tsfresh_b200.build): it recompiles k_seq.cu only and
links it with the tree's other objects.  `time` needs a CUDA device; it runs every phase's library in its own
process, the phases alternating in each round, and prints one JSON line: the card's name and power limit, the SEQ
times of every phase in ms, and the median time each phase accounts for (complete kernel minus the build without
it)."""
import argparse
import glob
import json
import os
import shutil
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
PHASES = ("none", "load_minmax", "lz_symbols", "lz_parse", "pe_counts_d6", "pe_d7_d8", "pe_keys_sort",
          "pe_finish_d6")      # index = TSFX_SEQ_SKIP
SEQ_CALCS = ("lempel_ziv_complexity", "permutation_entropy")


def build(out_dir):
    sys.path.insert(0, HERE)
    from tsfresh_b200 import build as b
    objs = [o for o in sorted(glob.glob(os.path.join(b.OBJ, "*.o"))) if os.path.basename(o) != "k_seq.o"]
    if not os.path.exists(os.path.join(b.OBJ, "k_seq.o")):
        raise SystemExit("build the tree first: python -m tsfresh_b200.build")
    for k, phase in enumerate(PHASES):
        pkg = os.path.join(out_dir, phase, "tsfresh_b200")
        os.makedirs(pkg, exist_ok=True)
        for py in glob.glob(os.path.join(b.HERE, "*.py")):
            shutil.copy(py, pkg)
        shutil.copytree(os.path.join(HERE, "include"), os.path.join(out_dir, phase, "include"), dirs_exist_ok=True)
        obj = os.path.join(pkg, "k_seq.o")
        cmd = [b.NVCC] + b.FLAGS + ["-DTSFX_SEQ_SKIP=%d" % k, "-c", os.path.join(b.CSRC, "k_seq.cu"), "-o", obj]
        subprocess.run(cmd, check=True)
        subprocess.run([b.NVCC, "-shared", "-o", os.path.join(pkg, "libtsfx.so"), obj] + objs + b.ARCH + ["-lcudart"],
                       check=True)
        os.remove(obj)
        # the copy has no csrc/: a stamp over what it does hold keeps _lib.load() from rebuilding it
        os.makedirs(os.path.join(pkg, "build"), exist_ok=True)
        with open(os.path.join(pkg, "build", "stamp"), "w") as f:
            f.write(b._digest([os.path.join(out_dir, phase, "include", "tsfx.h")]))
        print("built", phase, flush=True)


def one(root, n_series, length, reps):
    sys.path.insert(0, os.path.abspath(root))
    import torch
    from tsfresh_b200._lib import Context, DevicePlan
    from tsfresh_b200.plan import Plan
    from tsfresh_b200.settings import ComprehensiveFCParameters

    full = ComprehensiveFCParameters()
    plan = Plan({k: full[k] for k in SEQ_CALCS})
    gen = torch.Generator(device="cuda").manual_seed(44)
    x = torch.randn(n_series, length, device="cuda", generator=gen, dtype=torch.float32)
    out = torch.empty(n_series, plan.n_cols, device="cuda", dtype=torch.float64)
    ctx = Context(0)
    dp = DevicePlan(ctx, plan)
    try:
        dp.extract_dense_device(x.data_ptr(), n_series, length, out.data_ptr(), timing=True)      # warm-up
        ctx.sync()
        ms = []
        for _ in range(reps):
            dp.extract_dense_device(x.data_ptr(), n_series, length, out.data_ptr(), timing=True)
            ctx.sync()
            ms.append(ctx.timings()["seq"])
        kernels = ctx.last_kernels()
    finally:
        dp.close()
        ctx.close()
    print(json.dumps({"kernels": kernels, "seq_ms": ms}))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_all(out_dir, rounds, reps, n_series, length):
    ms = {p: [] for p in PHASES}
    kernels = None
    for _ in range(rounds):
        for phase in PHASES:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "one", os.path.join(out_dir, phase),
                                "--reps", str(reps), "--series", str(n_series), "--len", str(length)],
                               capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit("phase %s failed:\n%s" % (phase, r.stderr))
            line = json.loads(r.stdout.strip().splitlines()[-1])
            ms[phase] += [round(v, 3) for v in line["seq_ms"]]
            kernels = line["kernels"]
    med = {p: statistics.median(v) for p, v in ms.items()}
    print(json.dumps({"gpu": card(), "shape": [n_series, length], "kernels": kernels, "seq_ms": ms,
                      "phase_ms": {p: round(med["none"] - med[p], 2) for p in PHASES[1:]},
                      "complete_ms": round(med["none"], 2)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=("build", "time", "one"))
    ap.add_argument("dir")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--len", type=int, default=256)
    a = ap.parse_args()
    if a.what == "build":
        build(a.dir)
    elif a.what == "time":
        time_all(a.dir, a.rounds, a.reps, a.series, a.len)
    else:
        one(a.dir, a.series, a.len, a.reps)


if __name__ == "__main__":
    main()
