"""Per-group device time of the Comprehensive plan against the same plan with the parameter values beyond the grid:
autolag "t-stat" in place of "AIC", f_agg max / min / ptp / sum added to agg_autocorrelation and change_quantiles, attr
"intercept_stderr" added to the linregress calculators.  Dense float32 input on the device, CUDA events around every
kernel group (TSFX_FLAG_TIMING); the plans alternate, three runs each, after a warm-up.  Prints the card and its power
limit first: they belong to the numbers.

    python profiles/scripts/time_vocabulary.py [--shapes 1000000x256,250000x1024] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def plans():
    from tsfresh_b200.settings import ComprehensiveFCParameters
    base = dict(ComprehensiveFCParameters())
    tstat = dict(base, augmented_dickey_fuller=[dict(p, autolag="t-stat") if p.get("autolag", "AIC") == "AIC" else p
                                                for p in base["augmented_dickey_fuller"]])
    extra = dict(base)
    extra["agg_autocorrelation"] = base["agg_autocorrelation"] + [{"f_agg": f, "maxlag": 40} for f in ("max", "min", "ptp", "sum")]
    extra["change_quantiles"] = base["change_quantiles"] + [dict(p, f_agg=f) for p in base["change_quantiles"]
                                                             if p["f_agg"] == "mean" for f in ("max", "min", "ptp", "sum")]
    extra["linear_trend"] = base["linear_trend"] + [{"attr": "intercept_stderr"}]
    extra["agg_linear_trend"] = base["agg_linear_trend"] + [dict(p, attr="intercept_stderr") for p in base["agg_linear_trend"]
                                                             if p["attr"] == "slope"]
    return {"comprehensive": base, "tstat": tstat, "new_aggregators": extra}


def card():
    q = ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"]
    try:
        return subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1000000x256,250000x1024")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch

    from tsfresh_b200._lib import Context, DevicePlan
    from tsfresh_b200.plan import Plan
    print(json.dumps({"card": card()}))
    ctx = Context(0)
    for shape in a.shapes.split(","):
        n, L = (int(v) for v in shape.split("x"))
        x = torch.randn(n, L, device="cuda", dtype=torch.float32).cumsum(1)
        dps = {k: DevicePlan(ctx, Plan(v)) for k, v in plans().items()}
        outs = {k: torch.empty(n, Plan(v).n_cols, device="cuda", dtype=torch.float64) for k, v in plans().items()}
        for k, dp in dps.items():        # warm-up
            dp.extract_dense_device(x.data_ptr(), n, L, outs[k].data_ptr(), timing=True)
            ctx.sync()
        res = {k: [] for k in dps}
        for _ in range(a.runs):
            for k, dp in dps.items():
                dp.extract_dense_device(x.data_ptr(), n, L, outs[k].data_ptr(), timing=True)
                ctx.sync()
                res[k].append(ctx.timings())
        for k, runs in res.items():
            groups = {}
            for t in runs:
                for g, ms in t.items():
                    groups.setdefault(g, []).append(round(float(ms), 3))
            print(json.dumps({"shape": shape, "plan": k, "group_ms": groups}))
        for dp in dps.values():
            dp.close()
    ctx.close()


if __name__ == "__main__":
    main()
