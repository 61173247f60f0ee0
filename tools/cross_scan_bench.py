"""Forward + backward of cross_selective_scan (direction-aware grouped kernels) against the gathered composition (CrossScan gather,
x_proj / dt_proj einsums, the flat selective_scan_fn, CrossMerge), alternated in one process, CUDA events after warm-up.  Prints one
JSON line per shape with ms per step, library launches and the unique bytes each moves, plus the card name and power limit.

    python tools/cross_scan_bench.py [--iters 50] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vmambair_b200 import archs, ops  # noqa: E402
from vmambair_b200 import cross_scan as cs  # noqa: E402
from vmambair_b200.selective_scan import selective_scan_fn  # noqa: E402

SHAPES = [(4, 48, 64, 64), (4, 96, 64, 64), (1, 48, 256, 256)]  # (B, D, H, W), bf16, d_state 16


def composed(x, p, norm):
    B, D, H, W = x.shape
    L = H * W
    N, R = p["A_logs"].shape[1], p["dt_projs_weight"].shape[2]
    xs = cs.CrossScan.apply(x)
    x_dbl = torch.einsum("b k d l, k c d -> b k c l", xs, p["x_proj_weight"].to(x.dtype))
    dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
    dts = torch.einsum("b k r l, k d r -> b k d l", dts, p["dt_projs_weight"].to(x.dtype))
    ys = selective_scan_fn(xs.reshape(B, -1, L), dts.reshape(B, -1, L).contiguous(), -torch.exp(p["A_logs"].float()), Bs.contiguous(),
                           Cs.contiguous(), p["Ds"].float(), p["dt_projs_bias"].reshape(-1).float(), True)
    y = cs.CrossMerge.apply(ys.view(B, 4, D, H, W)).float()
    return norm(y.view(B, D, H, W)).to(x.dtype)


def ours(x, p, norm):
    return cs.cross_selective_scan(x, p["x_proj_weight"], None, p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"], p["Ds"], norm)


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                            timeout=20).stdout.strip().splitlines()[0]
    except Exception as e:  # the record still names the card
        pl = f"unknown ({e})"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    torch.manual_seed(0)
    name, pl = gpu_info()
    for B, D, H, W in SHAPES:
        m = archs.SS2D_1(d_model=D, ssm_ratio=1).cuda()
        p = dict(x_proj_weight=m.x_proj_weight, dt_projs_weight=m.dt_projs_weight, dt_projs_bias=m.dt_projs_bias, A_logs=m.A_logs, Ds=m.Ds)
        x = torch.randn(B, D, H, W, device="cuda", dtype=torch.bfloat16, requires_grad=True)
        g = torch.randn(B, D, H, W, device="cuda", dtype=torch.bfloat16)
        rec = {"shape": [B, D, H, W], "dtype": "bf16", "gpu": name, "power_limit": pl}
        times = {"ours": [], "gathered": []}
        for k, fn in (("ours", ours), ("gathered", composed)):
            n0 = ops.launch_count()
            fn(x, p, m.out_norm).backward(g)
            rec[f"{k}_launches"] = ops.launch_count() - n0
            recs = []
            ops.set_timing(recs)
            fn(x, p, m.out_norm).backward(g)
            ops.set_timing(None)
            torch.cuda.synchronize()
            rec[f"{k}_library_bytes"] = int(sum(r[1] for r in recs))
        for _ in range(a.rounds):  # alternate the two
            for k, fn in (("ours", ours), ("gathered", composed)):
                for _ in range(a.warmup):
                    fn(x, p, m.out_norm).backward(g)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(a.iters):
                    fn(x, p, m.out_norm).backward(g)
                e.record()
                torch.cuda.synchronize()
                times[k].append(s.elapsed_time(e) / a.iters)
        for k, v in times.items():
            rec[f"{k}_ms"] = [round(t, 4) for t in v]
            rec[f"{k}_ms_min"] = round(min(v), 4)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
