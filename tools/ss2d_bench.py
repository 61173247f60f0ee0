"""Standalone SS2D_1 on the fused kernels against its composed path (torch ops + this library's scan operator): SS2D_1(d_model=96) at
ssm_ratio 2 (E = 192, the module's default) and 1, B = 8, 64x64, bf16 autocast with fp32 parameters.  Times the inference forward
(no_grad) and one training forward + backward of each path, alternated in one process, CUDA events after warm-up, best of --rounds.
Prints one JSON line per (ssm_ratio, pass) with ms per call (every round and the best), the fused / composed speed-up, the largest
output difference between the paths, the card name and its power limit.

    python tools/ss2d_bench.py [--iters 20] [--warmup 3] [--rounds 5]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.scan_det_bench import alternate, gpu_info  # noqa: E402
from vmambair_b200 import archs  # noqa: E402

B, D, H, W = 8, 96, 64, 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ss2d_bench: needs a CUDA device")
    name, pl = gpu_info()
    for ratio in (2, 1):
        torch.manual_seed(ratio)
        m = archs.SS2D_1(d_model=D, ssm_ratio=ratio).cuda()
        x = torch.randn(B, D, H, W, device="cuda")
        dout = torch.randn(B, D, H, W, device="cuda", dtype=torch.bfloat16)
        xg = x.clone().requires_grad_()

        def infer(fused):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return m(x) if fused else m.forward_compose(x)

        def train(fused):
            archs.set_train_path("fused" if fused else "compose")
            try:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    y = m(xg)
                y.backward(dout)
            finally:
                archs.set_train_path("fused")

        diff = float((infer(True).float() - infer(False).float()).abs().max())
        for kind, fn in (("forward", infer), ("forward+backward", train)):
            rec = {"op": f"SS2D_1 {kind}", "B": B, "d_model": D, "ssm_ratio": ratio, "E": m.d_inner, "H": H, "W": W,
                   "dtype": "bf16 autocast", "gpu": name, "power_limit": pl}
            rec.update(alternate({"fused": lambda fn=fn: fn(True), "compose": lambda fn=fn: fn(False)}, a))
            rec["speedup"] = round(rec["compose_ms_min"] / rec["fused_ms_min"], 2)
            if kind == "forward":
                rec["max_abs_diff_fused_vs_compose"] = diff
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
