"""Launch-configuration sweep of the TMA-staged selective-scan forward: (rows per warp RB, state split SS) per batch size,
against the generic kernel (VMB_SCAN_TMA=0) on the same tensors; also checks that every configuration reproduces the generic
kernel's output.  u = (B, 4*C, L), N = 16, G = 4 -- SURVEY.md 8(d) micro-benchmark shape."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vmambair_b200 import ops
from tools.scan_bench import bench


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="+", default=[1, 2, 4, 8, 32])
    ap.add_argument("--C", type=int, default=96)
    ap.add_argument("--L", type=int, default=4096)
    ap.add_argument("--dtype", default="bf16")
    ap.add_argument("--ckpt", action="store_true")
    a = ap.parse_args()
    dev = "cuda"
    dt = {"bf16": torch.bfloat16, "fp32": torch.float32}[a.dtype]
    s = 2 if dt != torch.float32 else 4
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    K, N = 4, 16
    D = K * a.C
    for B in a.B:
        torch.manual_seed(0)
        u = torch.randn(B, D, a.L, device=dev).to(dt)
        delta = (0.5 * torch.rand(B, D, a.L, device=dev)).to(dt)
        A = -0.5 * torch.rand(D, N, device=dev)
        Bm = torch.randn(B, K, N, a.L, device=dev).to(dt)
        Cm = torch.randn(B, K, N, a.L, device=dev).to(dt)
        Dv = torch.randn(D, device=dev)
        bias = 0.5 * torch.rand(D, device=dev)
        run = lambda: ops.selective_scan_fwd(u, delta, A, Bm, Cm, Dv, bias, True, a.ckpt)
        os.environ["VMB_SCAN_TMA"] = "0"
        os.environ.pop("VMB_SCAN_RB", None)
        os.environ.pop("VMB_SCAN_SS", None)
        ref, _ = run()
        ms0 = bench(run, flush=flush)
        byts = B * (s * (3 * D * a.L + 2 * K * N * a.L) + 4 * (D * N + 2 * D))
        print(json.dumps(dict(B=B, cfg="generic", us_per_img=round(ms0 * 1e3 / B, 2), GBps=round(byts / ms0 / 1e6, 1))), flush=True)
        os.environ["VMB_SCAN_TMA"] = "1"
        cfgs = [(0, 0), (2, 1), (2, 2), (2, 4), (4, 1), (4, 2), (4, 4), (8, 1), (8, 2), (8, 4)]
        for rb, ss in cfgs:
            if rb:
                os.environ["VMB_SCAN_RB"], os.environ["VMB_SCAN_SS"] = str(rb), str(ss)
            try:
                out, _ = run()
                torch.cuda.synchronize()
            except RuntimeError as e:
                print(json.dumps(dict(B=B, cfg=f"rb{rb}ss{ss}", error=str(e)[:120])), flush=True)
                continue
            err = float((out.float() - ref.float()).abs().max())
            ms = bench(run, flush=flush)
            print(json.dumps(dict(B=B, cfg=f"rb{rb}ss{ss}" if rb else "auto", us_per_img=round(ms * 1e3 / B, 2),
                                  GBps=round(byts / ms / 1e6, 1), frac=round(byts / ms / 1e6 / 6486.5, 4),
                                  speedup_vs_generic=round(ms0 / ms, 2), max_abs_diff_vs_generic=err)), flush=True)


if __name__ == "__main__":
    main()
