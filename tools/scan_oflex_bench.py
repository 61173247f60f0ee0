"""Selective scan with fp32 output from bf16 inputs (selective_scan_cuda_oflex: out_float=True forward, fp32 dout backward) against
the plain bf16 operator (selective_scan_cuda_core: bf16 out, bf16 dout), forward and backward timed separately, the two variants
alternated in one process, CUDA events after warm-up.  Shapes: (B, D, L) = (8, 384, 4096) and (1, 384, 4096), N = 16, 4 groups
(the C = 96 four-direction scan at 64x64).  Prints one JSON line per shape with ms per call (every round and the best), the bytes
each variant moves, the card name and its power limit.

    python tools/scan_oflex_bench.py [--iters 50] [--warmup 5] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vmambair_b200 import ops  # noqa: E402

SHAPES = [(8, 384, 4096), (1, 384, 4096)]
N, G = 16, 4


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                            timeout=20).stdout.strip().splitlines()[0]
    except Exception as e:  # the record still names the card
        pl = f"unknown ({e})"
    return name, pl


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scan_oflex_bench: needs a CUDA device")
    name, pl = gpu_info()
    g = torch.Generator(device="cuda").manual_seed(0)
    for b, D, L in SHAPES:
        dt = torch.bfloat16
        u = torch.randn(b, D, L, device="cuda", generator=g).to(dt)
        delta = (0.1 * torch.randn(b, D, L, device="cuda", generator=g) - 4.0).to(dt)
        A = -torch.arange(1, N + 1, dtype=torch.float32, device="cuda").repeat(D, 1)
        Bm = torch.randn(b, G, N, L, device="cuda", generator=g).to(dt)
        Cm = torch.randn(b, G, N, L, device="cuda", generator=g).to(dt)
        Dv = torch.randn(D, device="cuda", generator=g)
        bias = torch.rand(D, device="cuda", generator=g)
        args = (u, delta, A, Bm, Cm, Dv, bias, True)
        dout32 = torch.randn(b, D, L, device="cuda", generator=g)
        variants = {}
        for k, of in (("core", False), ("oflex", True)):
            out, ck = ops.selective_scan_fwd(*args, need_ckpt=True, out_float=of)
            dout = dout32 if of else dout32.to(dt)
            variants[k] = (lambda of=of: ops.selective_scan_fwd(*args, need_ckpt=True, out_float=of),
                           lambda dout=dout, ck=ck, of=of: ops.selective_scan_bwd(*args[:7], dout, ck, True, dout_float=of))
        rec = {"B": b, "D": D, "L": L, "N": N, "G": G, "dtype": "bf16", "gpu": name, "power_limit": pl,
               "core_out_bytes": 2 * b * D * L, "oflex_out_bytes": 4 * b * D * L}
        times = {f"{k}_{p}": [] for k in variants for p in ("fwd", "bwd")}
        for _ in range(a.rounds):  # alternate the two variants
            for k, (f, bw) in variants.items():
                times[f"{k}_fwd"].append(timed(f, a.iters, a.warmup))
                times[f"{k}_bwd"].append(timed(bw, a.iters, a.warmup))
        for k, v in times.items():
            rec[f"{k}_ms"] = [round(t, 4) for t in v]
            rec[f"{k}_ms_min"] = round(min(v), 4)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
