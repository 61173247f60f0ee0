"""The z-gated selective scan (selective_scan_cuda: out_z = out * SiLU(z) from the forward launch, gate backward + scan backward)
against the ungated operator and against the composition a user would otherwise write (selective_scan_cuda_core under autograd, then
torch's out * F.silu(z)).  Forward alone (no_grad) and forward + backward, the variants alternated in one process, CUDA events after
warm-up.  Shapes: (B, D, L) = (8, 384, 4096) and (1, 384, 4096), bf16, N = 16, 4 groups.  Prints one JSON line per shape with ms per
call (every round and the best), the card name and its power limit.

    python tools/scan_z_bench.py [--iters 30] [--warmup 5] [--rounds 5]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.scan_oflex_bench import gpu_info, timed  # noqa: E402
from vmambair_b200.selective_scan import mamba_selective_scan_fn, selective_scan_fn  # noqa: E402

SHAPES = [(8, 384, 4096), (1, 384, 4096)]
N, G = 16, 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scan_z_bench: needs a CUDA device")
    name, pl = gpu_info()
    g = torch.Generator(device="cuda").manual_seed(0)
    for b, D, L in SHAPES:
        dt = torch.bfloat16
        mk = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)
        u, z, Bm, Cm = mk(b, D, L), mk(b, D, L), mk(b, G, N, L), mk(b, G, N, L)
        delta = (0.1 * torch.randn(b, D, L, device="cuda", generator=g) - 4.0).to(dt)
        A = -torch.arange(1, N + 1, dtype=torch.float32, device="cuda").repeat(D, 1)
        Dv = torch.randn(D, device="cuda", generator=g)
        bias = torch.rand(D, device="cuda", generator=g)
        dout = mk(b, D, L)
        leaves = [t.detach().requires_grad_() for t in (u, delta, A, Bm, Cm, Dv, z, bias)]
        uu, dd, AA, BB, CC, DD, zz, bb = leaves

        def gated():
            return mamba_selective_scan_fn(uu, dd, AA, BB, CC, DD, z=zz, delta_bias=bb, delta_softplus=True)

        def ungated():
            return mamba_selective_scan_fn(uu, dd, AA, BB, CC, DD, delta_bias=bb, delta_softplus=True)

        def composed():
            return selective_scan_fn(uu, dd, AA, BB, CC, DD, bb, True) * F.silu(zz)

        def fwd(f):
            def run():
                with torch.no_grad():
                    f()
            return run

        def fwd_bwd(f):
            def run():
                for t in leaves:
                    t.grad = None
                f().backward(dout)
            return run

        variants = {k: (fwd(f), fwd_bwd(f)) for k, f in (("gated", gated), ("ungated", ungated), ("composed", composed))}
        rec = {"B": b, "D": D, "L": L, "N": N, "G": G, "dtype": "bf16", "gpu": name, "power_limit": pl}
        times = {f"{k}_{p}": [] for k in variants for p in ("fwd", "fwd_bwd")}
        for _ in range(a.rounds):  # alternate the variants
            for k, (f, fb) in variants.items():
                times[f"{k}_fwd"].append(timed(f, a.iters, a.warmup))
                times[f"{k}_fwd_bwd"].append(timed(fb, a.iters, a.warmup))
        for k, v in times.items():
            rec[f"{k}_ms"] = [round(t, 4) for t in v]
            rec[f"{k}_ms_min"] = round(min(v), 4)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
