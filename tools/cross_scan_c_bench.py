"""Forward + backward of cross_selective_scanC (one fused kernel forward, per-image kernel + fixed-order batch sum backward) against
the reference's torch composition (CrossScanC gather, x_proj / dt_proj einsums and bias add, fp32 casts, the flat selective_scan_fn,
CrossMergeC, transpose), alternated in one process, CUDA events after warm-up.  Shapes: the RealSR channel calls (D = 1, N = 16,
L = C, R = ceil(C/16)) at B = 1, 4, 8, fp32 input as SS2D_1.cforward_corev2 pools it.  Prints one JSON line per shape with ms per
step (best of the rounds), library launches per step, the card name and its power limit.

    python tools/cross_scan_c_bench.py [--iters 100] [--warmup 10] [--rounds 3]
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

CS = [48, 96, 192, 384]
BS = [1, 4, 8]


def composed(x, m):
    """the reference's cross_selective_scanC (MambaRealSR11_arch.py:478-534) in torch around the library's flat scan"""
    B, D, L = x.shape
    N, R = m.Ac_logs.shape[1], m.dtc_projs_weight.shape[2]
    xs = cs.CrossScanC.apply(x)
    x_dbl = torch.einsum("b k d l, k c d -> b k c l", xs, m.xc_proj_weight)
    dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
    dts = torch.einsum("b k r l, k d r -> b k d l", dts, m.dtc_projs_weight)
    ys = selective_scan_fn(xs.reshape(B, -1, L).float(), dts.contiguous().view(B, -1, L).float(), -torch.exp(m.Ac_logs.float()),
                           Bs.contiguous().float(), Cs.contiguous().float(), m.Dsc.float(), m.dtc_projs_bias.view(-1).float(),
                           True).view(B, 2, -1, L)
    y = cs.CrossMergeC.apply(ys).transpose(1, 2).unsqueeze(2).contiguous()
    return m.channel_norm(y).to(x.dtype)


def ours(x, m):
    return cs.cross_selective_scanC(x, m.xc_proj_weight, None, m.dtc_projs_weight, m.dtc_projs_bias, m.Ac_logs, m.Dsc, m.channel_norm)


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
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    torch.manual_seed(0)
    name, pl = gpu_info()
    for C in CS:
        m = archs.SS2D_1(d_model=C, ssm_ratio=1, variant="realsr").cuda()
        for B in BS:
            x = torch.randn(B, 1, C, device="cuda", requires_grad=True)
            g = torch.randn(B, C, 1, 1, device="cuda")
            rec = {"B": B, "L": C, "R": m.dtc_projs_weight.shape[2], "N": m.Ac_logs.shape[1], "dtype": "fp32", "gpu": name,
                   "power_limit": pl}
            times = {"ours": [], "composed": []}
            for k, fn in (("ours", ours), ("composed", composed)):
                fn(x, m).backward(g)
                n0 = ops.launch_count()
                fn(x, m).backward(g)
                rec[f"{k}_launches"] = ops.launch_count() - n0
            for _ in range(a.rounds):  # alternate the two
                for k, fn in (("ours", ours), ("composed", composed)):
                    for _ in range(a.warmup):
                        fn(x, m).backward(g)
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    for _ in range(a.iters):
                        fn(x, m).backward(g)
                    e.record()
                    torch.cuda.synchronize()
                    times[k].append(s.elapsed_time(e) / a.iters)
            for k, v in times.items():
                rec[f"{k}_ms"] = [round(t, 4) for t in v]
                rec[f"{k}_ms_min"] = round(min(v), 4)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
