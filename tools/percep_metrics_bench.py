"""Time of the perceptual metrics per image pair: vmambair_b200.lpips.LPIPS and .dists.DISTS (the whole batch in one call) against the
fp32 torch restatements (oracle/lpips_ref.py, oracle/dists_ref.py) run the scripts' way, one pair at a time with one forward per
image, on the same weights, alternated in one process.  fp32 inputs, convolutions at torch's default TF32 setting.  Workloads:
B = 8 pairs of 3 x 512 x 512, and B = 1 pair of 3 x 1356 x 2040 (a full-size NTIRE2020 / DIV2K validation image).

Reported per workload and metric: median and min-max ms per pair over `--steps` alternated rounds (CUDA events after a device
synchronise), library launches per call, and from a separate torch.profiler run the kernel time in this library's kernels against
all other kernels (cuDNN's convolutions, and torch's elementwise kernels on the restatement's side); the largest difference between
the two sides' values; the card name and power limit.

    python tools/percep_metrics_bench.py [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dists_ref, lpips_ref  # noqa: E402
from tools.perceptual_bench import time_round  # noqa: E402
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import _pmetric  # noqa: E402
from vmambair_b200.dists import DISTS  # noqa: E402
from vmambair_b200.lpips import LPIPS  # noqa: E402

WORKLOADS = {"b8_512x512": (8, 512, 512), "b1_1356x2040": (1, 1356, 2040)}


def kernel_split(prof):
    """(ms in this library's kernels (namespace vmb), ms in all other kernels, kernel launches) of a profile"""
    lib = other = 0.0
    n = 0
    for ev in prof.key_averages():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = ev.self_device_time_total / 1e3
        n += ev.count
        if "vmb::" in ev.key or "_ZN3vmb" in ev.key:
            lib += t
        else:
            other += t
    return lib, other, n


def models():
    torch.manual_seed(0)
    lp, di = LPIPS(pretrained=False, pnet_rand=True), DISTS(load_weights=False, vgg_weights=None)
    convs = lpips_ref.seeded_vgg16_convs(1)
    with torch.no_grad():
        for i, (w, b) in zip(_pmetric.CONVS, convs):
            lp.net.module(i).weight.copy_(w)
            lp.net.module(i).bias.copy_(b)
            di._module(i).weight.copy_(w)
            di._module(i).bias.copy_(b)
        for lin in lp.lins:
            lin.model[1].weight.copy_(torch.rand_like(lin.model[1].weight))
    return lp.cuda(), di.cuda(), [(w.cuda(), b.cuda()) for w, b in convs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "percep_metrics_bench measures on a GPU"
    torch.backends.cudnn.allow_tf32 = True
    lp, di, convs = models()
    lins = [lin.model[1].weight for lin in lp.lins]
    sl = lp.scaling_layer
    out = {"workload": "LPIPS(vgg) and DISTS per image pair, fp32 inputs in [0, 1], TF32 convolutions"}
    for tag, (B, H, W) in WORKLOADS.items():
        g = torch.Generator(device="cuda").manual_seed(B)
        x = torch.rand(B, 3, H, W, device="cuda", generator=g)
        y = (x + 0.05 * torch.randn(B, 3, H, W, device="cuda", generator=g)).clamp(0, 1)
        res = {}

        def lib_lpips():
            with torch.no_grad():
                res["lib_lpips"] = lp(x, y, normalize=True).reshape(-1)

        def torch_lpips():  # Metric/LPIPS.py: one pair per call, one forward per image
            with torch.no_grad():
                res["torch_lpips"] = torch.cat([lpips_ref.lpips(convs, lins, sl.shift, sl.scale, x[i:i + 1], y[i:i + 1], True)[0]
                                                .reshape(-1) for i in range(B)])

        def lib_dists():
            with torch.no_grad():
                res["lib_dists"] = di(x, y).reshape(-1)

        def torch_dists():
            with torch.no_grad():
                res["torch_dists"] = torch.stack([dists_ref.dists(convs, di.alpha, di.beta, x[i:i + 1], y[i:i + 1]) for i in range(B)])

        sides = {"library_lpips": lib_lpips, "torch_lpips": torch_lpips, "library_dists": lib_dists, "torch_dists": torch_dists}
        ms, launches = time_round(sides, args.steps, args.warmup)
        split = {}
        for name, fn in sides.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_steps):
                    fn()
                torch.cuda.synchronize()
            lib, other, n = kernel_split(prof)
            k = args.profile_steps
            split[name] = {"library_kernel_ms_per_call": lib / k, "other_kernel_ms_per_call": other / k, "kernels_per_call": n / k}
        out[tag] = {
            "ms_per_pair": {k: {s: v / B for s, v in m.items()} for k, m in ms.items()}, "library_launches_per_call": launches,
            "profile": split,
            "max_abs_diff": {"lpips": (res["lib_lpips"] - res["torch_lpips"]).abs().max().item(),
                             "dists": (res["lib_dists"] - res["torch_dists"]).abs().max().item()},
            "values": {k: v.tolist() for k, v in res.items()}}
        del x, y
        torch.cuda.empty_cache()
    gpu, pl = gpu_info()
    out.update(gpu=gpu, power_limit=pl, steps=args.steps)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
