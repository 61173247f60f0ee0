"""Time of one Real-ESRNet synthesis step (MambaRealSR.feed_data's degradation, before crop and pool) at the recipe's shapes: batch 9,
3 x 600 x 600 GT, 21 x 21 blur and sinc kernels, RealSR/options/mambaSR11_x4.yml's options.  vmambair_b200.degradations against the
torch restatement oracle/degradations_ref.py run in float32 on the same draws: the stand-in for basicsr's chains of small torch ops
(without basicsr's host synchronisations, so the restatement's numbers flatter it).

Per round r (seed r for random, numpy and torch, so both sides take the same branches), the library and the restatement alternate;
each call is timed with CUDA events after a device synchronise.  Reported: the median ms per batch and the spread (min, max) over
`--rounds`; kernel launches per batch, counted with torch.profiler over the same seeds; per library kernel, its achieved bytes/s (the
bytes the operation must move, over its event-timed duration) against the H100 SXM's 3.35 TB/s; the card name and power limit.

    python tools/degrade_bench.py [--rounds 20] [--warmup 8]
"""
import argparse
import collections
import json
import os
import random
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import degradations_ref as R  # noqa: E402
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import degradations as D  # noqa: E402
from vmambair_b200 import ops  # noqa: E402

OPT = dict(gt_usm=False, resize_prob=[0.2, 0.7, 0.1], resize_range=[0.15, 1.5], gaussian_noise_prob=0.5, noise_range=[1, 30],
           poisson_scale_range=[0.05, 3], gray_noise_prob=0.4, jpeg_range=[30, 95], second_blur_prob=0.8,
           resize_prob2=[0.3, 0.4, 0.3], resize_range2=[0.3, 1.2], gaussian_noise_prob2=0.5, noise_range2=[1, 25],
           poisson_scale_range2=[0.05, 2.5], gray_noise_prob2=0.4, jpeg_range2=[30, 95], gt_size=256, queue_size=180)
HBM_BPS = 3.35e12


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "degrade_bench measures on a GPU"
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    b, H = 9, 600
    gt = torch.rand(b, 3, H, H, generator=g, device=dev)
    kern = [torch.rand(b, 21, 21, generator=g, device=dev) for _ in range(3)]
    kern = [k / k.sum((1, 2), keepdim=True) for k in kern]
    deg = D.RealESRNetDegradation(OPT, 4)
    sides = {"library": lambda: deg.degrade(gt, *kern)[0],
             "restatement_fp32": lambda: R.feed_data(gt, *kern, OPT, 4, dtype=torch.float32)[0]}
    for r in range(args.warmup):
        for fn in sides.values():
            seed_all(r)
            fn()
    torch.cuda.synchronize()
    times = collections.defaultdict(list)
    for r in range(args.rounds):
        for name, fn in sides.items():
            seed_all(1000 + r)
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
    # launches per batch over a few seeds, in a run of their own
    launches = {}
    nseeds = 4
    for name, fn in sides.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for r in range(nseeds):
                seed_all(1000 + r)
                fn()
            torch.cuda.synchronize()
        n = sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in ev.name)
        launches[name] = n / nseeds
    # per library operation: bytes / event time
    rec = []
    ops.set_timing(rec)
    for r in range(nseeds):
        seed_all(1000 + r)
        sides["library"]()
    torch.cuda.synchronize()
    ops.set_timing(None)
    per = collections.defaultdict(lambda: [0, 0.0, 0])
    for tag, nbytes, s, e in rec:
        per[tag][0] += nbytes
        per[tag][1] += s.elapsed_time(e) / 1e3
        per[tag][2] += 1
    kernels = {tag: {"calls": n, "ms_per_call": 1e3 * t / n, "bytes_per_s": nb / t, "of_3.35TBps": nb / t / HBM_BPS}
               for tag, (nb, t, n) in per.items()}
    name, pl = gpu_info()
    print(json.dumps({"workload": "realesrnet_degrade b=9 3x600x600", "gpu": name, "power_limit": pl, "rounds": args.rounds,
                      "ms_per_batch": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
                      "launches_per_batch": launches, "library_kernels": kernels}, indent=1))


if __name__ == "__main__":
    main()
