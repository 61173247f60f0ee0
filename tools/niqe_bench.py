#!/usr/bin/env python
"""NIQE (vmambair_b200.niqe) time per call and per image, by CUDA events: batches of 2040 x 1356 uint8 BGR images (the DIV2K size),
Y channel, crop 0.  Prints one JSON line with the device's name and power limit.

  python tools/niqe_bench.py [--batch 8] [--iters 20] [--params tests/golden/niqe_pris_params.npz]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vmambair_b200 import niqe, ops  # noqa: E402


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def images(b, h, w, dev):
    g = torch.Generator().manual_seed(0)
    y = torch.linspace(0, 12, h)[:, None, None]
    x = torch.linspace(0, 18, w)[None, :, None]
    base = 0.5 + 0.3 * torch.sin(x + y * torch.rand(1, 1, 3, generator=g) * 3)
    return ((base[None] + 0.08 * torch.randn(b, h, w, 3, generator=g)).clamp(0, 1) * 255).round().to(torch.uint8).to(dev)


def time_call(fn, iters):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--height", type=int, default=1356)
    ap.add_argument("--width", type=int, default=2040)
    ap.add_argument("--params", default=os.path.join(ROOT, "tests", "golden", "niqe_pris_params.npz"))
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    p = niqe.load_params(a.params)
    x = images(a.batch, a.height, a.width, dev)
    ms = time_call(lambda: niqe.niqe(x, params=p), a.iters)
    ms1 = time_call(lambda: niqe.niqe(x[:1], params=p), a.iters)
    n0 = ops.launch_count()
    score = niqe.niqe(x, params=p)
    launches = ops.launch_count() - n0
    print(json.dumps({"device": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "batch": a.batch,
                      "size": [a.height, a.width], "ms_per_call": round(ms, 4), "ms_per_image": round(ms / a.batch, 4),
                      "ms_batch1": round(ms1, 4), "launches_per_call": launches,
                      "scores": [round(v, 6) for v in score.cpu().tolist()]}))


if __name__ == "__main__":
    main()
