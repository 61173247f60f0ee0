"""End-to-end ms per image of RealESRGANer.enhance (vmambair_b200.enhance: image conversions on the GPU) against the reference's
host-side conversions around the same TiledInference network (RealSR/VmambaIR/utils.py:174-243: numpy float conversion, BGR -> RGB,
F.pad on the device, fp32 result copied back, then clamp / transpose / x 255 / round in numpy), numpy uint8 image in, numpy uint8
image out.  The two paths alternate in one process; every round times `--iters` images after warm-up, host clock around work that
ends in a synchronise (both paths return host arrays).  Also times the network alone on resident planes.  bf16, tile = 0.

  realsr: MambaRealSR11 (default configuration), 512 x 512 -> 2048 x 2048
  sisr:   MambaSISR6 (default configuration), 960 x 540 -> 3840 x 2160

Prints one JSON line per workload with ms per image (every round and the median), the card name and its power limit.

    python tools/enhance_bench.py [--iters 5] [--warmup 2] [--rounds 5] [--only realsr|sisr]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import archs  # noqa: E402
from vmambair_b200.enhance import RealESRGANer  # noqa: E402

WORKLOADS = {"realsr": (archs.MambaRealSR11, 512, 512), "sisr": (archs.MambaSISR6, 540, 960)}


def host_path(up, img):
    """the reference's conversions (pre_pad 10, scale 4: no mod pad) around up.runner"""
    h, w = img.shape[:2]
    x = img.astype(np.float32) / 255
    x = x[:, :, ::-1]  # cv2.cvtColor(BGR2RGB)
    t = torch.from_numpy(np.transpose(x, (2, 0, 1)).copy()).float().unsqueeze(0).to(up.device)
    t = F.pad(t, (0, up.pre_pad, 0, up.pre_pad), "reflect")
    y = up.runner(t)
    y = y[:, :, :h * up.scale, :w * up.scale]
    out = y.data.squeeze().float().cpu().clamp_(0, 1).numpy()
    out = np.transpose(out[[2, 1, 0], :, :], (1, 2, 0))
    return (out * 255.0).round().astype(np.uint8)


def per_image_ms(fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", choices=sorted(WORKLOADS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("enhance_bench: needs a CUDA device")
    name, pl = gpu_info()
    torch.manual_seed(0)
    for tag, (ctor, h, w) in WORKLOADS.items():
        if a.only and tag != a.only:
            continue
        up = RealESRGANer(4, None, model=ctor().eval(), tile=0, pre_pad=10, dtype=torch.bfloat16)
        img = np.random.default_rng(0).integers(0, 256, (h, w, 3)).astype(np.uint8)
        dev_path = lambda: up.enhance(img)
        ref_path = lambda: host_path(up, img)
        got, want, again = dev_path()[0], ref_path(), dev_path()[0]
        d = np.abs(got.astype(int) - want.astype(int))
        r = np.abs(got.astype(int) - again.astype(int))  # the network's own run-to-run spread (fp32 atomics, rounded to bf16)
        planes = torch.rand(1, 3, (h + 17) // 8 * 8, (w + 17) // 8 * 8, device="cuda").to(torch.bfloat16)  # pre_pad 10, then to 8
        net = lambda: up.runner(planes)
        for f in (dev_path, ref_path, net):
            for _ in range(a.warmup):
                f()
        rounds = {"enhance": [], "host_conversions": [], "network_only": []}
        for _ in range(a.rounds):
            rounds["enhance"].append(per_image_ms(dev_path, a.iters))
            rounds["host_conversions"].append(per_image_ms(ref_path, a.iters))
            rounds["network_only"].append(per_image_ms(net, a.iters))
        rec = {"workload": tag, "input": [h, w], "output": list(got.shape), "dtype": "bf16", "gpu": name, "power_limit": pl,
               "ms_per_image_median": {k: round(statistics.median(v), 3) for k, v in rounds.items()},
               "ms_per_image_rounds": {k: [round(x, 3) for x in v] for k, v in rounds.items()},
               "paths_max_abs_diff": int(d.max()), "paths_frac_diff": float((d > 0).mean()),
               "repeat_max_abs_diff": int(r.max()), "repeat_frac_diff": float((r > 0).mean())}
        print(json.dumps(rec), flush=True)
        del up
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
