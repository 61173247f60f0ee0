"""Per-image time of PSNR + SSIM on the Y channel with crop_border 4 (the SR configs' validation metrics): vmambair_b200.metrics on the
device against the reference's host computation (float64 numpy / cv2, restated here operation by operation: to_y_channel, the mean
squared error, and five cv2.filter2D passes of the 11 x 11 Gaussian window per SSIM).

  div2k: one 2040 x 1356 uint8 BGR pair (HWC, resident on the device)
  4k:    one 3840 x 2160 uint8 BGR pair
  batch: B = 8, 512 x 512: float32 (8, 3, H, W) network output through tensor2img (quantize=True) against uint8 ground truth

Device: CUDA events around `--iters` calls of psnr_ssim after `--warmup` calls, per SSIM convention ('valid': pip basicsr's;
'reference': the vendored _ssim_cly).  Host: a host clock around one evaluation of the same pair.  The device and host measurements
alternate for `--rounds` rounds; the medians are reported, with the card name and its power limit, as one JSON line per workload.

    python tools/metrics_bench.py [--iters 20] [--warmup 3] [--rounds 5] [--host-rounds 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200.metrics import TAPS, psnr_ssim  # noqa: E402

try:
    import cv2
except ImportError:  # the host side is then reported as not measured
    cv2 = None

WORKLOADS = {"div2k": (1, 1356, 2040, False), "4k": (1, 2160, 3840, False), "batch": (8, 512, 512, True)}


def host_y(img):
    x = img.astype(np.float64).astype(np.float32) / 255.
    y = np.dot(x, [24.966, 128.553, 65.481]) + 16.0
    return (y / 255.).astype(np.float32) * 255.


def host_metrics(sr, gt, convention):
    """the reference's calculate_psnr and SSIM (Y, crop 4) of one uint8 HWC pair on the host"""
    a, b = (host_y(x.astype(np.float64)[4:-4, 4:-4]).astype(np.float64) for x in (sr, gt))
    mse = np.mean((a.astype(np.float32) - b.astype(np.float32)) ** 2)
    psnr = 20. * np.log10(255. / np.sqrt(mse))
    k = np.array(TAPS)[:, None]
    win = np.outer(k, k.T)
    kw = {} if convention == "valid" else {"borderType": cv2.BORDER_REPLICATE}
    f = [cv2.filter2D(v, -1, win, **kw) for v in (a, b, a * a, b * b, a * b)]
    if convention == "valid":
        f = [v[5:-5, 5:-5] for v in f]
    mu1, mu2 = f[0], f[1]
    s1, s2, s12 = f[2] - mu1 ** 2, f[3] - mu2 ** 2, f[4] - mu1 * mu2
    c1, c2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    ssim = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 ** 2 + mu2 ** 2 + c1) * (s1 + s2 + c2))
    return psnr, ssim.mean()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "metrics_bench needs a CUDA device"
    dev = torch.device("cuda", 0)
    name, power = gpu_info()
    for wl, (B, H, W, quant) in WORKLOADS.items():
        rng = np.random.default_rng(0)
        gt = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
        sr = np.clip(gt.astype(np.int16) + rng.integers(-12, 13, gt.shape), 0, 255).astype(np.uint8)
        gt_d = torch.from_numpy(gt).to(dev)
        if quant:  # the network output whose tensor2img is `sr`
            sr_d = torch.from_numpy(sr[..., ::-1].transpose(0, 3, 1, 2).astype(np.float32) / 255).to(dev)
        else:
            sr_d = torch.from_numpy(sr).to(dev)
        dev_ms = {"valid": [], "reference": []}
        host_ms = {"valid": [], "reference": []}
        for r in range(args.rounds):
            for conv in ("valid", "reference"):
                for _ in range(args.warmup):
                    psnr_ssim(sr_d, gt_d, 4, True, conv, quantize=quant)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(args.iters):
                    psnr_ssim(sr_d, gt_d, 4, True, conv, quantize=quant)
                e.record()
                e.synchronize()
                dev_ms[conv].append(s.elapsed_time(e) / (args.iters * B))
                if cv2 is not None and r < args.host_rounds:
                    t0 = time.perf_counter()
                    for i in range(B):
                        host_metrics(sr[i], gt[i], conv)
                    host_ms[conv].append((time.perf_counter() - t0) * 1e3 / B)
        rec = {"workload": wl, "batch": B, "H": H, "W": W, "input": "float32 (B,3,H,W) tensor2img vs uint8" if quant else "uint8 HWC",
               "gpu": name, "power_limit": power, "host_cpus": os.cpu_count(),
               "cv2_threads": cv2.getNumThreads() if cv2 is not None else None}
        for conv in ("valid", "reference"):
            rec[f"device_ms_per_image_{conv}"] = round(statistics.median(dev_ms[conv]), 4)
            rec[f"device_ms_rounds_{conv}"] = [round(v, 4) for v in dev_ms[conv]]
            rec[f"host_ms_per_image_{conv}"] = round(statistics.median(host_ms[conv]), 1) if host_ms[conv] else "not measured"
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
