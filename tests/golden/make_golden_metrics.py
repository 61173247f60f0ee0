#!/usr/bin/env python
"""Generate tests/golden/metrics_ref.npz from the REAL reference's image metrics: calculate_psnr / calculate_ssim
(Deraining/basicsr/metrics/psnr_ssim.py, with to_y_channel and bgr2ycbcr), Deraining/Deraining/utils.py's calculate_ssim (the per-channel
valid-region SSIM of pip basicsr) and tensor2img (SRGAN/VmambaIR/utils/img_util.py).  Runs on a development machine with the reference
checkout (../reference or $VMB_REFERENCE_DIR) and cv2; no test imports it.

  python tests/golden/make_golden_metrics.py

Nothing is copied from the reference: its functions are AST-extracted at run time (psnr_ssim.py imports skimage, so the module itself is
not imported), and `.cuda()` is stubbed so that _ssim_3d runs its float32 Conv3d on the CPU.  Stored: the seeded inputs, the
reference's results, cv2.getGaussianKernel(11, 1.5), and the SHA-256 of to_y_channel over all 2^24 8-bit BGR triples (a 4096 x 4096
image whose pixel i holds B = i >> 16, G = (i >> 8) & 255, R = i & 255), whose float32 bytes are hashed in row order.
"""
import ast
import hashlib
import math
import os
import sys

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402

OUT = mg.OUT


def extract(path, names, ns):
    tree = ast.parse(open(path).read())
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert {f.name for f in fns} == set(names), (path, names)
    exec(compile(ast.Module(fns, []), path, "exec"), ns)


def reference():
    ns = {"np": np, "cv2": cv2, "torch": torch, "math": math}
    b = f"{mg.REF}/Deraining/basicsr"
    extract(f"{b}/utils/matlab_functions.py", ["bgr2ycbcr", "_convert_input_type_range", "_convert_output_type_range"], ns)
    extract(f"{b}/metrics/metric_util.py", ["reorder_image", "to_y_channel"], ns)
    extract(f"{b}/metrics/psnr_ssim.py", ["calculate_psnr", "calculate_ssim", "_ssim_cly", "_ssim_3d", "_3d_gaussian_calculator",
                                           "_generate_3d_gaussian_kernel"], ns)
    utils = {"np": np, "cv2": cv2, "math": math}
    extract(f"{mg.REF}/Deraining/Deraining/utils.py", ["calculate_ssim", "ssim"], utils)
    ns["utils_ssim"] = utils["calculate_ssim"]
    extract(f"{mg.REF}/SRGAN/VmambaIR/utils/img_util.py", ["tensor2img"], ns)
    return ns


def cases(rng):
    """(name, img1, img2, crop_border, input_order, as_tensor); img2 is img1 plus seeded noise unless the case says otherwise"""
    def u8(*s):
        return rng.integers(0, 256, s, dtype=np.uint8)

    def noisy(x, hi, sd):
        y = x.astype(np.float64) + rng.normal(0, sd, x.shape)
        return np.clip(np.rint(y) if x.dtype.kind == "u" else y, 0, hi).astype(x.dtype)

    out = []
    a = u8(37, 45, 3)
    out.append(("u8_hwc_crop4", a, noisy(a, 255, 6), 4, "HWC", False))
    a = rng.integers(0, 65536, (29, 33, 3), dtype=np.uint16)
    out.append(("u16_hwc_crop0", a, noisy(a, 65535, 900), 0, "HWC", False))
    a = rng.random((24, 31, 3), dtype=np.float32)
    out.append(("f32_unit_crop3", a, noisy(a, 1, 0.03).astype(np.float32), 3, "HWC", False))
    a = rng.random((40, 28, 3)) * 255
    out.append(("f64_255_crop5", a, noisy(a, 255, 4.0), 5, "HWC", False))
    a = u8(3, 26, 30)
    out.append(("u8_chw_crop2", a, noisy(a, 255, 10), 2, "CHW", False))
    a = u8(33, 21)
    out.append(("u8_gray_crop1", a, noisy(a, 255, 8), 1, "HWC", False))
    a = u8(50, 47, 3)
    out.append(("u8_odd_crop7", a, noisy(a, 255, 3), 7, "HWC", False))
    a = u8(9, 14, 3)
    out.append(("u8_small", a, noisy(a, 255, 12), 0, "HWC", False))
    a = u8(15, 18, 3)
    out.append(("u8_small_after_crop", a, noisy(a, 255, 12), 3, "HWC", False))
    a = u8(23, 19, 3)
    out.append(("u8_identical", a, a.copy(), 2, "HWC", False))
    a = rng.random((3, 27, 25), dtype=np.float32) * 255
    out.append(("tensor_f32_255", a, noisy(a, 255, 5).astype(np.float32), 4, "HWC", True))
    a = u8(1, 3, 22, 26)
    out.append(("tensor_u8_4d", a, noisy(a, 255, 7), 1, "HWC", True))
    return out


def net_output(rng, h, w):
    """(3, h, w) float32 RGB with exact (k + 0.5) / 255 ties (k + 0.5 is exact times 255 in float32 only where the product rounds to it;
    both sides of the tie are covered) and values outside [0, 1]"""
    x = rng.normal(0.5, 0.35, (3, h, w)).astype(np.float32)
    k = rng.integers(0, 255, (3, h, w))
    tie = rng.random((3, h, w)) < 0.3
    x[tie] = ((k[tie] + 0.5) / 255).astype(np.float32)
    return x


def main():
    ref = reference()
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    rng = np.random.default_rng(20261017)
    data = {"gauss": cv2.getGaussianKernel(11, 1.5)[:, 0]}
    names = []
    for name, a, b, crop, order, as_tensor in cases(rng):
        names.append(name)
        data[f"{name}/img1"], data[f"{name}/img2"] = a, b
        data[f"{name}/meta"] = np.array([crop, order == "CHW", as_tensor])
        x1, x2 = (torch.from_numpy(a), torch.from_numpy(b)) if as_tensor else (a, b)
        for y in (0, 1):
            data[f"{name}/psnr_y{y}"] = np.float64(ref["calculate_psnr"](x1, x2, crop, order, test_y_channel=bool(y)))
            with np.errstate(all="ignore"):
                data[f"{name}/ssim_y{y}"] = np.float64(ref["calculate_ssim"](x1, x2, crop, order, test_y_channel=bool(y)))
            # the valid-region convention on the same cropped (and Y-converted) float64 images
            h1 = ref["reorder_image"](a.squeeze(0).transpose(1, 2, 0) if as_tensor and a.ndim == 4 else
                                      a.transpose(1, 2, 0) if as_tensor else a, order).astype(np.float64)
            h2 = ref["reorder_image"](b.squeeze(0).transpose(1, 2, 0) if as_tensor and b.ndim == 4 else
                                      b.transpose(1, 2, 0) if as_tensor else b, order).astype(np.float64)
            if crop:
                h1, h2 = h1[crop:-crop, crop:-crop], h2[crop:-crop, crop:-crop]
            if y:
                h1, h2 = ref["to_y_channel"](h1).astype(np.float64), ref["to_y_channel"](h2).astype(np.float64)
            with np.errstate(all="ignore"):
                data[f"{name}/ssim_valid_y{y}"] = np.float64(ref["utils_ssim"](h1, h2, 0))
    # network outputs through tensor2img, scored against a uint8 ground truth
    for i, (h, w) in enumerate([(20, 24), (17, 29)]):
        x = net_output(rng, h, w)
        gt = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        q = ref["tensor2img"](torch.from_numpy(x))
        data[f"quant{i}/x"], data[f"quant{i}/gt"], data[f"quant{i}/tensor2img"] = x, gt, q
        for y in (0, 1):
            data[f"quant{i}/psnr_y{y}"] = np.float64(ref["calculate_psnr"](q, gt, 2, test_y_channel=bool(y)))
            data[f"quant{i}/ssim_y{y}"] = np.float64(ref["calculate_ssim"](q, gt, 2, test_y_channel=bool(y)))
    # every 8-bit BGR triple through to_y_channel, hashed
    sha = hashlib.sha256()
    i = np.arange(4096 * 256, dtype=np.int64)
    for r0 in range(0, 4096, 256):
        j = i + r0 * 4096
        img = np.stack([j >> 16, (j >> 8) & 255, j & 255], axis=-1).reshape(256, 4096, 3).astype(np.float64)
        sha.update(np.ascontiguousarray(ref["to_y_channel"](img)[..., 0], dtype="<f4").tobytes())
    data["y_all_triples_sha256"] = np.frombuffer(sha.digest(), dtype=np.uint8)
    data["cases"] = np.array(names)
    path = os.path.join(OUT, "metrics_ref.npz")
    np.savez_compressed(path, **data)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
