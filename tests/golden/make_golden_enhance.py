#!/usr/bin/env python
"""Generate tests/golden/enhance_ref.npz (+ the networks' weights, enhance_net_{realsr,sisr}.npz) and enhance_cv2.npz from the REAL reference's `RealESRGANer`
(RealSR/VmambaIR/utils.py:14-243) and from OpenCV.  Runs on a development machine with the reference checkout (../reference or
$VMB_REFERENCE_DIR) and cv2; no test imports it.

  python tests/golden/make_golden_enhance.py

Nothing is copied from the reference: the class is AST-extracted at run time, as make_golden.py does for selective_scan_ref, and
driven on the CPU in fp32 with tiny reference networks (MambaRealSR11 / MambaSISR6, loaded through make_golden.py's stubs; the scan
is the reference's own selective_scan_ref).  Only seeded inputs, the networks' weights and the outputs are stored.  Every geometry
is one the unmodified reference can run: H + pre_pad and W + pre_pad are multiples of 8, and so is every tile.
"""
import ast
import math
import os
import queue
import sys
import tempfile
import threading

import cv2
import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402

OUT = mg.OUT

# (name, net, mode, dtype, hi (exclusive upper bound of the values), h, w, pre_pad, tile, tile_pad, outscale, alpha_upsampler)
CASES = [
    ("rgb8", "realsr", "RGB", np.uint8, 256, 22, 30, 10, 0, 10, None, "realesrgan"),
    ("rgba8_net", "realsr", "RGBA", np.uint8, 256, 22, 30, 10, 0, 10, None, "realesrgan"),
    ("rgba8_linear", "realsr", "RGBA", np.uint8, 256, 22, 30, 10, 0, 10, None, "bilinear"),
    ("gray8", "sisr", "L", np.uint8, 256, 24, 32, 0, 0, 10, None, "realesrgan"),
    ("rgb16", "sisr", "RGB", np.uint16, 65536, 24, 32, 0, 0, 10, 3.5, "realesrgan"),
    ("rgba16_linear", "sisr", "RGBA", np.uint16, 65536, 24, 16, 0, 0, 10, None, "bilinear"),
    ("rgb16_low", "realsr", "RGB", np.uint16, 257, 22, 30, 10, 0, 10, None, "realesrgan"),
    ("rgb8_tiled", "realsr", "RGB", np.uint8, 256, 22, 30, 10, 16, 8, None, "realesrgan"),
    ("rgba8_tiled", "sisr", "RGBA", np.uint8, 256, 32, 24, 0, 16, 8, None, "realesrgan"),
    ("rgb8_same", "sisr", "RGB", np.uint8, 256, 24, 32, 0, 0, 10, 4.0, "realesrgan"),
    ("rgb8_down", "realsr", "RGB", np.uint8, 256, 22, 30, 10, 0, 10, 2.0, "realesrgan"),
    ("gray16_up", "realsr", "L", np.uint16, 65536, 22, 14, 10, 0, 10, 3.5, "realesrgan"),
]


def load_realesrganer():
    path = f"{mg.REF}/RealSR/VmambaIR/utils.py"
    tree = ast.parse(open(path).read())
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "RealESRGANer"][0]
    ns = {"cv2": cv2, "math": math, "np": np, "os": os, "queue": queue, "threading": threading, "torch": torch, "F": F,
          "ROOT_DIR": OUT, "load_file_from_url": None}
    exec(compile(ast.Module([cls], []), path, "exec"), ns)
    return ns["RealESRGANer"]


def nets():
    mg.install_stubs()
    mg.load_file("VmambaIR.archs.common", f"{mg.REF}/SRGAN/VmambaIR/archs/common.py")
    realsr = mg.load_file("ref_realsr", f"{mg.REF}/RealSR/VmambaIR/archs/MambaRealSR11_arch.py")
    sisr = mg.load_file("ref_sisr", f"{mg.REF}/SRGAN/VmambaIR/archs/MambaSISR6_arch.py")
    out = {}
    for i, (tag, ctor) in enumerate((("realsr", realsr.MambaRealSR11), ("sisr", sisr.MambaSISR6))):
        torch.manual_seed(40 + i)
        net = ctor(dim=8, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).eval()
        with torch.no_grad():  # randomise the constant-initialised parameters, as make_golden.gen_block does
            for n, p in net.named_parameters():
                p.data = p.data.clone()  # some reference parameters are expanded views, which load_state_dict cannot write
                if n.endswith("body.weight") or n.endswith("Ds") or n.endswith("Dsc"):
                    p.data = p.data.clone() + 0.2 * torch.randn(p.shape)
                p.data = p.data.half().float()  # fp16-representable weights: stored as fp16 without loss
        out[tag] = net
    return out


def image(rng, mode, dtype, hi, h, w):
    shape = (h, w) if mode == "L" else (h, w, 3 if mode == "RGB" else 4)
    img = rng.integers(0, hi, shape).astype(dtype)
    img.flat[0] = hi - 1  # the maximum is hi - 1 whatever the draw: 65535, 256 (a uint16 image read as 8-bit) or 255
    return img


def gen_enhance():
    Ref = load_realesrganer()
    models = nets()
    rec = {}
    with tempfile.TemporaryDirectory() as d:
        paths = {}
        for tag, net in models.items():
            paths[tag] = os.path.join(d, f"{tag}.pth")
            torch.save({"params_ema": net.state_dict()}, paths[tag])
            np.savez_compressed(f"{OUT}/enhance_net_{tag}.npz", **{k: v.numpy().astype(np.float16) for k, v in net.state_dict().items()})
        rng = np.random.default_rng(5)
        for name, tag, mode, dtype, hi, h, w, pre_pad, tile, tile_pad, outscale, alpha in CASES:
            img = image(rng, mode, dtype, hi, h, w)
            up = Ref(4, paths[tag], model=models[tag], tile=tile, tile_pad=tile_pad, pre_pad=pre_pad, half=False,
                     device=torch.device("cpu"))
            with torch.no_grad():
                out, got_mode = up.enhance(img.copy(), outscale=outscale, alpha_upsampler=alpha)
            assert got_mode == mode, (name, got_mode)
            rec[f"{name}/img"] = img
            rec[f"{name}/out"] = out
            rec[f"{name}/params"] = np.array([pre_pad, tile, tile_pad, -1.0 if outscale is None else outscale, float(alpha == "realesrgan")])
            rec[f"{name}/net"] = np.array(tag)
            print(name, img.shape, img.dtype, "->", out.shape, out.dtype)
    np.savez_compressed(f"{OUT}/enhance_ref.npz", **rec)
    print("enhance_ref.npz", os.path.getsize(f"{OUT}/enhance_ref.npz") // 1024, "KiB")


def gen_cv2():
    """standalone OpenCV results: INTER_LANCZOS4 on uint8 / uint16 images, COLOR_BGR2GRAY and INTER_LINEAR on float32"""
    rng = np.random.default_rng(6)
    rec = {}
    lanczos = [  # (h, w, channels, factor)
        (17, 23, 3, 3.5), (32, 24, 4, 0.5), (13, 9, 1, 2.0), (40, 36, 3, 0.37), (8, 8, 3, 1.3), (21, 31, 4, 1.75)]
    for i, (h, w, c, f) in enumerate(lanczos):
        for dt, hi in ((np.uint8, 256), (np.uint16, 65536)):
            img = rng.integers(0, hi, (h, w) if c == 1 else (h, w, c)).astype(dt)
            size = (int(w * f), int(h * f))
            rec[f"lanczos{i}_{dt.__name__}/src"] = img
            rec[f"lanczos{i}_{dt.__name__}/dst"] = cv2.resize(img, size, interpolation=cv2.INTER_LANCZOS4)
    # BGR2GRAY: pixel counts that are multiples of 16 (OpenCV's vector loop covers every pixel)
    g = rng.random((48, 40, 3), dtype=np.float32)
    g[0, :4] = [[0, 0, 0], [1, 1, 1], [0.5, 0.5, 0.5], [1, 0, 1]]
    rec["gray/src"], rec["gray/dst"] = g, cv2.cvtColor(g, cv2.COLOR_BGR2GRAY)
    for i, (h, w, f) in enumerate(((23, 31, 4), (16, 12, 2), (9, 14, 4))):
        a = (rng.integers(0, 256, (h, w)).astype(np.float32) / 255).astype(np.float32)
        rec[f"linear{i}/src"], rec[f"linear{i}/dst"] = a, cv2.resize(a, (w * f, h * f), interpolation=cv2.INTER_LINEAR)
    np.savez_compressed(f"{OUT}/enhance_cv2.npz", **rec)
    print("enhance_cv2.npz", os.path.getsize(f"{OUT}/enhance_cv2.npz") // 1024, "KiB")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_cv2()
    gen_enhance()
