"""Image-level inference: the reference's `RealESRGANer` (RealSR/VmambaIR/utils.py:14-243) on this library's kernels.

`RealESRGANer(scale, model_path, model, ...).enhance(img, outscale, alpha_upsampler) -> (output, img_mode)` keeps the reference's
names, arguments and results.  What the reference does on the host in numpy / cv2 around the network runs on the GPU here, in three
kernels of vmambair_b200/csrc/image_io.cu (a fourth one finds the maximum of a uint16 image):

  * image -> planes: / max_range, BGR -> RGB, gray -> 3 channels, the alpha plane, and the reflect pads (pre_pad, the mod pad of
    scale 1 / 2, then the pad to the networks' multiple of 8) as index arithmetic, written once in the compute dtype;
  * the network through `TiledInference` (tiles batched); in the 'realesrgan' alpha mode the RGB image and its alpha (repeated three
    times) go through the network as one batch of two instead of two passes;
  * planes -> image: post_process's crops, clamp, RGB -> BGR, cv2's BGR2GRAY for gray images and for the network-upscaled alpha, or
    cv2 INTER_LINEAR of the input alpha, x max_range, numpy's round half to even, uint8 / uint16;
  * outscale != scale: cv2 INTER_LANCZOS4 on the uint8 / uint16 result.

Inputs: numpy (H, W) / (H, W, 3) / (H, W, 4) uint8 or uint16 arrays (staged through pinned memory; the result comes back as
numpy), or uint8 / uint16 torch tensors on the host or a GPU (the result is a tensor on the same device).  As in the reference, an
image is 16-bit when its maximum exceeds 256: a uint16 image whose values are all <= 256 is processed and returned as 8-bit.

One extension: the VmambaIR networks need H and W to be multiples of 8, and the reference's helper fails on other sizes.  Here the
padded image is reflect-padded further to the next multiple of 8 and the result cropped, so every size runs.  Sizes that are already
multiples of 8 after pre_pad and the mod pad are unaffected.  Tiles (tile, tile_pad) must themselves be multiples of 8, as for
`TiledInference`.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .checkpoint import load_network
from .tiling import TiledInference

NET_MULTIPLE = 8  # the networks' H, W granularity (three 2x downsamplings)


def max_range_of(img_max: int, dtype) -> int:
    """the reference's 16-bit test (np.max(img) > 256, utils.py:178): 65535 or 255"""
    return 65535 if dtype in (np.uint16, torch.uint16) and img_max > 256 else 255


def mod_scale_of(scale: int):
    """the reference's mod pad (pre_process, utils.py:80-84): scale 2 -> 2, scale 1 -> 4, otherwise none"""
    return {2: 2, 1: 4}.get(scale)


def pad_plan(h: int, w: int, pre_pad: int, scale: int, multiple: int = NET_MULTIPLE):
    """((pre_pad, mod pad, pad to `multiple`) for H, the same for W): the three successive bottom / right reflect pads"""
    mod = mod_scale_of(scale)

    def one(n):
        n1 = n + pre_pad
        m = (mod - n1 % mod) % mod if mod else 0
        return pre_pad, m, (multiple - (n1 + m) % multiple) % multiple
    ph, pw = one(h), one(w)
    # F.pad(..., 'reflect') needs every pad smaller than the size it pads
    for n, pads in ((h, ph), (w, pw)):
        size = n
        for p in pads:
            if p >= size:
                raise ValueError(f"enhance: a {h} x {w} image is too small for pre_pad={pre_pad} (reflect padding needs pad < size)")
            size += p
    return ph, pw


def image_mode(shape) -> str:
    """'L' for (H, W), 'RGB' for (H, W, 3), 'RGBA' for (H, W, 4) (enhance, utils.py:184-196)"""
    if len(shape) == 2:
        return "L"
    if len(shape) == 3 and shape[2] in (3, 4):
        return "RGB" if shape[2] == 3 else "RGBA"
    raise ValueError(f"enhance: expected an (H, W), (H, W, 3) or (H, W, 4) image, got shape {tuple(shape)}")


def output_size(h: int, w: int, scale: int, outscale=None):
    """(height, width) of enhance's result: h*scale x w*scale, or (int(h*outscale), int(w*outscale)) when outscale != scale"""
    if outscale is not None and outscale != float(scale):
        return int(h * outscale), int(w * outscale)
    return h * scale, w * scale


class RealESRGANer:
    """RealESRGANer(scale, model_path, model, tile, tile_pad, pre_pad, half, device, gpu_id) as in the reference.

    model_path: a BasicSR checkpoint ("params_ema", else "params"; strict), or None to keep `model`'s weights.
    half: fp16 compute (the reference's model.half()); dtype: torch.bfloat16 (the library's fast path), torch.float16 or
    torch.float32, overriding `half`.  max_batch: tiles per network call (TiledInference)."""

    def __init__(self, scale, model_path, model=None, tile=0, tile_pad=10, pre_pad=10, half=False, device=None, gpu_id=None,
                 dtype=None, max_batch=8):
        if model is None:
            raise ValueError("RealESRGANer: `model` (a vmambair_b200.archs network) is required")
        if not torch.cuda.is_available():
            raise RuntimeError("RealESRGANer: needs a CUDA device (there is no CPU path)")
        self.scale, self.tile_size, self.tile_pad, self.pre_pad, self.half = int(scale), int(tile), int(tile_pad), int(pre_pad), half
        self.mod_scale = mod_scale_of(self.scale)
        if device is None:
            device = f"cuda:{gpu_id}" if gpu_id else "cuda"
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"RealESRGANer: device must be a CUDA device, got {self.device}")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        if model_path is not None:
            load_network(model, model_path, strict=True, param_key="params_ema")
        model.eval()
        self.dtype = dtype if dtype is not None else (torch.float16 if half else torch.float32)
        if self.dtype not in (torch.float32, torch.bfloat16, torch.float16):
            raise ValueError(f"RealESRGANer: dtype must be float32, bfloat16 or float16, got {self.dtype}")
        self.runner = TiledInference(model, scale=self.scale, multiple=NET_MULTIPLE, tile_size=self.tile_size, tile_pad=self.tile_pad,
                                     dtype=self.dtype, device=self.device, max_batch=max_batch)

    def _to_device(self, img):
        """-> (device tensor, numpy input?)"""
        if isinstance(img, np.ndarray):
            if img.dtype not in (np.uint8, np.uint16):
                raise TypeError(f"enhance: image dtype must be uint8 or uint16, got {img.dtype}")
            staged = torch.empty(img.shape, dtype=torch.uint8 if img.dtype == np.uint8 else torch.uint16, pin_memory=True)
            staged.numpy()[...] = img
            return staged.to(self.device, non_blocking=True), True
        if isinstance(img, torch.Tensor):
            if img.dtype not in (torch.uint8, torch.uint16):
                raise TypeError(f"enhance: image dtype must be uint8 or uint16, got {img.dtype}")
            return (img if img.is_cuda else img.to(self.device, non_blocking=img.is_pinned())), False
        raise TypeError(f"enhance: expected a numpy array or a torch tensor, got {type(img).__name__}")

    @torch.no_grad()
    def enhance(self, img, outscale=None, alpha_upsampler="realesrgan"):
        mode = image_mode(tuple(img.shape))
        h, w = int(img.shape[0]), int(img.shape[1])
        src_device = img.device if isinstance(img, torch.Tensor) else None
        x, as_numpy = self._to_device(img)
        dev = x.device
        with torch.cuda.device(dev):
            if x.dtype == torch.uint16:
                max_range = max_range_of(int(ops.image_max(x).item()), torch.uint16)
            else:
                max_range = 255
            out_dtype = torch.uint16 if max_range == 65535 else torch.uint8
            ph, pw = pad_plan(h, w, self.pre_pad, self.scale)
            net_alpha = mode == "RGBA" and alpha_upsampler == "realesrgan"
            planes = ops.image_to_planes(x, max_range, ph, pw, alpha_plane=net_alpha, dtype=self.dtype)
            y = self.runner(planes)
            alpha_src = x[:, :, 3] if mode == "RGBA" and not net_alpha else None
            channels = {"L": 1, "RGB": 3, "RGBA": 4}[mode]
            out = ops.planes_to_image(y, h * self.scale, w * self.scale, channels, max_range, out_dtype, alpha_src=alpha_src)
            if outscale is not None and outscale != float(self.scale):
                oh, ow = output_size(h, w, self.scale, outscale)
                out = ops.resize_lanczos4(out, ow, oh)
            if as_numpy:
                host = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
                host.copy_(out, non_blocking=True)
                torch.cuda.current_stream(dev).synchronize()
                return host.numpy(), mode
            if src_device is not None and src_device.type == "cpu":
                return out.cpu(), mode
            return out, mode
