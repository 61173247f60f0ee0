"""Image metrics: PSNR and SSIM as the reference scores restored images, on deterministic float64 kernels (csrc/metrics.cu).

`calculate_psnr(img1, img2, crop_border, input_order='HWC', test_y_channel=False)` and `calculate_ssim(...)` are drop-ins for
Deraining/basicsr/metrics/psnr_ssim.py: same names, arguments and results (a Python float).  They take numpy arrays (staged through
pinned memory) or torch tensors on the host or a GPU; a tensor is (C, H, W) or (1, C, H, W), as there.  `calculate_ssim` is the
vendored one: `_ssim_cly` (11 x 11 Gaussian, replicated borders, full-size map) on the Y channel, `_ssim_3d` (the same filter across
the channels too, constants from the image's range) otherwise.  `calculate_ssim(..., ssim='valid')` gives the other convention
instead, the one the SR configs score with (pip basicsr, Deraining/Deraining/utils.py): the mean over the channels of the map where the
window fits (nan for images under 11 pixels).

`psnr_ssim(img, img2, crop_border=0, test_y_channel=True, ssim='valid', quantize=False)` is the batched form the drop-ins run at
B = 1.  It returns (psnr, ssim), two (B,) float64 CUDA tensors, without synchronising the host.  An image is a (B, H, W, C) uint8 /
uint16 / float32 / float64 CUDA tensor in BGR order (C = 1 or 3); with quantize=True a floating-point image is instead a (B, 3, H, W)
float32 / bf16 / fp16 RGB network output, read through the reference's tensor2img (clamp to [0, 1], x 255 rounded half to even, uint8, BGR).
`to_y_channel(img)` is the reference's Y channel (metric_util.to_y_channel) of such a batch, as float32 planes.

Conventions kept from the reference: `max_value` is 1 when image 1's largest value (after the Y conversion) is <= 1, else 255; the Y
channel is the reference's exact float32 / float64 chain; with the Y channel the squared differences are float32, as the reference's,
but they are summed in float64 (the reference sums in float32).  Deviations: a crop that leaves no pixel, mismatched shapes, a bad
input_order, and input_order='CHW' for a tensor (which the reference transposes twice) raise ValueError.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops

SSIM_CONVENTIONS = ("valid", "reference")


# cv2.getGaussianKernel(11, 1.5), the reference's SSIM window (outer product of these with themselves).  OpenCV evaluates it in
# software floating point and adjusts the centre tap so that the taps sum to exactly 1; a plain float64 evaluation of
# exp(-(i - 5)^2 / (2 1.5^2)) / sum differs from it in the last bits, so the values are spelled out (tests pin them to cv2's).
_HALF = ("0x1.0d956b52a1d6ep-10", "0x1.f1fe01ae5a5b5p-8", "0x1.26eb175d83f66p-5", "0x1.bff0fe8e98418p-4", "0x1.b43c3f52b19f3p-3")
TAPS = tuple(float.fromhex(h) for h in _HALF + ("0x1.106560aa892bfp-2",) + _HALF[::-1])


def channel_mix(channels: int, taps=TAPS):
    """the 11-tap filter with replicated ends across `channels` values (_ssim_3d's Conv3d, padding_mode='replicate', on the channel
    axis) as a channels x channels matrix: mix[c][p] = sum of taps[k] over k with clamp(c + k - 5, 0, channels - 1) == p"""
    r = len(taps) // 2
    mix = [[0.0] * channels for _ in range(channels)]
    for c in range(channels):
        for k, w in enumerate(taps):
            mix[c][min(max(c + k - r, 0), channels - 1)] += w
    return mix


class _View:
    """a (B, H, W, C) BGR view of a CUDA tensor's storage: element offset, element strides, tensor2img or not"""

    def __init__(self, t, offset, shape, strides, quantize):
        self.t, self.offset, self.shape, self.strides, self.quantize = t, offset, shape, strides, quantize

    def crop(self, c):
        B, H, W, C = self.shape
        if H - 2 * c <= 0 or W - 2 * c <= 0:
            raise ValueError(f"crop_border={c} leaves no pixel of a {H} x {W} image")
        off = self.offset + c * self.strides[1] + c * self.strides[2]
        return _View(self.t, off, (B, H - 2 * c, W - 2 * c, C), self.strides, self.quantize)

    def src(self):
        return ops.metric_src(self.t, self.offset, self.strides, self.quantize)


def _view(t, quantize, who="psnr_ssim"):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dim() == 4):
        raise ValueError(f"{who}: images must be 4-D CUDA tensors")
    if quantize and t.is_floating_point():
        if t.shape[1] != 3 or t.dtype not in ops.MSRC_Q:
            raise ValueError(f"{who}: quantize=True takes (B, 3, H, W) float32 / bf16 / fp16 RGB, got {tuple(t.shape)} {t.dtype}")
        B, _, H, W = t.shape
        sb, sc, sh, sw = t.stride()
        return _View(t, 2 * sc, (B, H, W, 3), (sb, sh, sw, -sc), True)  # channel 0 (B) is plane 2
    if t.shape[3] not in (1, 3) or t.dtype not in ops.MSRC:
        raise ValueError(f"{who}: images must be (B, H, W, 1 or 3) uint8 / uint16 / float32 / float64, got {tuple(t.shape)} {t.dtype}")
    return _View(t, 0, tuple(t.shape), t.stride(), False)


def _run(v1, v2, test_y_channel, ssim):
    """-> (mse, max of image 1, psnr, ssim), each (B,) float64 on the device; ssim None: PSNR only (ssim None)"""
    if v1.shape != v2.shape:
        raise ValueError(f"image shapes differ: {v1.shape} and {v2.shape}")
    if ssim is not None and ssim not in SSIM_CONVENTIONS:
        raise ValueError(f"ssim must be one of {SSIM_CONVENTIONS}, got {ssim!r}")
    if v1.t.device != v2.t.device:
        raise ValueError(f"images on different devices: {v1.t.device} and {v2.t.device}")
    B, H, W, C = v1.shape
    s1, s2, t = v1.src(), v2.src(), v1.t
    mse, mx, psnr = ops.psnr_sums(t, s1, s2, B, H, W, C, test_y_channel)
    if ssim is None:
        val = None
    elif ssim == "valid":
        val = ops.ssim_mean(t, s1, s2, B, H, W, C, test_y_channel, "valid", TAPS)
    elif test_y_channel:
        val = ops.ssim_mean(t, s1, s2, B, H, W, C, True, "replicate", TAPS)
    else:
        val = ops.ssim_mean(t, s1, s2, B, H, W, C, False, "replicate3d", TAPS, channel_mix(C), mx)
    return mse, mx, psnr, val


def psnr_ssim(img, img2, crop_border=0, test_y_channel=True, ssim="valid", quantize=False):
    """(psnr, ssim) of each image pair of a batch, as two (B,) float64 CUDA tensors; no host synchronisation.

    img, img2: (B, H, W, C) uint8 / uint16 / float32 / float64 BGR (C = 1 or 3); with quantize=True a floating-point image is a
    (B, 3, H, W) float32 / bf16 / fp16 RGB network output, scored after tensor2img (so a uint8 ground truth pairs with a float
    output).  crop_border pixels are dropped on each
    edge.  ssim='valid': the per-channel mean of the valid-region map (the SR configs, pip basicsr); 'reference': the vendored
    calculate_ssim (_ssim_cly on Y, _ssim_3d otherwise).  PSNR is evaluated on the device (float64 log10)."""
    v1, v2 = _view(img, quantize), _view(img2, quantize)
    c = _check_crop(crop_border)
    _, _, psnr, val = _run(v1.crop(c), v2.crop(c), bool(test_y_channel), ssim)
    return psnr, val


def to_y_channel(img, quantize=False):
    """the reference's to_y_channel of a (B, H, W, C) image batch (as psnr_ssim takes them) -> (B, H, W) float32 CUDA tensor, bit for
    bit (x 255 scale, no rounding)"""
    v = _view(img, quantize)
    B, H, W, C = v.shape
    return ops.to_y_channel_planes(v.t, v.src(), B, H, W, C)


def _check_crop(crop_border):
    c = int(crop_border)
    if c < 0 or c != crop_border:
        raise ValueError(f"crop_border must be a non-negative integer, got {crop_border!r}")
    return c


def _device_image(img, input_order, device):
    """a reference-style input (numpy array or tensor) -> (1, H, W, C) view on `device` (reorder_image, tensor squeeze / transpose)"""
    if input_order not in ("HWC", "CHW"):
        raise ValueError(f"Wrong input_order {input_order}. Supported input_orders are 'HWC' and 'CHW'")
    if isinstance(img, torch.Tensor):
        if input_order == "CHW":
            raise ValueError("input_order='CHW' with a tensor: the reference transposes a tensor to HWC itself, then again")
        t = img.detach()
        if t.dim() == 4 and t.shape[0] == 1:
            t = t.squeeze(0)
        if t.dim() != 3:
            raise ValueError(f"a tensor image must be (C, H, W) or (1, C, H, W), got {tuple(img.shape)}")
        t = t.permute(1, 2, 0)
        if t.dtype not in ops.MSRC:  # 16-bit floats are exact in float32, integers in float64 (the reference's astype(float64))
            t = t.float() if t.is_floating_point() else t.double()
        t = t.to(device, non_blocking=t.is_pinned()) if not t.is_cuda else t
    elif isinstance(img, np.ndarray):
        a = img[..., None] if img.ndim == 2 else img
        if a.ndim != 3:
            raise ValueError(f"an array image must be (H, W) or (H, W, C), got shape {img.shape}")
        if input_order == "CHW":
            a = a.transpose(1, 2, 0)
        if a.dtype not in (np.uint8, np.uint16, np.float32, np.float64):
            a = a.astype(np.float64)
        staged = torch.empty(a.shape, dtype=torch.from_numpy(a[:0, :0, :0]).dtype, pin_memory=True)
        staged.numpy()[...] = a
        t = staged.to(device, non_blocking=True)
    else:
        raise TypeError(f"expected a numpy array or a torch tensor, got {type(img).__name__}")
    if t.shape[2] not in (1, 3):
        raise ValueError(f"images must have 1 or 3 channels, got {t.shape[2]}")
    return _view(t.unsqueeze(0), False)


def _pair(img1, img2, crop_border, input_order):
    if tuple(img1.shape) != tuple(img2.shape):
        raise ValueError(f"Image shapes are different: {tuple(img1.shape)}, {tuple(img2.shape)}.")
    c = _check_crop(crop_border)
    devs = [x.device for x in (img1, img2) if isinstance(x, torch.Tensor) and x.is_cuda]
    dev = devs[0] if devs else torch.device("cuda", torch.cuda.current_device())
    return _device_image(img1, input_order, dev).crop(c), _device_image(img2, input_order, dev).crop(c)


def calculate_psnr(img1, img2, crop_border, input_order="HWC", test_y_channel=False):
    """PSNR (psnr_ssim.py:9-63) as a Python float; inf for identical images.  The MSE is summed on the device in float64; the last
    step, 20 log10(max_value / sqrt(mse)), runs in numpy as the reference writes it, so integer images give its float bit for bit."""
    v1, v2 = _pair(img1, img2, crop_border, input_order)
    mse, mx, _, _ = _run(v1, v2, bool(test_y_channel), None)
    mse, mx = torch.stack([mse[0], mx[0]]).cpu().tolist()
    mse = np.float64(mse)
    if mse == 0:
        return float("inf")
    max_value = 1. if mx <= 1 else 255.
    return float(20. * np.log10(max_value / np.sqrt(mse)))


def calculate_ssim(img1, img2, crop_border, input_order="HWC", test_y_channel=False, ssim="reference"):
    """SSIM (psnr_ssim.py:225-303) as a Python float.  ssim='reference' (default): the vendored calculate_ssim; 'valid': the
    per-channel valid-region mean of pip basicsr / Deraining/Deraining/utils.py (nan when the cropped image is under 11 pixels)."""
    v1, v2 = _pair(img1, img2, crop_border, input_order)
    return float(_run(v1, v2, bool(test_y_channel), ssim)[3][0].item())
