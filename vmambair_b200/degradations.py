"""Real-ESRNet training-pair synthesis on the device: the second-order degradation of `MambaRealSR.feed_data`
(RealSR/VmambaIR/models/MambaRealSR_model.py:145-260) and the basicsr operators it is built from, on the kernels of csrc/degrade.cu.

Drop-ins, with basicsr's names, signatures and results (float32 NCHW CUDA tensors; any other dtype raises TypeError):
  * `filter2D(img, kernel)`: per-plane k x k cross-correlation with reflect pads, one (1, k, k) kernel or one per image (b, k, k);
  * `USMSharp(radius=50, sigma=0)`, an nn.Module with `forward(img, weight=0.5, threshold=10)`;
  * `DiffJPEG(differentiable=False)`, `forward(x, quality)` with a number or a (b,) tensor of qualities;
  * `random_add_gaussian_noise_pt(img, sigma_range, gray_prob, clip, rounds)` and `random_add_poisson_noise_pt(img, scale_range,
    gray_prob, clip, rounds)`.
`RealESRNetDegradation(opt, scale)(gt, kernel1, kernel2, sinc_kernel) -> (lq, gt)` is feed_data's training branch, with the same
option keys.  `degrade()` is its synthesis alone (no crop, no pair pool) and never synchronises with the host.

Random draws.  Host decisions consume Python `random` and `numpy.random` in the reference's order, so a seeded run takes the reference's
branches; `RealESRNetDegradation.log` lists them.  Device draws stay on torch's default generator, all float32 on the input's device,
in this order:
  Gaussian noise: rand(b) sigma, rand(b) gray, randn(H, W) gray noise, randn(b, c, H, W);
  Poisson noise:  rand(b) scale, rand(b) gray, poisson(gray rates) (b, 1, H, W), poisson(rates) (b, c, H, W);
  JPEG quality in the pipeline: new_zeros(b).uniform_(lo, hi).
Deviations from basicsr: the gray noise is drawn whether or not an image of the batch is gray (deciding would read the device); DiffJPEG
leaves the caller's quality tensor as it is (basicsr overwrites it with the factor); quality 100 (a zero quantisation step) keeps the
coefficients instead of producing NaN.
"""
from __future__ import annotations

import random

import numpy as np
import torch
from torch.nn import functional as F

from . import ops

MAX_KERNEL = 51
RESIZE_MODES = ("area", "bilinear", "bicubic")


def _check_img(img, who, channels=None):
    if not isinstance(img, torch.Tensor) or img.dtype != torch.float32:
        raise TypeError(f"{who}: expects a float32 tensor, got {getattr(img, 'dtype', type(img))}")
    if img.dim() != 4 or not img.is_cuda or (channels is not None and img.shape[1] != channels):
        raise ValueError(f"{who}: expects a (b, {channels or 'c'}, H, W) CUDA tensor, got {tuple(img.shape)} on {img.device}")
    return img.contiguous()


def _check_k(k, H, W, who):
    if k % 2 != 1 or k > MAX_KERNEL:
        raise ValueError(f"{who}: kernel size {k} must be odd and at most {MAX_KERNEL}")
    if H <= k // 2 or W <= k // 2:
        raise ValueError(f"{who}: a {H} x {W} image is too small for the reflect pad {k // 2} of a {k} x {k} kernel")


def _filter2d(img, kernel, quantize_out=False):
    img = _check_img(img, "filter2D")
    if not isinstance(kernel, torch.Tensor) or kernel.dtype != torch.float32:
        raise TypeError(f"filter2D: expects a float32 kernel, got {getattr(kernel, 'dtype', type(kernel))}")
    b, _, H, W = img.shape
    if kernel.dim() != 3 or kernel.shape[0] not in (1, b) or kernel.shape[1] != kernel.shape[2]:
        raise ValueError(f"filter2D: kernel must be (1, k, k) or ({b}, k, k), got {tuple(kernel.shape)}")
    _check_k(kernel.shape[-1], H, W, "filter2D")
    kernel = kernel.to(img.device).contiguous()
    return ops.filter2d(img, kernel, per_image=kernel.shape[0] != 1, quantize_out=quantize_out)


def filter2D(img, kernel):
    """basicsr filter2D: each plane of (b, c, H, W) img cross-correlated with kernel (1, k, k) or (b, k, k), reflect pads of k // 2"""
    return _filter2d(img, kernel)


def gaussian_kernel_1d(ksize: int, sigma: float = 0.0) -> np.ndarray:
    """cv2.getGaussianKernel(ksize, sigma) as float64 (ksize, 1): OpenCV's fixed taps for ksize <= 9 and sigma <= 0, otherwise
    exp(-x^2 / (2 sigma^2)) scaled by 1 / sum, with sigma = 0.3 ((ksize - 1) / 2 - 1) + 0.8 when sigma <= 0"""
    fixed = {1: [1.0], 3: [0.25, 0.5, 0.25], 5: [0.0625, 0.25, 0.375, 0.25, 0.0625],
             7: [0.03125, 0.109375, 0.21875, 0.28125, 0.21875, 0.109375, 0.03125],
             9: [4 / 256, 13 / 256, 30 / 256, 51 / 256, 60 / 256, 51 / 256, 30 / 256, 13 / 256, 4 / 256]}
    if ksize in fixed and sigma <= 0:
        return np.array(fixed[ksize], dtype=np.float64).reshape(-1, 1)
    s = sigma if sigma > 0 else ((ksize - 1) * 0.5 - 1) * 0.3 + 0.8
    x = np.arange(ksize, dtype=np.float64) - (ksize - 1) * 0.5
    t = np.exp((-0.5 / (s * s)) * x * x)
    return (t * (1.0 / t.sum())).reshape(-1, 1)


class USMSharp(torch.nn.Module):
    """basicsr USMSharp: unsharp masking with a (radius | 1) x (radius | 1) Gaussian; `kernel` is basicsr's (1, k, k) float32 buffer,
    the device runs its separable factors (two launches)"""

    def __init__(self, radius=50, sigma=0):
        super().__init__()
        if radius % 2 == 0:
            radius += 1
        if radius > MAX_KERNEL:
            raise ValueError(f"USMSharp: radius {radius} above {MAX_KERNEL}")
        self.radius = radius
        g = gaussian_kernel_1d(radius, sigma)
        self.taps = [float(v) for v in g.astype(np.float32).ravel()]
        self.register_buffer("kernel", torch.FloatTensor(np.dot(g, g.transpose())).unsqueeze_(0))

    def forward(self, img, weight=0.5, threshold=10):
        img = _check_img(img, "USMSharp")
        _check_k(self.radius, img.shape[2], img.shape[3], "USMSharp")
        return ops.usm_sharp(img, self.taps, weight, threshold)


def quality_to_factor(quality: float) -> float:
    """basicsr's JPEG quality -> quantisation-table factor of a Python number (the device does the same per image in float32)"""
    return (5000.0 / quality if quality < 50 else 200.0 - quality * 2) / 100.0


def _jpeg(x, quality, clamp_in=False, quantize_out=False):
    x = _check_img(x, "DiffJPEG", channels=3)
    if isinstance(quality, (int, float)):
        return ops.jpeg(x, factor=quality_to_factor(quality), clamp_in=clamp_in, quantize_out=quantize_out)
    q = quality.to(device=x.device, dtype=torch.float32).reshape(-1).contiguous()
    if q.numel() != x.shape[0]:
        raise ValueError(f"DiffJPEG: {q.numel()} qualities for {x.shape[0]} images")
    return ops.jpeg(x, quality=q, clamp_in=clamp_in, quantize_out=quantize_out)


class DiffJPEG(torch.nn.Module):
    """basicsr DiffJPEG(differentiable=False): JPEG compression and decompression of (b, 3, H, W) RGB in [0, 1], one kernel, with a
    quality per image ((b,) tensor, on the device without a host read) or one number for all"""

    def __init__(self, differentiable=False):
        super().__init__()
        if differentiable:
            raise NotImplementedError("DiffJPEG: only differentiable=False (rounding) is implemented")

    def forward(self, x, quality):
        return _jpeg(x, quality)


def random_add_gaussian_noise_pt(img, sigma_range=(0, 1.0), gray_prob=0, clip=True, rounds=False):
    """basicsr random_add_gaussian_noise_pt; draws: rand(b) sigma, rand(b) gray, randn(H, W), randn(b, c, H, W)"""
    img = _check_img(img, "random_add_gaussian_noise_pt")
    b, c, h, w = img.shape
    kw = dict(dtype=torch.float32, device=img.device)
    u_sigma, u_gray = torch.rand(b, **kw), torch.rand(b, **kw)
    noise_gray = torch.randn(h, w, **kw)
    noise = torch.randn(b, c, h, w, **kw)
    return ops.noise_apply(img, ops.NOISE_GAUSSIAN, noise, noise_gray, u_sigma, u_gray, sigma_range, gray_prob, clip, rounds)


def random_add_poisson_noise_pt(img, scale_range=(0, 1.0), gray_prob=0, clip=True, rounds=False):
    """basicsr random_add_poisson_noise_pt of 3-channel images; draws: rand(b) scale, rand(b) gray, poisson(gray rates),
    poisson(rates)"""
    img = _check_img(img, "random_add_poisson_noise_pt", channels=3)
    b = img.shape[0]
    kw = dict(dtype=torch.float32, device=img.device)
    u_scale, u_gray = torch.rand(b, **kw), torch.rand(b, **kw)
    rates, rates_gray, vals, vals_gray = ops.noise_levels(img)
    p_gray = torch.poisson(rates_gray)
    p = torch.poisson(rates)
    return ops.noise_apply(img, ops.NOISE_POISSON, p, p_gray, u_scale, u_gray, scale_range, gray_prob, clip, rounds,
                           vals=vals, vals_gray=vals_gray)


class RealESRNetDegradation:
    """MambaRealSR.feed_data's training branch: `(lq, gt) = deg(gt, kernel1, kernel2, sinc_kernel)`.

    opt holds the recipe's keys (gt_usm, resize_prob, resize_range, gaussian_noise_prob, noise_range, poisson_scale_range,
    gray_noise_prob, jpeg_range, second_blur_prob, resize_prob2, resize_range2, gaussian_noise_prob2, noise_range2,
    poisson_scale_range2, gray_noise_prob2, jpeg_range2, gt_size, queue_size); scale is the SR scale.  The final
    clamp(round(255 x)) / 255 runs in the last kernel of the chain.  `log` lists the host decisions of the last call."""

    def __init__(self, opt, scale):
        self.opt, self.scale = opt, scale
        self.queue_size = opt.get("queue_size", 180)
        self.usm_sharpener = USMSharp()
        self.log = []

    def _resize_decision(self, prob, rng):
        updown = random.choices(["up", "down", "keep"], prob)[0]
        if updown == "up":
            return updown, np.random.uniform(1, rng[1])
        if updown == "down":
            return updown, np.random.uniform(rng[0], 1)
        return updown, 1

    def _noise(self, out, stage):
        o, sfx = self.opt, "" if stage == 1 else "2"
        if np.random.uniform() < o["gaussian_noise_prob" + sfx]:
            self.log.append((f"noise{stage}", "gaussian"))
            return random_add_gaussian_noise_pt(out, sigma_range=o["noise_range" + sfx], clip=True, rounds=False,
                                                gray_prob=o["gray_noise_prob" + sfx])
        self.log.append((f"noise{stage}", "poisson"))
        return random_add_poisson_noise_pt(out, scale_range=o["poisson_scale_range" + sfx], gray_prob=o["gray_noise_prob" + sfx],
                                           clip=True, rounds=False)

    @torch.no_grad()
    def degrade(self, gt, kernel1, kernel2, sinc_kernel):
        """-> (lq, gt): the LQ of the whole GT batch, rounded to 8-bit levels, and the GT (USM-sharpened when opt['gt_usm'])"""
        o, s = self.opt, self.scale
        self.log = []
        gt = _check_img(gt, "RealESRNetDegradation", channels=3)
        if o["gt_usm"] is True:
            gt = self.usm_sharpener(gt)
        b, _, ori_h, ori_w = gt.shape
        # first degradation: blur, resize, noise, JPEG
        out = filter2D(gt, kernel1)
        updown, scale = self._resize_decision(o["resize_prob"], o["resize_range"])
        mode = random.choice(RESIZE_MODES)
        self.log.append(("resize1", updown, float(scale), mode))
        out = F.interpolate(out, scale_factor=scale, mode=mode)
        out = self._noise(out, 1)
        jpeg_p = out.new_zeros(b).uniform_(*o["jpeg_range"])
        out = _jpeg(out, jpeg_p, clamp_in=True)
        # second degradation
        blur2 = bool(np.random.uniform() < o["second_blur_prob"])
        self.log.append(("blur2", blur2))
        if blur2:
            out = filter2D(out, kernel2)
        updown, scale = self._resize_decision(o["resize_prob2"], o["resize_range2"])
        mode = random.choice(RESIZE_MODES)
        self.log.append(("resize2", updown, float(scale), mode))
        out = F.interpolate(out, size=(int(ori_h / s * scale), int(ori_w / s * scale)), mode=mode)
        out = self._noise(out, 2)
        # [resize back + sinc] and JPEG, in a random order; the last kernel rounds to 8-bit levels
        if np.random.uniform() < 0.5:
            mode = random.choice(RESIZE_MODES)
            self.log.append(("final", "sinc_first", mode))
            out = F.interpolate(out, size=(ori_h // s, ori_w // s), mode=mode)
            out = filter2D(out, sinc_kernel)
            jpeg_p = out.new_zeros(b).uniform_(*o["jpeg_range2"])
            out = _jpeg(out, jpeg_p, clamp_in=True, quantize_out=True)
        else:
            jpeg_p = out.new_zeros(b).uniform_(*o["jpeg_range2"])
            out = _jpeg(out, jpeg_p, clamp_in=True)
            mode = random.choice(RESIZE_MODES)
            self.log.append(("final", "jpeg_first", mode))
            out = F.interpolate(out, size=(ori_h // s, ori_w // s), mode=mode)
            out = _filter2d(out, sinc_kernel, quantize_out=True)
        return out, gt

    def paired_random_crop(self, gt, lq):
        """basicsr paired_random_crop of a batch: one random.randint top, then left, on the LQ grid"""
        gt_size, s = self.opt["gt_size"], self.scale
        lq_size = gt_size // s
        h_lq, w_lq = lq.shape[-2:]
        if gt.shape[-2] != h_lq * s or gt.shape[-1] != w_lq * s:
            raise ValueError(f"GT {tuple(gt.shape[-2:])} is not {s}x the LQ {(h_lq, w_lq)}")
        if h_lq < lq_size or w_lq < lq_size:
            raise ValueError(f"LQ {(h_lq, w_lq)} is smaller than the patch {lq_size}")
        top = random.randint(0, h_lq - lq_size)
        left = random.randint(0, w_lq - lq_size)
        self.log.append(("crop", top, left))
        lq = lq[:, :, top:top + lq_size, left:left + lq_size]
        gt = gt[:, :, int(top * s):int(top * s) + gt_size, int(left * s):int(left * s) + gt_size]
        return gt, lq

    @torch.no_grad()
    def _dequeue_and_enqueue(self, lq, gt):
        """the reference's training-pair pool of queue_size pairs (CPU torch.randperm shuffle once full)"""
        b, c, h, w = lq.shape
        if not hasattr(self, "queue_lr"):
            assert self.queue_size % b == 0, f"queue size {self.queue_size} should be divisible by batch size {b}"
            self.queue_lr = torch.zeros(self.queue_size, c, h, w, device=lq.device)
            self.queue_gt = torch.zeros(self.queue_size, *gt.shape[1:], device=gt.device)
            self.queue_ptr = 0
        if self.queue_ptr == self.queue_size:
            idx = torch.randperm(self.queue_size)
            self.queue_lr = self.queue_lr[idx]
            self.queue_gt = self.queue_gt[idx]
            lq_dequeue = self.queue_lr[0:b].clone()
            gt_dequeue = self.queue_gt[0:b].clone()
            self.queue_lr[0:b] = lq.clone()
            self.queue_gt[0:b] = gt.clone()
            return lq_dequeue, gt_dequeue
        self.queue_lr[self.queue_ptr:self.queue_ptr + b] = lq.clone()
        self.queue_gt[self.queue_ptr:self.queue_ptr + b] = gt.clone()
        self.queue_ptr += b
        return lq, gt

    def __call__(self, gt, kernel1, kernel2, sinc_kernel):
        lq, gt = self.degrade(gt, kernel1, kernel2, sinc_kernel)
        gt, lq = self.paired_random_crop(gt, lq)
        lq, gt = self._dequeue_and_enqueue(lq, gt)
        return lq.contiguous(), gt
