"""Torch restatement of basicsr's Real-ESRGAN degradation operators and of MambaRealSR.feed_data's synthesis
(RealSR/VmambaIR/models/MambaRealSR_model.py:145-260), written from their documented behaviour.  Test infrastructure only: the tests
run it in float64 and compare vmambair_b200.degradations with it; tools/degrade_bench.py runs it in float32 as the stand-in for
basicsr's chains of small torch ops.

Every operator computes in its input's dtype.  The random tensors are arguments (or, in the `add_*` and `feed_data` helpers, drawn
from torch's default generator in float32 in the library's documented order), so a test can feed both sides the same draws.  What
basicsr evaluates on float32 tensors before any image arithmetic -- the JPEG quality factor, the noise sigma / scale, the Poisson levels
and rates -- is evaluated in float32 here too, exactly as torch does it."""
import random

import numpy as np
import torch
from torch.nn import functional as F

RESIZE_MODES = ("area", "bilinear", "bicubic")

# ITU-T T.81 K.1 as printed, and the chroma top-left 4 x 4; basicsr applies both transposed
Q_Y = torch.tensor([[16, 11, 10, 16, 24, 40, 51, 61], [12, 12, 14, 19, 26, 58, 60, 55], [14, 13, 16, 24, 40, 57, 69, 56],
                    [14, 17, 22, 29, 51, 87, 80, 62], [18, 22, 37, 56, 68, 109, 103, 77], [24, 35, 55, 64, 81, 104, 113, 92],
                    [49, 64, 78, 87, 103, 121, 120, 101], [72, 92, 95, 98, 112, 100, 103, 99]], dtype=torch.float64)
Q_C = torch.full((8, 8), 99.0, dtype=torch.float64)
Q_C[:4, :4] = torch.tensor([[17, 18, 24, 47], [18, 21, 26, 66], [24, 26, 56, 99], [47, 66, 99, 99]], dtype=torch.float64)
RGB2YCC = torch.tensor([[0.299, 0.587, 0.114], [-0.168736, -0.331264, 0.5], [0.5, -0.418688, -0.081312]], dtype=torch.float64)
YCC2RGB = torch.tensor([[1.0, 0.0, 1.402], [1.0, -0.344136, -0.714136], [1.0, 1.772, 0.0]], dtype=torch.float64)


def dct_matrix(dtype=torch.float64):
    """C[x][u] = alpha(u) / 2 cos((2x + 1) u pi / 16): the orthonormal DCT-II of a block P is C^T P C (cv2.dct), its inverse C D C^T"""
    x = torch.arange(8, dtype=torch.float64)
    c = torch.cos((2 * x[:, None] + 1) * x[None, :] * torch.pi / 16) * 0.5
    c[:, 0] /= 2 ** 0.5
    return c.to(dtype)


def dct8(p):
    """orthonormal 8 x 8 DCT-II of the last two dims (x the row): D[u][v] = 1/4 a(u) a(v) sum (p[x][y]) cos((2x+1)u pi/16) cos((2y+1)v pi/16)"""
    C = dct_matrix(p.dtype).to(p.device)
    return torch.einsum("xu,...xy,yv->...uv", C, p, C)


def idct8(d):
    """the exact inverse of dct8"""
    C = dct_matrix(d.dtype).to(d.device)
    return torch.einsum("xu,...uv,yv->...xy", C, d, C)


def filter2d(img, kernel):
    """basicsr filter2D: reflect pads of k // 2, then per-plane cross-correlation with (1, k, k) or (b, k, k) kernels"""
    k = kernel.shape[-1]
    b, c, h, w = img.shape
    x = F.pad(img, (k // 2,) * 4, mode="reflect")
    kern = kernel.to(img.dtype)
    if kernel.shape[0] == 1:
        return F.conv2d(x.reshape(b * c, 1, *x.shape[-2:]), kern.view(1, 1, k, k)).view(b, c, h, w)
    kern = kern.view(b, 1, k, k).repeat(1, c, 1, 1).view(b * c, 1, k, k)
    return F.conv2d(x.reshape(1, b * c, *x.shape[-2:]), kern, groups=b * c).view(b, c, h, w)


def usm_kernel(radius=51, sigma=0):
    """USMSharp's kernel: np.outer of cv2.getGaussianKernel(radius, sigma) with itself, float64 (1, k, k)"""
    import cv2
    g = cv2.getGaussianKernel(radius, sigma)
    return torch.from_numpy(np.dot(g, g.transpose())).unsqueeze(0)


def usm(img, kernel, weight=0.5, threshold=10):
    """USMSharp.forward; also returns |residual| 255 (tests keep away from the threshold)"""
    blur = filter2d(img, kernel)
    residual = img - blur
    mag = residual.abs() * 255
    soft = filter2d((mag > threshold).to(img.dtype), kernel)
    sharp = torch.clip(img + weight * residual, 0, 1)
    return soft * sharp + (1 - soft) * img, mag


def quality_to_factor(quality):
    """basicsr's per-element quality -> factor on a float32 tensor: (q < 50 ? 5000 / q : 200 - q 2) / 100"""
    q = quality.to(torch.float32)
    return torch.where(q < 50, 5000.0 / q, 200.0 - q * 2) / 100.0


def _blocks(p):
    """(b, H, W) -> (b, H / 8, W / 8, 8, 8)"""
    b, h, w = p.shape
    return p.view(b, h // 8, 8, w // 8, 8).permute(0, 1, 3, 2, 4)


def _merge(blk):
    b, nh, nw = blk.shape[:3]
    return blk.permute(0, 1, 3, 2, 4).reshape(b, nh * 8, nw * 8)


def jpeg(x, factor, clamp_in=False, return_ratios=False):
    """DiffJPEG(differentiable=False)(x, quality) with factor = quality_to_factor(quality), (b,) or a number; a zero step keeps the
    coefficient.  return_ratios: also the pre-rounding D / step of the luma blocks (b, H16 / 8, W16 / 8, 8, 8) and of the chroma
    blocks (b, 2, H16 / 16, W16 / 16, 8, 8)"""
    dt = x.dtype
    if clamp_in:
        x = torch.clamp(x, 0, 1)
    b, _, h, w = x.shape
    x = F.pad(x, (0, (16 - w % 16) % 16, 0, (16 - h % 16) % 16))
    ycc = torch.einsum("bchw,dc->bdhw", x * 255, RGB2YCC.to(x)) + torch.tensor([0.0, 128.0, 128.0]).to(x).view(1, 3, 1, 1)
    chroma = F.avg_pool2d(ycc[:, 1:], 2)
    f = torch.as_tensor(factor, dtype=torch.float32, device=x.device).to(dt).reshape(-1, 1, 1, 1, 1)

    def code(p, table):
        d = dct8(_blocks(p - 128))
        step = table.T.to(dt).to(x.device) * f
        ratio = d / step
        dq = torch.where(step == 0, d, torch.round(ratio) * step)
        return _merge(idct8(dq)) + 128, ratio

    y, ry = code(ycc[:, 0], Q_Y)
    cb, rcb = code(chroma[:, 0], Q_C)
    cr, rcr = code(chroma[:, 1], Q_C)
    up = lambda t: t.repeat_interleave(2, 1).repeat_interleave(2, 2)
    ycc = torch.stack([y, up(cb) - 128, up(cr) - 128], 1)
    rgb = torch.einsum("bchw,dc->bdhw", ycc, YCC2RGB.to(ycc))
    out = (torch.clamp(rgb, 0, 255) / 255)[:, :, :h, :w]
    return (out, ry, torch.stack([rcb, rcr], 1)) if return_ratios else out


def quant255(x):
    return torch.clamp((x * 255.0).round(), 0, 255) / 255.0


def gray(img):
    """torchvision rgb_to_grayscale (separate roundings in img's dtype), (b, 1, H, W)"""
    r, g, b = img.unbind(1)
    return (0.2989 * r + 0.587 * g + 0.114 * b).unsqueeze(1)


def poisson_levels(img32):
    """generate_poisson_noise_pt's levels of a float32 batch, as basicsr computes them: (rates, rates_gray, vals, vals_gray), float32"""
    out = []
    for q in (quant255(img32), quant255(gray(img32))):
        counts = [len(torch.unique(q[i])) for i in range(q.shape[0])]
        vals = q.new_tensor([2 ** np.ceil(np.log2(n)) for n in counts]).view(-1, 1, 1, 1)
        out.append((q * vals, vals.view(-1)))
    (rates, vals), (rates_g, vals_g) = out
    return rates, rates_g, vals, vals_g


def _finish(out, clip, rounds):
    if clip and rounds:
        return quant255(out)
    if clip:
        return torch.clamp(out, 0, 1)
    if rounds:
        return (out * 255.0).round() / 255.0
    return out


def _param(u, rng):
    """rand(b) (hi - lo) + lo and its float32 roundings, as basicsr draws sigma / scale"""
    return u.float() * float(rng[1] - rng[0]) + float(rng[0])


def gaussian_noise(img, u_sigma, u_gray, noise_gray, noise, sigma_range, gray_prob, clip=True, rounds=False):
    """random_add_gaussian_noise_pt from its draws; arithmetic in img's dtype"""
    dt = img.dtype
    sigma = _param(u_sigma, sigma_range).to(dt).view(-1, 1, 1, 1)
    g = (u_gray.float() < gray_prob).to(dt).view(-1, 1, 1, 1)
    n = noise.to(dt) * sigma / 255.0
    ng = noise_gray.to(dt) * sigma / 255.0
    return _finish(img + (n * (1 - g) + ng * g), clip, rounds)


def poisson_noise(img, u_scale, u_gray, p_gray, p, vals, vals_gray, scale_range, gray_prob, clip=True, rounds=False):
    """random_add_poisson_noise_pt from its draws (p, p_gray: torch.poisson of poisson_levels' rates); arithmetic in img's dtype"""
    dt = img.dtype
    scale = _param(u_scale, scale_range).to(dt).view(-1, 1, 1, 1)
    g = (u_gray.float() < gray_prob).to(dt).view(-1, 1, 1, 1)
    # the levels are basicsr's float32 ones (poisson_levels), whatever dtype the rest runs in
    noise = p.to(dt) / vals.to(dt).view(-1, 1, 1, 1) - quant255(img.float()).to(dt)
    noise_g = p_gray.to(dt) / vals_gray.to(dt).view(-1, 1, 1, 1) - quant255(gray(img.float())).to(dt)
    return _finish(img + (noise * (1 - g) + noise_g * g) * scale, clip, rounds)


def add_gaussian_noise(img, sigma_range, gray_prob, clip=True, rounds=False):
    b, c, h, w = img.shape
    kw = dict(dtype=torch.float32, device=img.device)
    u_sigma, u_gray = torch.rand(b, **kw), torch.rand(b, **kw)
    noise_gray = torch.randn(h, w, **kw)
    noise = torch.randn(b, c, h, w, **kw)
    return gaussian_noise(img, u_sigma, u_gray, noise_gray, noise, sigma_range, gray_prob, clip, rounds)


def add_poisson_noise(img, scale_range, gray_prob, clip=True, rounds=False):
    b = img.shape[0]
    kw = dict(dtype=torch.float32, device=img.device)
    u_scale, u_gray = torch.rand(b, **kw), torch.rand(b, **kw)
    rates, rates_g, vals, vals_g = poisson_levels(img.float())
    p_gray = torch.poisson(rates_g)
    p = torch.poisson(rates)
    return poisson_noise(img, u_scale, u_gray, p_gray, p, vals, vals_g, scale_range, gray_prob, clip, rounds)


def _resize_decision(prob, rng):
    updown = random.choices(["up", "down", "keep"], prob)[0]
    if updown == "up":
        return updown, np.random.uniform(1, rng[1])
    if updown == "down":
        return updown, np.random.uniform(rng[0], 1)
    return updown, 1


def feed_data(gt, kernel1, kernel2, sinc_kernel, opt, scale, dtype=torch.float64):
    """MambaRealSR.feed_data's synthesis, up to the final rounding, in `dtype` -> (lq, gt, log of host decisions); consumes random,
    numpy.random and torch's generator as the library does"""
    log = []
    gt = gt.to(dtype)
    if opt["gt_usm"] is True:
        gt = usm(gt, usm_kernel())[0]
    b, _, ori_h, ori_w = gt.shape

    def noise(out, stage):
        sfx = "" if stage == 1 else "2"
        if np.random.uniform() < opt["gaussian_noise_prob" + sfx]:
            log.append((f"noise{stage}", "gaussian"))
            return add_gaussian_noise(out, opt["noise_range" + sfx], opt["gray_noise_prob" + sfx])
        log.append((f"noise{stage}", "poisson"))
        return add_poisson_noise(out, opt["poisson_scale_range" + sfx], opt["gray_noise_prob" + sfx])

    def quality(rng):
        return quality_to_factor(torch.zeros(b, dtype=torch.float32, device=gt.device).uniform_(*rng))

    out = filter2d(gt, kernel1)
    updown, s = _resize_decision(opt["resize_prob"], opt["resize_range"])
    mode = random.choice(RESIZE_MODES)
    log.append(("resize1", updown, float(s), mode))
    out = F.interpolate(out, scale_factor=s, mode=mode)
    out = noise(out, 1)
    out = jpeg(out, quality(opt["jpeg_range"]), clamp_in=True)
    blur2 = bool(np.random.uniform() < opt["second_blur_prob"])
    log.append(("blur2", blur2))
    if blur2:
        out = filter2d(out, kernel2)
    updown, s = _resize_decision(opt["resize_prob2"], opt["resize_range2"])
    mode = random.choice(RESIZE_MODES)
    log.append(("resize2", updown, float(s), mode))
    out = F.interpolate(out, size=(int(ori_h / scale * s), int(ori_w / scale * s)), mode=mode)
    out = noise(out, 2)
    if np.random.uniform() < 0.5:
        mode = random.choice(RESIZE_MODES)
        log.append(("final", "sinc_first", mode))
        out = F.interpolate(out, size=(ori_h // scale, ori_w // scale), mode=mode)
        out = filter2d(out, sinc_kernel)
        out = jpeg(out, quality(opt["jpeg_range2"]), clamp_in=True)
    else:
        out = jpeg(out, quality(opt["jpeg_range2"]), clamp_in=True)
        mode = random.choice(RESIZE_MODES)
        log.append(("final", "jpeg_first", mode))
        out = F.interpolate(out, size=(ori_h // scale, ori_w // scale), mode=mode)
        out = filter2d(out, sinc_kernel)
    return quant255(out), gt, log
