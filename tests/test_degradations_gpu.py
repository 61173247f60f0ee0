"""The degradation kernels (csrc/degrade.cu, vmambair_b200.degradations) against the float64 restatement oracle/degradations_ref.py, on
the recipe's shapes (batch 9, 600 x 600 GT, 150 x 150 LQ) and on ragged ones; then the whole Real-ESRNet synthesis against the
restatement of feed_data, with the same host and device draws."""
import random

import numpy as np
import pytest
import torch

from oracle import degradations_ref as R
from vmambair_b200 import degradations as D
from vmambair_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"

OPT = dict(gt_usm=False, resize_prob=[0.2, 0.7, 0.1], resize_range=[0.15, 1.5], gaussian_noise_prob=0.5, noise_range=[1, 30],
           poisson_scale_range=[0.05, 3], gray_noise_prob=0.4, jpeg_range=[30, 95], second_blur_prob=0.8,
           resize_prob2=[0.3, 0.4, 0.3], resize_range2=[0.3, 1.2], gaussian_noise_prob2=0.5, noise_range2=[1, 25],
           poisson_scale_range2=[0.05, 2.5], gray_noise_prob2=0.4, jpeg_range2=[30, 95], gt_size=256, queue_size=180)


def _img(b, H, W, seed, c=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand(b, c, H, W, generator=g, device=DEV)


def _kernels(n, k, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    kern = torch.rand(n, k, k, generator=g, device=DEV) + 0.05
    return kern / kern.sum((1, 2), keepdim=True)


@pytest.mark.parametrize("b,H,W,k", [(9, 600, 600, 21), (9, 150, 150, 21), (2, 150, 150, 7), (2, 150, 150, 51), (2, 37, 53, 7),
                                     (3, 4, 45, 7), (2, 26, 70, 51), (1, 11, 11, 21)])
@pytest.mark.parametrize("per_image", [False, True])
@pytest.mark.parametrize("quantize", [False, True])
def test_filter2d(b, H, W, k, per_image, quantize):
    img = _img(b, H, W, H * W + k)
    kern = _kernels(b if per_image else 1, k, k)
    got = D._filter2d(img, kern, quantize_out=quantize)
    ref = R.filter2d(img.double(), kern.double())
    if quantize:  # the float32 result, rounded to 8-bit levels in the same kernel
        assert torch.equal(got, R.quant255(D.filter2D(img, kern)))
    else:
        assert (got.double() - ref).abs().max().item() <= 2e-5


@pytest.mark.parametrize("b,H,W", [(2, 96, 128), (3, 26, 41), (1, 150, 150)])
def test_usm_sharp(b, H, W):
    usm = D.USMSharp()
    kern = R.usm_kernel().to(DEV)
    checked = 0
    for seed in range(30):
        g = torch.Generator(device=DEV).manual_seed(seed)
        # a smooth image with some edges: residuals on both sides of the threshold
        img = torch.nn.functional.interpolate(torch.rand(b, 3, H // 8 + 1, W // 8 + 1, generator=g, device=DEV), size=(H, W),
                                              mode="bicubic").clamp(0, 1)
        ref, mag = R.usm(img.double(), kern)
        if (mag - 10).abs().min().item() <= 1e-3:
            continue  # a pixel at the threshold: the mask is not determined by the restatement
        assert ((mag > 10).any() and (mag < 10).any()).item()
        assert (usm(img).double() - ref).abs().max().item() <= 5e-5
        checked += 1
    assert checked >= 2


def _mcu_flip_mask(ry, rc):
    """(b, H16 / 16, W16 / 16) bool: MCUs with a pre-rounding coefficient within 1e-3 of a half-integer"""
    near = lambda r: ((r - r.floor() - 0.5).abs() < 1e-3).flatten(-2).any(-1)
    y = near(ry)
    b, nh, nw = y.shape
    y = y.view(b, nh // 2, 2, nw // 2, 2).any(4).any(2)
    return y | near(rc).any(1)


@pytest.mark.parametrize("b,H,W", [(9, 600, 600), (9, 150, 150), (3, 37, 53), (2, 8, 24), (1, 150, 97)])
@pytest.mark.parametrize("scalar", [False, True])
def test_jpeg(b, H, W, scalar):
    # smooth content (quadratic per channel, out-of-range parts clamped): few coefficients away from zero, so few at a rounding tie
    g = torch.Generator(device=DEV).manual_seed(H + W)
    c = torch.rand(b, 3, 6, 1, 1, generator=g, device=DEV) - 0.5
    y, xx = torch.meshgrid(torch.linspace(0, 1, H, device=DEV), torch.linspace(0, 1, W, device=DEV), indexing="ij")
    x = 0.5 + sum(c[:, :, i] * t for i, t in enumerate((1, xx, y, xx * xx, xx * y, y * y))) * 1.2
    g = torch.Generator(device=DEV).manual_seed(b)
    quality = 63.0 if scalar else torch.empty(b, device=DEV).uniform_(30, 95, generator=g)
    q_before = None if scalar else quality.clone()
    factor = D.quality_to_factor(quality) if scalar else R.quality_to_factor(quality)
    xc = x.clamp(0, 1)
    got = D.DiffJPEG()(xc, quality)
    if not scalar:
        assert torch.equal(quality, q_before)  # not rewritten in place
        assert torch.equal(D._jpeg(x, quality, clamp_in=True), got)
        assert torch.equal(D._jpeg(x, quality, clamp_in=True, quantize_out=True), R.quant255(got))
    ref, ry, rc = R.jpeg(xc.double(), factor, return_ratios=True)
    flips = _mcu_flip_mask(ry, rc)
    # a 1e-3 window around each of an MCU's 384 coefficients: even on smooth content a few percent of MCUs fall in it; the exclusion
    # must leave most of the image checked
    assert flips.float().mean().item() < 0.15 or flips.numel() < 30
    assert (~flips).any().item()
    keep = ~flips.repeat_interleave(16, 1).repeat_interleave(16, 2)[:, :H, :W]
    err = (got.double() - ref).abs().amax(1)
    assert err[keep].max().item() <= 1e-4


def _replay(seed):
    torch.manual_seed(seed)


@pytest.mark.parametrize("b,c,H,W", [(9, 3, 150, 150), (2, 3, 37, 53), (3, 1, 20, 30)])
@pytest.mark.parametrize("gray_prob", [0.0, 0.4, 1.0])
def test_gaussian_noise(b, c, H, W, gray_prob):
    img = _img(b, H, W, 7, c)
    _replay(11)
    got = D.random_add_gaussian_noise_pt(img, sigma_range=(1, 30), gray_prob=gray_prob, clip=True, rounds=False)
    _replay(11)
    kw = dict(device=DEV)
    u_s, u_g = torch.rand(b, **kw), torch.rand(b, **kw)
    ng, n = torch.randn(H, W, **kw), torch.randn(b, c, H, W, **kw)
    ref = R.gaussian_noise(img.double(), u_s, u_g, ng, n, (1, 30), gray_prob)
    assert (got.double() - ref).abs().max().item() <= 1e-6
    _replay(11)
    unclipped = D.random_add_gaussian_noise_pt(img, sigma_range=(1, 30), gray_prob=gray_prob, clip=False, rounds=False)
    assert (unclipped.min() < 0).item() and torch.equal(unclipped.clamp(0, 1), got)
    _replay(11)
    rounded = D.random_add_gaussian_noise_pt(img, sigma_range=(1, 30), gray_prob=gray_prob, clip=True, rounds=True)
    assert torch.equal(rounded, R.quant255(unclipped))


@pytest.mark.parametrize("b,H,W", [(9, 150, 150), (2, 37, 53), (4, 9, 16)])
@pytest.mark.parametrize("gray_prob", [0.0, 0.4, 1.0])
def test_poisson_noise(b, H, W, gray_prob):
    img = _img(b, H, W, 5) * 1.1 - 0.05
    img[0] = (img[0] * 3).round() / 3  # an image with few levels
    if b > 1:
        img[1, :, :, : W // 2] = 0.5
    rates, rates_g, vals, vals_g = ops.noise_levels(img)
    r_rates, r_rates_g, r_vals, r_vals_g = R.poisson_levels(img)
    assert torch.equal(rates, r_rates) and torch.equal(rates_g, r_rates_g)
    assert torch.equal(vals, r_vals) and torch.equal(vals_g, r_vals_g)
    _replay(3)
    got = D.random_add_poisson_noise_pt(img, scale_range=(0.05, 3), gray_prob=gray_prob, clip=True, rounds=False)
    _replay(3)
    u_s, u_g = torch.rand(b, device=DEV), torch.rand(b, device=DEV)
    p_g = torch.poisson(r_rates_g)
    p = torch.poisson(r_rates)
    ref = R.poisson_noise(img.double(), u_s, u_g, p_g, p, r_vals, r_vals_g, (0.05, 3), gray_prob)
    assert (got.double() - ref).abs().max().item() <= 1e-6


def test_raises():
    img = _img(1, 30, 30, 0)
    with pytest.raises(TypeError):
        D.filter2D(img.double(), _kernels(1, 7, 0))
    with pytest.raises(TypeError):
        D.filter2D(img, _kernels(1, 7, 0).half())
    with pytest.raises(TypeError):
        D.random_add_gaussian_noise_pt(img.half(), (1, 2))
    with pytest.raises(TypeError):
        D.USMSharp()(img.to(torch.bfloat16))
    for k in (4, 53):
        with pytest.raises(ValueError):
            D.filter2D(img, torch.ones(1, k, k, device=DEV))
    with pytest.raises(ValueError):
        D.filter2D(_img(1, 10, 30, 0), _kernels(1, 21, 0))  # H = k // 2
    with pytest.raises(ValueError):
        D.filter2D(_img(1, 30, 25, 0), _kernels(1, 51, 0))
    with pytest.raises(ValueError):
        D.USMSharp()(_img(1, 25, 60, 0))
    D.filter2D(_img(1, 11, 11, 0), _kernels(1, 21, 0))  # H = k // 2 + 1 is fine


def _seed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def _recipe_inputs(b, H, seed):
    gt = _img(b, H, H, seed)
    return gt, _kernels(b, 21, seed + 1), _kernels(b, 21, seed + 2), _kernels(b, 21, seed + 3)


def test_pipeline_matches_the_restatement():
    deg = D.RealESRNetDegradation(OPT, 4)
    seen = set()
    for seed in (0, 1, 2, 3):
        gt, k1, k2, sinc = _recipe_inputs(9, 400, 100 + seed)
        _seed(seed)
        lq, gt_out = deg.degrade(gt, k1, k2, sinc)
        log = deg.log
        _seed(seed)
        ref, _, ref_log = R.feed_data(gt, k1, k2, sinc, OPT, 4)
        assert log == ref_log
        assert lq.shape == (9, 3, 100, 100) and torch.equal(gt_out, gt)
        assert torch.equal(lq, R.quant255(lq))  # on 8-bit levels
        d = (lq.double() - ref).abs()
        assert (d <= 1.5 / 255).double().mean().item() >= 0.995, (seed, log)
        assert d.mean().item() <= 1e-4, (seed, log)
        seen |= {e[1] for e in log if e[0] in ("noise1", "noise2", "final")} | {e[-1] for e in log if e[0] in ("resize1", "resize2", "final")}
    assert {"gaussian", "poisson", "sinc_first", "jpeg_first", "area", "bilinear", "bicubic"} <= seen


def test_pipeline_crop_and_pool():
    opt = dict(OPT, gt_size=64, queue_size=4)
    deg = D.RealESRNetDegradation(opt, 4)
    gt, k1, k2, sinc = _recipe_inputs(2, 128, 9)
    for step in range(3):
        _seed(step)
        lq, gt_out = deg(gt, k1, k2, sinc)
        assert lq.shape == (2, 3, 16, 16) and gt_out.shape == (2, 3, 64, 64) and lq.is_contiguous()
        top, left = deg.log[-1][1:]
        if step < 2:  # the pool is filling: the batch's own crop
            assert torch.equal(gt_out, gt[:, :, 4 * top:4 * top + 64, 4 * left:4 * left + 64])


def test_degrade_does_not_synchronise():
    deg = D.RealESRNetDegradation(dict(OPT, gt_usm=True), 4)
    gt, k1, k2, sinc = _recipe_inputs(9, 600, 1)
    for seed in range(4):  # every branch once, outside the check (first launches load modules)
        _seed(seed)
        deg.degrade(gt, k1, k2, sinc)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for seed in range(4):
            _seed(seed)
            deg.degrade(gt, k1, k2, sinc)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
