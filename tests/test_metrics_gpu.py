"""vmambair_b200.metrics (csrc/metrics.cu) against the reference's results (tests/golden/metrics_ref.npz) and the numpy restatement
oracle/metrics_ref.py.  Bounds: integer images without the Y channel, PSNR bit for bit; Y-PSNR within Y_PSNR_DB of the reference's
float32 value (derived in tests/test_metrics_cpu.py) and 1e-12 relative of the restatement summed in float64; float64 SSIM within 1e-10;
_ssim_3d within 1e-5 of its float32 Conv3d."""
import hashlib
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import metrics_ref as R
from vmambair_b200 import archs, metrics
from vmambair_b200.enhance import RealESRGANer
from vmambair_b200.metrics import calculate_psnr, calculate_ssim, psnr_ssim

from .test_metrics_cpu import CASES, FILTER_ABS, SSIM3D_ABS, Y_PSNR_DB, G, close, hwc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def inputs(case, where):
    """the case's two images as the reference received them: numpy arrays, or tensors on the host ('cpu') or the GPU ('cuda')"""
    crop, chw, tensor = (int(v) for v in G[f"{case}/meta"])
    a, b = G[f"{case}/img1"], G[f"{case}/img2"]
    if tensor or where != "numpy":
        if not tensor:  # an array as the reference's tensor form, (C, H, W)
            a, b = (x[None] if x.ndim == 2 else x if chw else x.transpose(2, 0, 1) for x in (a, b))
        dev = DEV if where == "cuda" else "cpu"
        a, b = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (a, b))
    return a, b, crop, "CHW" if chw and not isinstance(a, torch.Tensor) else "HWC"


@pytest.mark.parametrize("where", ["numpy", "cpu", "cuda"])
@pytest.mark.parametrize("case", CASES)
def test_dropins_match_the_reference(case, where):
    a, b, crop, order = inputs(case, where)
    h1, h2 = hwc(case)
    integer = G[f"{case}/img1"].dtype.kind == "u"
    p0 = calculate_psnr(a, b, crop, order)
    if integer:
        assert p0 == G[f"{case}/psnr_y0"], (p0, G[f"{case}/psnr_y0"])
    else:
        assert close(p0, G[f"{case}/psnr_y0"], 1e-9)
    p1 = calculate_psnr(a, b, crop, order, test_y_channel=True)
    assert close(p1, G[f"{case}/psnr_y1"], Y_PSNR_DB)
    want = R.psnr(h1, h2, True, accumulate="float64")
    assert close(p1, want, 1e-12 * abs(want)), (p1, want)
    assert close(calculate_ssim(a, b, crop, order, test_y_channel=True), G[f"{case}/ssim_y1"], FILTER_ABS)
    assert close(calculate_ssim(a, b, crop, order), G[f"{case}/ssim_y0"], SSIM3D_ABS)
    for y in (0, 1):
        got = calculate_ssim(a, b, crop, order, test_y_channel=bool(y), ssim="valid")
        assert close(got, G[f"{case}/ssim_valid_y{y}"], FILTER_ABS), (y, got)
    assert isinstance(p0, float) and isinstance(p1, float)


def test_identical_images_and_empty_maps():
    a = G["u8_identical/img1"]
    assert calculate_psnr(a, a, 2) == float("inf") and calculate_psnr(a, a, 2, test_y_channel=True) == float("inf")
    for y in (False, True):
        assert calculate_ssim(a, a, 2, test_y_channel=y) == 1.0
        assert calculate_ssim(a, a, 2, test_y_channel=y, ssim="valid") == 1.0
    s = G["u8_small/img1"]
    assert np.isnan(calculate_ssim(s, G["u8_small/img2"], 0, ssim="valid"))
    assert np.isnan(calculate_ssim(s, G["u8_small/img2"], 0, test_y_channel=True, ssim="valid"))


def test_invalid_arguments_raise():
    a = G["u8_hwc_crop4/img1"]
    t = torch.from_numpy(a.transpose(2, 0, 1).copy())
    with pytest.raises(ValueError):
        calculate_psnr(a, a[:-1], 0)
    with pytest.raises(ValueError):
        calculate_ssim(a, a, 0, input_order="WHC")
    with pytest.raises(ValueError):
        calculate_psnr(t, t, 0, input_order="CHW")
    with pytest.raises(ValueError):
        calculate_psnr(a, a, 19)  # 37 rows: nothing left
    with pytest.raises(ValueError):
        calculate_ssim(a, a, -1)
    with pytest.raises(ValueError):
        calculate_psnr(np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8, 4), np.uint8), 0)
    with pytest.raises(ValueError):
        psnr_ssim(torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=DEV), torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device=DEV), ssim="x")


def test_y_channel_of_every_triple_is_bit_exact():
    j = torch.arange(1 << 24, device=DEV, dtype=torch.int32)
    img = torch.stack([j >> 16, (j >> 8) & 255, j & 255], dim=-1).to(torch.uint8).view(1, 4096, 4096, 3)
    y = metrics.to_y_channel(img)[0].cpu().numpy()
    sha = hashlib.sha256()  # the layout and row order of tests/test_metrics_cpu.py::all_triples_y_sha256
    for r0 in range(0, 4096, 256):
        sha.update(np.ascontiguousarray(y[r0:r0 + 256], dtype="<f4").tobytes())
    assert sha.digest() == G["y_all_triples_sha256"].tobytes()


def _pairs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    b = (a.int() + torch.randint(-9, 10, a.shape, generator=g)).clamp(0, 255).to(torch.uint8)
    return a.to(DEV), b.to(DEV)


def _bits(t):
    return t.double().cpu().numpy().view(np.int64)


@pytest.mark.parametrize("ssim", ["valid", "reference"])
@pytest.mark.parametrize("y", [True, False])
def test_batch_equals_separate_calls_and_strided_views(ssim, y):
    a, b = _pairs(4, 61, 77, 1)
    p, s = psnr_ssim(a, b, 3, y, ssim)
    for i in range(4):
        pi, si = psnr_ssim(a[i:i + 1], b[i:i + 1], 3, y, ssim)
        assert _bits(pi)[0] == _bits(p)[i] and _bits(si)[0] == _bits(s)[i]
    # the same pixels inside larger tensors (rows, pixels, channels and the batch all strided) and channels-first storage
    big = torch.zeros(8, 70, 90, 5, dtype=torch.uint8, device=DEV)
    big[::2, 4:65, 6:83, 1:4] = a
    view = big[::2, 4:65, 6:83, 1:4]
    chf = b.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    pv, sv = psnr_ssim(view, chf, 3, y, ssim)
    assert (_bits(pv) == _bits(p)).all() and (_bits(sv) == _bits(s)).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_quantized_network_output(dtype):
    for i in (0, 1):
        x = torch.from_numpy(G[f"quant{i}/x"]).to(dtype)
        gt = G[f"quant{i}/gt"]
        q = R.tensor2img(x.float().numpy())  # restated tensor2img (pinned to the reference's in tests/test_metrics_cpu.py)
        xd = x.to(DEV).unsqueeze(0)
        gd = torch.from_numpy(gt).to(DEV).unsqueeze(0)
        qd = torch.from_numpy(q.copy()).to(DEV).unsqueeze(0)
        for y in (True, False):
            for ssim in ("valid", "reference"):
                got = psnr_ssim(xd, gd, 2, y, ssim, quantize=True)
                want = psnr_ssim(qd, gd, 2, y, ssim)
                assert all((_bits(g) == _bits(w)).all() for g, w in zip(got, want))
        if dtype == torch.float32:
            assert np.array_equal(q, G[f"quant{i}/tensor2img"])
            assert calculate_psnr(q, gt, 2) == G[f"quant{i}/psnr_y0"]
            assert close(calculate_ssim(q, gt, 2), G[f"quant{i}/ssim_y0"], SSIM3D_ABS)
        # a strided network output (a channel slice of a wider batch) reads the same
        wide = torch.zeros(2, 5, *x.shape[1:], dtype=dtype, device=DEV)
        wide[1, 1:4] = x.to(DEV)
        got = psnr_ssim(wide[1:2, 1:4], gd, 2, True, "valid", quantize=True)
        want = psnr_ssim(xd, gd, 2, True, "valid", quantize=True)
        assert all((_bits(g) == _bits(w)).all() for g, w in zip(got, want))


def test_deterministic():
    a, b = _pairs(2, 300, 260, 2)
    first = [psnr_ssim(a, b, 4, y, s) for y in (True, False) for s in ("valid", "reference")]
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        torch.use_deterministic_algorithms(True)
        try:
            second = [psnr_ssim(a, b, 4, y, s) for y in (True, False) for s in ("valid", "reference")]
        finally:
            torch.use_deterministic_algorithms(False)
    for (p1, s1), (p2, s2) in zip(first, second):
        assert (_bits(p1) == _bits(p2)).all() and (_bits(s1) == _bits(s2)).all()


def test_full_size_pair_against_the_restatement():
    """a 2040 x 1356 pair (DIV2K's size), Y, crop 4, both SSIM conventions"""
    rng = np.random.default_rng(7)
    gt = rng.integers(0, 256, (1356, 2040, 3), dtype=np.uint8)
    sr = np.clip(gt.astype(np.int16) + rng.integers(-12, 13, gt.shape), 0, 255).astype(np.uint8)
    h1, h2 = (x.astype(np.float64)[4:-4, 4:-4] for x in (sr, gt))
    want = R.psnr(h1, h2, True, accumulate="float64")
    assert close(calculate_psnr(sr, gt, 4, test_y_channel=True), want, 1e-12 * want)
    p, s = psnr_ssim(torch.from_numpy(sr).to(DEV)[None], torch.from_numpy(gt).to(DEV)[None], 4, True, "valid")
    assert abs(p.item() - want) <= 1e-12 * want
    assert abs(s.item() - R.ssim(h1, h2, True, "valid")) <= FILTER_ABS
    assert abs(calculate_ssim(sr, gt, 4, test_y_channel=True) - R.ssim(h1, h2, True, "reference")) <= FILTER_ABS


def test_enhance_output_scored_end_to_end():
    with np.load(os.path.join(GOLDEN, "enhance_net_sisr.npz")) as f:
        sd = {k: torch.from_numpy(f[k].astype(np.float32)) for k in f.files}
    net = archs.MambaSISR6(dim=8, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1)
    net.load_state_dict(sd)
    up = RealESRGANer(4, None, model=net, pre_pad=0)
    rng = np.random.default_rng(11)
    lr = rng.integers(0, 256, (24, 32, 3), dtype=np.uint8)
    gt = rng.integers(0, 256, (96, 128, 3), dtype=np.uint8)
    sr, _ = up.enhance(lr)
    h1, h2 = (x.astype(np.float64)[4:-4, 4:-4] for x in (sr, gt))
    assert calculate_psnr(sr, gt, 4) == R.psnr(h1, h2)
    want = R.psnr(h1, h2, True, accumulate="float64")
    assert close(calculate_psnr(sr, gt, 4, test_y_channel=True), want, 1e-12 * want)
    assert close(calculate_ssim(sr, gt, 4, test_y_channel=True), R.ssim(h1, h2, True, "reference"), FILTER_ABS)
    assert close(calculate_ssim(sr, gt, 4, test_y_channel=True, ssim="valid"), R.ssim(h1, h2, True, "valid"), FILTER_ABS)
    assert close(calculate_ssim(sr, gt, 4), R.ssim(h1, h2, False, "reference"), 1e-10)
