"""The metric restatement (oracle/metrics_ref.py) against the reference's own results (tests/golden/metrics_ref.npz, written by
tests/golden/make_golden_metrics.py): bit for bit where the reference computes in float64 without a filter, within the float64
filter's rounding (1e-10) for the cv2.filter2D SSIMs, and within the bounds below where the reference computes in float32."""
import hashlib
import os

import numpy as np
import pytest
from scipy.ndimage import correlate1d

from oracle import metrics_ref as R
from vmambair_b200 import metrics

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "metrics_ref.npz")
G = np.load(GOLDEN)
CASES = [str(c) for c in G["cases"]]

# Y-PSNR: the reference sums the float32 squared differences with numpy's float32 pairwise sum and takes sqrt / log10 in float32.
# Relative error of that mse: at most ~(16 + log2(N / 128) + 2) eps32 (eight sequential adds per lane of a 128-element block, one
# level per pairwise halving, the square and the mean's division), under 2.2e-6 for N <= 2^22 pixels, i.e. 4.343 x 2.2e-6 < 1e-5 dB.
# The float32 log10 of a value below 3 and 20 x it round by at most 2.4e-7 x 20 and 3.8e-6 / 2 dB.  Together under 2e-5 dB.
Y_PSNR_DB = 2e-5
FILTER_ABS = 1e-10  # float64 SSIM: cv2.filter2D's DFT against a direct float64 filter
SSIM3D_ABS = 1e-5   # _ssim_3d runs its Conv3d in float32


def hwc(case):
    """the reference's float64 HWC image pair, cropped (reorder_image / the tensor transpose, astype(float64), crop)"""
    crop, chw, tensor = (int(v) for v in G[f"{case}/meta"])
    out = []
    for k in ("img1", "img2"):
        a = G[f"{case}/{k}"]
        if tensor:
            a = (a[0] if a.ndim == 4 else a).transpose(1, 2, 0)
        elif a.ndim == 2:
            a = a[..., None]
        elif chw:
            a = a.transpose(1, 2, 0)
        a = a.astype(np.float64)
        out.append(a[crop:-crop, crop:-crop] if crop else a)
    return out


def close(a, b, tol):
    return (np.isnan(a) and np.isnan(b)) or a == b or abs(a - b) <= tol


def test_gaussian_taps():
    assert np.array_equal(np.array(metrics.TAPS), G["gauss"])
    assert np.abs(R.TAPS - G["gauss"]).max() <= 1e-16


def test_channel_mix_is_the_replicate_padded_filter():
    for c in (1, 3):
        want = correlate1d(np.eye(c), np.array(metrics.TAPS), axis=0, mode="nearest")  # column p: the filter of one-hot channel p
        assert np.abs(np.array(metrics.channel_mix(c)) - want).max() <= 4e-16  # summation order


@pytest.mark.parametrize("case", CASES)
def test_psnr(case):
    a, b = hwc(case)
    assert R.psnr(a, b) == G[f"{case}/psnr_y0"] or (np.isinf(R.psnr(a, b)) and np.isinf(G[f"{case}/psnr_y0"]))
    y = G[f"{case}/psnr_y1"]
    assert close(R.psnr(a, b, True), y, 0.0)
    assert close(R.psnr(a, b, True, accumulate="float64"), y, Y_PSNR_DB)


@pytest.mark.parametrize("case", CASES)
def test_ssim(case):
    a, b = hwc(case)
    assert close(R.ssim(a, b, True, "reference"), G[f"{case}/ssim_y1"], FILTER_ABS)
    assert close(R.ssim(a, b, False, "reference"), G[f"{case}/ssim_y0"], SSIM3D_ABS)
    for y in (0, 1):
        assert close(R.ssim(a, b, bool(y), "valid"), G[f"{case}/ssim_valid_y{y}"], FILTER_ABS), y


def test_edge_cases_are_covered():
    assert np.isnan(G["u8_small/ssim_valid_y0"]) and np.isnan(G["u8_small_after_crop/ssim_valid_y1"])
    assert np.isinf(G["u8_identical/psnr_y0"]) and G["u8_identical/ssim_y1"] == 1.0


@pytest.mark.parametrize("i", [0, 1])
def test_tensor2img_and_quantized_scores(i):
    q = R.tensor2img(G[f"quant{i}/x"])
    assert np.array_equal(q, G[f"quant{i}/tensor2img"])
    x = G[f"quant{i}/x"]
    assert ((x * np.float32(255)) % 1 == 0.5).any(), "the case holds exact .5 ties"
    a, b = (v.astype(np.float64)[2:-2, 2:-2] for v in (q, G[f"quant{i}/gt"]))
    assert R.psnr(a, b) == G[f"quant{i}/psnr_y0"]
    assert close(R.psnr(a, b, True), G[f"quant{i}/psnr_y1"], 0.0)
    assert close(R.ssim(a, b, True, "reference"), G[f"quant{i}/ssim_y1"], FILTER_ABS)
    assert close(R.ssim(a, b, False, "reference"), G[f"quant{i}/ssim_y0"], SSIM3D_ABS)


def all_triples_y_sha256(to_y):
    """SHA-256 of to_y over all 2^24 BGR triples laid out as tests/golden/make_golden_metrics.py does (float32 bytes, row order)"""
    sha = hashlib.sha256()
    i = np.arange(4096 * 256, dtype=np.int64)
    for r0 in range(0, 4096, 256):
        j = i + r0 * 4096
        img = np.stack([j >> 16, (j >> 8) & 255, j & 255], axis=-1).reshape(256, 4096, 3).astype(np.float64)
        sha.update(np.ascontiguousarray(to_y(img), dtype="<f4").tobytes())
    return sha.digest()


def test_y_channel_of_every_triple():
    assert all_triples_y_sha256(R.to_y_channel) == G["y_all_triples_sha256"].tobytes()
