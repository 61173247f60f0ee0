"""NumPy restatement of the reference's image metrics (Deraining/basicsr/metrics/psnr_ssim.py, metric_util.py::to_y_channel,
utils/matlab_functions.py::bgr2ycbcr, Deraining/Deraining/utils.py) and of tensor2img (SRGAN/VmambaIR/utils/img_util.py).  Test
infrastructure only: the tests compare vmambair_b200.metrics with it, and it with the reference's own outputs (tests/golden).

Images are float64 (H, W, C) arrays in BGR order (C = 1 or 3), already cropped, as the reference holds them after astype(np.float64).
The 11 x 11 Gaussian filters run separably in float64 (scipy.ndimage.correlate1d); OpenCV's filter2D takes a DFT for a kernel this
size, so the two agree to ~1e-13, not bit for bit."""
import math

import numpy as np
from scipy.ndimage import correlate1d

C1_255, C2_255 = (0.01 * 255) ** 2, (0.03 * 255) ** 2


def gaussian_taps():
    """cv2.getGaussianKernel(11, 1.5): t_i = exp(-0.5 / 1.5^2 * (i - 5)^2), each times 1 / sum(t), in float64"""
    t = [math.exp(-0.5 / (1.5 * 1.5) * (i - 5.0) ** 2) for i in range(11)]
    s = 1.0 / sum(t)
    return np.array([v * s for v in t])


TAPS = gaussian_taps()


def to_y_channel(img):
    """(H, W, C) float64 -> (H, W) float32: to_y_channel's precision chain (x / 255 in float32; the BGR dot product + 16 in float64,
    left to right; / 255 in float64, cast to float32; x 255 in float32); one channel: the float32 round trip"""
    x = img.astype(np.float32) / np.float32(255)
    if img.shape[2] == 3:
        d = x.astype(np.float64)
        y = ((d[..., 0] * 24.966 + d[..., 1] * 128.553) + d[..., 2] * 65.481) + 16.0
        x = (y / 255.0).astype(np.float32)
    else:
        x = x[..., 0]
    return x * np.float32(255)


def tensor2img(t):
    """(3, H, W) RGB float tensor / array -> (H, W, 3) uint8 BGR: clamp to [0, 1], x 255 in float32 rounded half to even"""
    a = np.asarray(t, dtype=np.float32).clip(0, 1).transpose(1, 2, 0)[..., ::-1]
    return (a * np.float32(255)).round().astype(np.uint8)


def psnr(img1, img2, test_y_channel=False, accumulate=None):
    """calculate_psnr on cropped float64 images.  Without the Y channel: float64 throughout, as the reference.  With it: float32
    (a - b)^2; accumulate=None sums them as the reference does (np.mean and log10 in float32), accumulate='float64' sums them in
    float64 and takes log10 in float64 (what the device computes)."""
    if test_y_channel:
        a, b = to_y_channel(img1), to_y_channel(img2)
        sq = (a - b) ** 2
        mse = np.mean(sq, dtype=np.float64) if accumulate == "float64" else np.mean(sq)
    else:
        a = img1
        mse = np.mean((img1 - img2) ** 2)
    if mse == 0:
        return float("inf")
    max_value = 1. if a.max() <= 1 else 255.
    if accumulate == "float64":
        return float(20. * np.log10(max_value / np.sqrt(np.float64(mse))))
    return float(20. * np.log10(max_value / np.sqrt(mse)))


def _filter(x, mode):
    """11 x 11 Gaussian window of float64 plane(s) x (H, W[, C]); mode 'mirror' (OpenCV's default border) or 'nearest' (replicate)"""
    return correlate1d(correlate1d(x, TAPS, axis=0, mode=mode), TAPS, axis=1, mode=mode)


def _ssim_map(mu1, mu2, f11, f22, f12, C1, C2):
    mu1_sq, mu2_sq, mu1_mu2 = mu1 ** 2, mu2 ** 2, mu1 * mu2
    s1, s2, s12 = f11 - mu1_sq, f22 - mu2_sq, f12 - mu1_mu2
    return ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))


def _moments(a, b, mode):
    return [_filter(v, mode) for v in (a, b, a * a, b * b, a * b)]


def ssim_valid_plane(a, b):
    """_ssim / utils.ssim: the mean of the map where the window fits (nan when none does)"""
    if a.shape[0] < 11 or a.shape[1] < 11:
        return float("nan")
    m = [v[5:-5, 5:-5] for v in _moments(a, b, "mirror")]
    return float(_ssim_map(*m, C1_255, C2_255).mean())


def ssim(img1, img2, test_y_channel=False, convention="valid"):
    """SSIM on cropped float64 images.  convention 'valid': the channels' mean of ssim_valid_plane (pip basicsr, utils.py), on Y
    with test_y_channel; 'reference': psnr_ssim.calculate_ssim (_ssim_cly on Y, _ssim_3d otherwise), in float64"""
    if test_y_channel:
        planes = [to_y_channel(img1).astype(np.float64)], [to_y_channel(img2).astype(np.float64)]
    else:
        planes = [img1[..., c] for c in range(img1.shape[2])], [img2[..., c] for c in range(img2.shape[2])]
    if convention == "valid":
        return float(np.array([ssim_valid_plane(a, b) for a, b in zip(*planes)]).mean())
    if test_y_channel:
        return float(_ssim_map(*_moments(planes[0][0], planes[1][0], "nearest"), C1_255, C2_255).mean())
    # _ssim_3d: the 2-D window on every channel, then the same 11 taps across the channels, ends replicated
    max_value = 1 if img1.max() <= 1 else 255
    m = [correlate1d(_filter(v, "nearest"), TAPS, axis=2, mode="nearest") for v in (img1, img2, img1 * img1, img2 * img2, img1 * img2)]
    return float(_ssim_map(*m, (0.01 * max_value) ** 2, (0.03 * max_value) ** 2).mean())
