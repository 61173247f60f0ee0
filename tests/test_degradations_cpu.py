"""The float64 restatement of the degradation operators (oracle/degradations_ref.py) and the library's host-side pieces, pinned against
independent code: cv2's DCT and Gaussian kernel, scipy's correlate, torchvision's gray conversion and numpy's unique."""
import cv2
import numpy as np
import pytest
import torch
from scipy.ndimage import correlate
from torchvision.transforms import _functional_tensor as TF

from oracle import degradations_ref as R
from vmambair_b200 import degradations as D


def test_dct_stage_is_cv2_dct():
    rng = np.random.default_rng(0)
    blocks = rng.uniform(-128, 127, (20, 8, 8))
    got = R.dct8(torch.from_numpy(blocks)).numpy()
    for b, g in zip(blocks, got):
        np.testing.assert_allclose(g, cv2.dct(b), rtol=0, atol=1e-11)
        np.testing.assert_allclose(R.idct8(torch.from_numpy(g)).numpy(), b, rtol=0, atol=1e-11)


@pytest.mark.parametrize("ksize,sigma", [(1, 0), (3, 0), (5, 0), (7, 0), (9, 0), (11, 0), (21, 0), (51, 0), (21, 2.5), (7, 1.2)])
def test_gaussian_kernel_is_cv2s(ksize, sigma):
    np.testing.assert_allclose(D.gaussian_kernel_1d(ksize, sigma), cv2.getGaussianKernel(ksize, sigma), rtol=1e-14, atol=0)


def test_usm_kernel_is_outer_of_cv2_gaussian():
    g = cv2.getGaussianKernel(51, 0)
    want = np.outer(g, g)
    np.testing.assert_allclose(R.usm_kernel()[0].numpy(), want, rtol=0, atol=0)
    usm = D.USMSharp()
    assert usm.radius == 51 and tuple(usm.kernel.shape) == (1, 51, 51) and usm.kernel.dtype == torch.float32
    np.testing.assert_allclose(usm.kernel[0].numpy(), want.astype(np.float32), rtol=2e-7, atol=0)
    np.testing.assert_allclose(usm.taps, g.ravel().astype(np.float32), rtol=2e-7, atol=0)


@pytest.mark.parametrize("k,H,W", [(3, 9, 13), (7, 4, 30), (21, 11, 40), (21, 37, 23)])
@pytest.mark.parametrize("per_image", [False, True])
def test_filter2d_is_scipy_mirror_correlation(k, H, W, per_image):
    g = torch.Generator().manual_seed(k * H + W)
    img = torch.rand(2, 3, H, W, generator=g, dtype=torch.float64)
    kern = torch.rand(2 if per_image else 1, k, k, generator=g, dtype=torch.float64)
    got = R.filter2d(img, kern).numpy()
    for b in range(2):
        for c in range(3):
            want = correlate(img[b, c].numpy(), kern[b if per_image else 0].numpy(), mode="mirror")
            np.testing.assert_allclose(got[b, c], want, rtol=0, atol=1e-12)


def test_gray_is_torchvisions():
    img = torch.rand(3, 3, 17, 19, generator=torch.Generator().manual_seed(1))
    assert torch.equal(R.gray(img), TF.rgb_to_grayscale(img, 1))


def test_poisson_levels_count_with_numpy_unique():
    g = torch.Generator().manual_seed(2)
    imgs = [torch.full((3, 20, 24), 0.5), torch.randint(0, 2, (3, 20, 24), generator=g) / 255.0,
            torch.randint(0, 3, (3, 20, 24), generator=g) * 0.3, torch.rand(3, 20, 24, generator=g),
            torch.rand(3, 20, 24, generator=g) * 1.2 - 0.1]
    img = torch.stack(imgs).float()
    rates, rates_g, vals, vals_g = R.poisson_levels(img)
    for i, x in enumerate(img.numpy()):
        for v, src in ((vals, x), (vals_g, TF.rgb_to_grayscale(torch.from_numpy(x)[None], 1)[0].numpy())):
            q = np.clip(np.round(src * np.float32(255)), 0, 255) / np.float32(255)
            assert v[i].item() == 2.0 ** np.ceil(np.log2(len(np.unique(q))))
    assert vals.tolist()[:3] == [1.0, 2.0, 4.0]


@pytest.mark.parametrize("q,want", [(30, 5000 / 30 / 100), (49.5, 5000 / 49.5 / 100), (50, 1.0), (95, 0.1)])
def test_quality_to_factor(q, want):
    got = R.quality_to_factor(torch.tensor([q], dtype=torch.float32))
    assert got.dtype == torch.float32 and abs(got.item() - want) <= 1e-7 * want
    assert abs(D.quality_to_factor(q) - want) <= 1e-15 * want


def test_quality_100_round_trip_of_a_smooth_image():
    y, x = torch.meshgrid(torch.linspace(0, 1, 64, dtype=torch.float64), torch.linspace(0, 1, 96, dtype=torch.float64), indexing="ij")
    img = torch.stack([0.3 + 0.3 * x, 0.5 + 0.2 * torch.sin(2 * y), 0.4 + 0.2 * x * y])[None]
    assert (R.jpeg(img, D.quality_to_factor(100)) - img).abs().max().item() < 1 / 255  # 4:2:0 chroma alone
    assert (R.jpeg(img, D.quality_to_factor(95)) - img).abs().max().item() < 3 / 255


def test_diffjpeg_differentiable_is_not_implemented():
    with pytest.raises(NotImplementedError):
        D.DiffJPEG(differentiable=True)


def test_non_float32_raises_type_error():
    with pytest.raises(TypeError):
        D.filter2D(torch.zeros(1, 3, 8, 8, dtype=torch.float64), torch.ones(1, 3, 3))
    with pytest.raises(TypeError):
        D.DiffJPEG()(torch.zeros(1, 3, 8, 8, dtype=torch.float16), 50)
