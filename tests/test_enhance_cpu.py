"""vmambair_b200.enhance host logic and the numpy restatements of OpenCV (vmambair_b200.image_ref) against OpenCV's own results,
stored by tests/golden/make_golden_enhance.py (no OpenCV needed here)."""
import os

import numpy as np
import pytest
import torch

from vmambair_b200 import enhance, image_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def cv():
    with np.load(os.path.join(GOLDEN, "enhance_cv2.npz")) as f:
        return {k: f[k] for k in f.files}


def test_image_mode():
    assert enhance.image_mode((5, 7)) == "L"
    assert enhance.image_mode((5, 7, 3)) == "RGB"
    assert enhance.image_mode((5, 7, 4)) == "RGBA"
    for bad in ((5, 7, 1), (5, 7, 2), (5,), (2, 5, 7, 3)):
        with pytest.raises(ValueError):
            enhance.image_mode(bad)


def test_max_range_follows_the_reference_16_bit_test():
    assert enhance.max_range_of(255, np.uint8) == 255
    assert enhance.max_range_of(256, np.uint16) == 255  # uint16 with max <= 256: processed and returned as 8-bit
    assert enhance.max_range_of(257, np.uint16) == 65535
    assert enhance.max_range_of(65535, torch.uint16) == 65535


@pytest.mark.parametrize("h,w,pre_pad,scale,want", [
    (22, 30, 10, 4, ((10, 0, 0), (10, 0, 0))),        # H + pre_pad already a multiple of 8
    (21, 30, 10, 4, ((10, 0, 1), (10, 0, 0))),
    (13, 17, 0, 4, ((0, 0, 3), (0, 0, 7))),
    (13, 18, 10, 2, ((10, 1, 0), (10, 0, 4))),        # scale 2: mod pad to even, then to 8
    (13, 17, 10, 1, ((10, 1, 0), (10, 1, 4))),        # scale 1: mod pad to a multiple of 4
])
def test_pad_plan(h, w, pre_pad, scale, want):
    ph, pw = enhance.pad_plan(h, w, pre_pad, scale)
    assert (ph, pw) == want
    assert (h + sum(ph)) % 8 == 0 and (w + sum(pw)) % 8 == 0


def test_pad_plan_rejects_pads_reflect_cannot_make():
    with pytest.raises(ValueError):
        enhance.pad_plan(8, 30, 10, 4)  # pre_pad 10 >= H 8: F.pad 'reflect' fails in the reference too
    with pytest.raises(ValueError):
        enhance.pad_plan(1, 1, 0, 4)    # a 1-pixel image cannot be reflected to 8


def test_output_size():
    assert enhance.output_size(22, 30, 4) == (88, 120)
    assert enhance.output_size(22, 30, 4, 4.0) == (88, 120)
    assert enhance.output_size(22, 30, 4, 3.5) == (77, 105)
    assert enhance.output_size(22, 30, 4, 2) == (44, 60)


def test_output_dtype_rules_in_the_reference_fixtures():
    with np.load(os.path.join(GOLDEN, "enhance_ref.npz")) as f:
        names = sorted({k.split("/")[0] for k in f.files})
        assert len(names) == 12
        for n in names:
            img, out = f[f"{n}/img"], f[f"{n}/out"]
            want = np.uint16 if enhance.max_range_of(int(img.max()), img.dtype) == 65535 else np.uint8
            assert out.dtype == want, n
            pre_pad, tile, tile_pad, outscale, _ = f[f"{n}/params"]
            assert out.shape[:2] == enhance.output_size(*img.shape[:2], 4, None if outscale < 0 else float(outscale)), n
            assert out.ndim == img.ndim, n


def test_requires_a_model():
    with pytest.raises((ValueError, RuntimeError)):
        enhance.RealESRGANer(4, None, model=None)


@pytest.mark.parametrize("i", range(6))
@pytest.mark.parametrize("depth", ["uint8", "uint16"])
def test_lanczos4_restatement_is_bit_exact(cv, i, depth):
    src, dst = cv[f"lanczos{i}_{depth}/src"], cv[f"lanczos{i}_{depth}/dst"]
    got = image_ref.resize_lanczos4(src, (dst.shape[1], dst.shape[0]))
    assert got.dtype == dst.dtype and got.shape == dst.shape
    np.testing.assert_array_equal(got, dst)


def test_bgr2gray_restatement_is_bit_exact(cv):
    np.testing.assert_array_equal(image_ref.bgr2gray(cv["gray/src"]), cv["gray/dst"])


def test_fma32_rounds_once():
    a, b = np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12)
    c = np.float32(-1)
    # a*b - 1 = 2^-11 + 2^-24 exactly: representable, and lost if a*b were rounded to float32 first
    assert image_ref.fma32(a, b, c) == np.float32(2 ** -11 + 2 ** -24)


@pytest.mark.parametrize("i", range(3))
def test_linear_restatement_within_one_ulp(cv, i):
    """OpenCV's float INTER_LINEAR runs through Intel IPP where the build has it; IPP differs from OpenCV's generic loop (which the
    restatement follows) by at most 2^-23 (one float32 ulp of 1.0), which after x max_range and rounding is at most 1 LSB"""
    src, dst = cv[f"linear{i}/src"], cv[f"linear{i}/dst"]
    got = image_ref.resize_linear(src, (dst.shape[1], dst.shape[0]))
    assert got.shape == dst.shape
    assert np.abs(got - dst).max() <= np.spacing(np.float32(1))
    for m in (255.0, 65535.0):
        d = np.abs(np.round(got * np.float32(m)).astype(np.int64) - np.round(dst * np.float32(m)).astype(np.int64))
        assert d.max() <= 1
