"""numpy restatements of the OpenCV operations `RealESRGANer.enhance` uses (RealSR/VmambaIR/utils.py:174-243), written out operation
by operation in the precision and order OpenCV 4 evaluates them, so that the CUDA kernels of vmambair_b200/csrc/image_io.cu can be
checked bit for bit without OpenCV:

  * resize_lanczos4   cv2.resize(img, (w, h), interpolation=cv2.INTER_LANCZOS4) on uint8 / uint16 (H, W[, C])
  * bgr2gray          cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) on float32 (H, W, 3)
  * resize_linear     cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR) on float32 (H, W)

OpenCV's generic resize clamps source indices at the border (a replicated border) in both directions.  Coefficients and source
positions follow resize.cpp: fx = float((dx + 0.5) / (dw / sw) - 0.5), sx = floor(fx), fx -= sx; Lanczos-4 taps at sx - 3 .. sx + 4
with sin / cos in double and the eight weights normalised in float.  8-bit images use 11-bit fixed-point weights and round the
22-bit vertical sum; 16-bit images are filtered in float and rounded half to even, then saturated.
"""
from __future__ import annotations

import math

import numpy as np

_S45 = 0.70710678118654752440084436210485
_CS = ((1, 0), (-_S45, -_S45), (0, 1), (_S45, -_S45), (-1, 0), (_S45, _S45), (0, -1), (-_S45, _S45))
COEF_SCALE = 2048  # INTER_RESIZE_COEF_SCALE: 8-bit fixed-point weights


def src_positions(dst: int, src: int):
    """(sx, fx) per destination index: the source index left of the sample point and the float32 fraction past it"""
    scale = 1.0 / (float(dst) / float(src))
    f = np.array([np.float32((d + 0.5) * scale - 0.5) for d in range(dst)], dtype=np.float32)
    s = np.floor(f).astype(np.int64)
    return s, (f - s.astype(np.float32)).astype(np.float32)


def lanczos4_coeffs(x: np.float32) -> np.ndarray:
    """interpolateLanczos4: the eight float32 weights for fraction x"""
    x = np.float32(x)
    y0 = float(-(x + np.float32(3))) * math.pi * 0.25
    s0, c0 = math.sin(y0), math.cos(y0)
    c = np.zeros(8, np.float32)
    total = np.float32(0)
    for i in range(8):
        yi = np.float32(x + np.float32(3) - np.float32(i))
        if abs(yi) >= np.float32(1e-6):
            y = float(-yi) * math.pi * 0.25
            c[i] = np.float32((_CS[i][0] * s0 + _CS[i][1] * c0) / (y * y))
        else:
            c[i] = np.float32(1e30)
        total = np.float32(total + c[i])
    inv = np.float32(np.float32(1) / total)
    return (c * inv).astype(np.float32)


def _taps(dst: int, src: int):
    """(index (dst, 8) clamped to the image, weights (dst, 8) float32)"""
    s, f = src_positions(dst, src)
    idx = np.clip(s[:, None] - 3 + np.arange(8)[None, :], 0, src - 1)
    w = np.stack([lanczos4_coeffs(v) for v in f])
    return idx, w


def resize_lanczos4(img: np.ndarray, dsize) -> np.ndarray:
    """cv2.resize(img, dsize=(w, h), interpolation=cv2.INTER_LANCZOS4) for uint8 / uint16 images (H, W) or (H, W, C)"""
    if img.dtype not in (np.uint8, np.uint16):
        raise TypeError(f"resize_lanczos4: uint8 / uint16 only, got {img.dtype}")
    dw, dh = int(dsize[0]), int(dsize[1])
    sh, sw = img.shape[:2]
    xi, xw = _taps(dw, sw)
    yi, yw = _taps(dh, sh)
    src = img if img.ndim == 3 else img[:, :, None]
    if img.dtype == np.uint8:
        ax = np.array([[_sat_short(v * np.float32(COEF_SCALE)) for v in r] for r in xw], np.int64)
        ay = np.array([[_sat_short(v * np.float32(COEF_SCALE)) for v in r] for r in yw], np.int64)
        rows = np.zeros((sh, dw, src.shape[2]), np.int64)
        for k in range(8):
            rows += src[:, xi[:, k], :].astype(np.int64) * ax[None, :, k, None]
        acc = np.zeros((dh, dw, src.shape[2]), np.int64)
        for k in range(8):
            acc += rows[yi[:, k]] * ay[:, k, None, None]
        wrap = lambda v: (v + (1 << 31)) % (1 << 32) - (1 << 31)  # OpenCV's int32 sums
        out = np.clip(wrap(wrap(acc) + (1 << 21)) >> 22, 0, 255).astype(np.uint8)
    else:
        rows = np.zeros((sh, dw, src.shape[2]), np.float32)
        for k in range(8):
            rows = (rows + src[:, xi[:, k], :].astype(np.float32) * xw[None, :, k, None]).astype(np.float32)
        acc = (rows[yi[:, 0]] * yw[:, 0, None, None]).astype(np.float32)
        for k in range(1, 8):
            acc = (acc + rows[yi[:, k]] * yw[:, k, None, None]).astype(np.float32)
        out = np.clip(np.rint(acc), 0, 65535).astype(np.uint16)
    return out if img.ndim == 3 else out[:, :, 0]


def _sat_short(v: np.float32) -> int:
    return int(np.clip(np.rint(v), -32768, 32767))


# cv2's BGR2GRAY weights, as float32 (color_rgb.simd.hpp: B2Y / G2Y / R2Y)
GRAY_B, GRAY_G, GRAY_R = np.float32(0.114), np.float32(0.587), np.float32(0.299)


def fma32(a, b, c) -> np.ndarray:
    """float32 fused multiply-add a*b + c, rounded once: a*b is exact in float64, the float64 sum is rounded to odd (TwoSum error
    term), and rounding that to float32 is then the correctly rounded result"""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    bits = s.view(np.int64)
    even = (bits & 1) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def bgr2gray(img: np.ndarray) -> np.ndarray:
    """cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) on float32 (H, W, 3) as OpenCV's vector loop evaluates it: fma(r, 0.299, fma(b, 0.114,
    g*0.587)) in float32 (its scalar tail, the last pixels of an image whose pixel count is not a multiple of the vector width,
    computes b*0.114 + g*0.587 + r*0.299 instead)"""
    img = img.astype(np.float32, copy=False)
    b, g, r = img[..., 0], img[..., 1], img[..., 2]
    return fma32(r, GRAY_R, fma32(b, GRAY_B, (g * GRAY_G).astype(np.float32)))


def resize_linear(img: np.ndarray, dsize) -> np.ndarray:
    """cv2.resize(img, dsize=(w, h), interpolation=cv2.INTER_LINEAR) on float32 (H, W): half-pixel centres, replicated border,
    horizontal pass s0*a0 + s1*a1, then vertical pass r0*b0 + r1*b1, each in float32.  This is OpenCV's generic resize; builds with
    Intel IPP run float INTER_LINEAR through IPP instead, whose results differ from these by at most 2^-23 on [0, 1] images."""
    img = img.astype(np.float32, copy=False)
    dw, dh = int(dsize[0]), int(dsize[1])
    sh, sw = img.shape

    def taps(dst, src):
        s, f = src_positions(dst, src)
        f = np.where(s < 0, np.float32(0), f).astype(np.float32)
        s = np.maximum(s, 0)
        f = np.where(s >= src - 1, np.float32(0), f).astype(np.float32)
        s = np.minimum(s, src - 1)
        return s, np.minimum(s + 1, src - 1), (np.float32(1) - f).astype(np.float32), f

    x0, x1, a0, a1 = taps(dw, sw)
    y0, y1, b0, b1 = taps(dh, sh)
    rows = (img[:, x0] * a0[None, :] + img[:, x1] * a1[None, :]).astype(np.float32)
    return (rows[y0] * b0[:, None] + rows[y1] * b1[:, None]).astype(np.float32)
