"""NIQE, the no-reference metric of the reference's niqe.py (Deraining/basicsr/metrics), on deterministic sm_90a kernels
(csrc/niqe.cu): for restored images that have no ground truth, such as the real-world SR recipe's test set.

`niqe(img, crop_border=0, convert_to='y', quantize=False, params=None)` scores a batch without a host synchronisation and returns a
(B,) float64 CUDA tensor.  It takes the batches `metrics.psnr_ssim` takes: (B, H, W, C) uint8 / uint16 / float32 / float64 BGR CUDA
tensors (C = 1 or 3), or with quantize=True (B, 3, H, W) float32 / bf16 / fp16 RGB network outputs read through tensor2img.
convert_to: 'y' (to_y_channel, bit for bit as metrics.to_y_channel), 'gray' (cv2's BGR2GRAY in float32; C = 3) or None (a one-channel
image's values as they are, the reference's input_order='HW').  `niqe_features(...)` returns the (B, blocks, 36) float64 features
instead, the reference's `distparam`: row w * nbh + h for block (h, w), scale 1's 18 features then scale 2's.

`calculate_niqe(img, crop_border, input_order='HWC', convert_to='y', params=None)` is the drop-in, on a numpy image as the reference
takes it; it returns the reference's (1, 1) float64 ndarray.

A call is three launches (the r(gamma) table is built once per device): the plane cut to whole 96 x 96 blocks and its half, the
features of every block at both scales, the score of every image.  Each image's result does not depend on the batch it is in.

Conventions kept from the reference: the float32 cast first; the crop, then the cut to whole blocks, before any filtering (the 7 x 7
window replicates the cut plane's edges); MSCN values as scipy stores them (each filter summed in float64, rounded once to float32);
rolls circular within a block; alpha = 0.2 for a block whose distribution has no negative or no positive value (np.argmin of an
all-NaN array), NaN betas, and the covariance over the NaN-free rows only.  Deviations: the half plane is the float32 2 x 2 mean
((a + b) + (c + d)) * 0.25 of img / 255, times 255, where cv2's INTER_LINEAR resize differs by up to 2 ulp; the distribution
statistics are float64 sums (the reference's are float32 means), which moves a score by ~1e-7 relative, and an alpha by one table
step now and then; the score solves with a Cholesky factor instead of pinv; 'gray' is (B .114 + G .587) + R .299 in float32, which
can differ from cv2's by an ulp.  Where the reference raises, `niqe` gives NaN, and `calculate_niqe` raises np.linalg.LinAlgError
(fewer than two NaN-free blocks) or ValueError (no whole block after the crop; the reference's cv2.error).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib, metrics, ops

BLOCK = _lib.NIQE_BLOCK
DEFAULT_PARAMS = os.path.join("basicsr", "metrics", "niqe_pris_params.npz")


class NiqeParams:
    """The pristine model: mu (36,), cov (36, 36) and the 7 x 7 Gaussian window, float64 on the host; mu and cov are copied to a
    device once, on first use there."""

    def __init__(self, mu, cov, window):
        self.mu = np.asarray(mu, dtype=np.float64).reshape(-1)
        self.cov = np.ascontiguousarray(cov, dtype=np.float64)
        self.window = np.ascontiguousarray(window, dtype=np.float64)
        if self.mu.shape != (36,) or self.cov.shape != (36, 36) or self.window.shape != (7, 7):
            raise ValueError(f"NIQE parameters must be mu (1, 36), cov (36, 36) and a (7, 7) window, got {self.mu.shape}, "
                             f"{self.cov.shape}, {self.window.shape}")
        self._dev = {}

    def on(self, device):
        """-> (mu, cov) float64 tensors on `device`"""
        if device not in self._dev:
            self._dev[device] = (torch.from_numpy(self.mu).to(device), torch.from_numpy(self.cov).to(device))
        return self._dev[device]


_LOADED = {}
_TABLES = {}


def load_params(path=None):
    """The pristine parameters (niqe_pris_params.npz: mu_pris_param, cov_pris_param, gaussian_window) from `path`, or without one from
    basicsr/metrics/niqe_pris_params.npz under the working directory, where the reference reads them.  Cached per file."""
    if path is not None and os.path.isfile(path):
        f = path
    elif path is None and os.path.isfile(DEFAULT_PARAMS):
        f = DEFAULT_PARAMS
    else:
        raise FileNotFoundError(f"NIQE: no pristine parameters: path {path!r} is not a file, and the reference's {DEFAULT_PARAMS} is "
                                f"not under {os.getcwd()}; pass path=<niqe_pris_params.npz>")
    key = os.path.abspath(f)
    if key not in _LOADED:
        with np.load(f) as z:
            _LOADED[key] = NiqeParams(z["mu_pris_param"], z["cov_pris_param"], z["gaussian_window"])
    return _LOADED[key]


def _table(device):
    """r(gamma) of estimate_aggd_param, (9801,) float64, built once per device"""
    if device not in _TABLES:
        _TABLES[device] = ops.niqe_table(device)
    return _TABLES[device]


def _convert(convert_to, channels):
    if convert_to not in ("y", "gray", None):
        raise ValueError(f"convert_to must be 'y', 'gray' or None, got {convert_to!r}")
    if convert_to == "gray" and channels != 3:
        raise ValueError(f"convert_to='gray' takes 3-channel BGR images, got {channels} channel(s)")
    if convert_to is None and channels != 1:
        raise ValueError(f"convert_to=None takes one-channel images, got {channels} channels")
    return convert_to


def _run(v, crop_border, convert_to, params, planes=False):
    """the NIQE of every image of view v -> (features (B, blocks, 36), scores (B,)); planes=True: a dict with the plane, half plane,
    both MSCN planes and the table as well"""
    B, H, W, C = v.shape
    convert = _convert(convert_to, C)
    c = metrics._check_crop(crop_border)
    hc, wc = max(H - 2 * c, 0) // BLOCK * BLOCK, max(W - 2 * c, 0) // BLOCK * BLOCK
    params = load_params() if params is None else params
    dev = v.t.device
    mu, cov = params.on(dev)
    out = {}
    if hc and wc:
        src = ops.metric_src(v.t, v.offset + c * v.strides[1] + c * v.strides[2], v.strides, v.quantize)
        table = _table(dev)
        plane, half = ops.niqe_prep(v.t, src, B, hc, wc, C, convert)
        r = ops.niqe_features(plane, half, table, params.window.reshape(-1).tolist(), mscn=planes)
        feats, m1, m2 = r if planes else (r, None, None)
        out.update(plane=plane, half=half, mscn=m1, mscn_half=m2, table=table)
    else:
        feats = torch.empty((B, 0, _lib.NIQE_FEATURES), dtype=torch.float64, device=dev)
    score = ops.niqe_score(feats, mu, cov)
    if planes:
        out.update(features=feats, score=score)
        return out
    return feats, score


def niqe(img, crop_border=0, convert_to="y", quantize=False, params=None):
    """(B,) float64 CUDA tensor: the NIQE score of each image of the batch (lower is better); NaN where the reference raises.  No host
    synchronisation.  params: a NiqeParams (load_params); None: load_params()."""
    return _run(metrics._view(img, quantize, "niqe"), crop_border, convert_to, params)[1]


def niqe_features(img, crop_border=0, convert_to="y", quantize=False, params=None):
    """(B, blocks, 36) float64 CUDA tensor: the reference's distparam of each image (the arguments are niqe's)"""
    return _run(metrics._view(img, quantize, "niqe_features"), crop_border, convert_to, params)[0]


def calculate_niqe(img, crop_border, input_order="HWC", convert_to="y", params=None):
    """niqe.py's calculate_niqe: img a numpy (H, W), (H, W, C) or (C, H, W) image in [0, 255], BGR -> (1, 1) float64 ndarray.
    input_order 'HW' takes a 2-D plane as it is; 'HWC' / 'CHW' convert it with convert_to ('y' or 'gray')."""
    if not isinstance(img, np.ndarray):
        raise TypeError(f"calculate_niqe: expected a numpy array, got {type(img).__name__}")
    if input_order not in ("HW", "HWC", "CHW"):
        raise ValueError(f"Wrong input_order {input_order}. Supported input_orders are 'HW', 'HWC' and 'CHW'")
    if convert_to not in ("y", "gray"):
        raise ValueError(f"convert_to must be 'y' or 'gray', got {convert_to!r}")
    dev = torch.device("cuda", torch.cuda.current_device())
    if input_order == "HW":
        if img.ndim != 2:
            raise ValueError(f"input_order='HW' takes a 2-D image, got shape {img.shape}")
        v, convert_to = metrics._device_image(img, "HWC", dev), None
    else:
        v = metrics._device_image(img, input_order, dev)
    feats, score = _run(v, crop_border, convert_to, params)
    if feats.shape[1] == 0:
        raise ValueError(f"calculate_niqe: a {v.shape[1]} x {v.shape[2]} image with crop_border={crop_border} has no whole "
                         f"{BLOCK} x {BLOCK} block")
    feats, score = feats[0].cpu().numpy(), score.cpu().numpy()
    if int((~np.isnan(feats).any(axis=1)).sum()) < 2:
        raise np.linalg.LinAlgError("SVD did not converge: fewer than two blocks have NaN-free features")
    return score.reshape(1, 1)


__all__ = ["NiqeParams", "calculate_niqe", "load_params", "niqe", "niqe_features"]
