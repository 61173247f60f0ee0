"""DISTS, the structure and texture similarity the reference ships next to LPIPS: a drop-in for the `DISTS` class of
RealSR/Metric/dists.py (identical in SRGAN/) on deterministic sm_90a kernels (csrc/percep_metrics.cu).

The module has the reference's structure and state_dict (`alpha`, `beta`, `mean`, `std`, `stage1..5` with torchvision's VGG16
layers under their indices and an `L2pooling` with its `filter` buffer at 4 / 9 / 16 / 23), so a strict load works both ways, and a
seeded construction draws the reference's `alpha` and `beta`.  Its forward never calls the sub-modules.  Both images of each pair
run as one 2B batch: one launch normalises it and sums the statistics of the raw input, each convolution is one cuDNN call
(torch's TF32 flag applies), the ReLUs without a feature run on vmb_percep_stage, and at each of the five feature layers one
kernel reads the conv output once, sums each channel's statistics in float64 and writes the L2-pooled input of the next
convolution.  One CTA forms S1 and S2 per channel and the weighted score.  No host synchronisation, no atomics.

`calculate_dists(img_restored, img_gt, model)` is Metric/dists.py's loop body, batched, on cv2-style uint8 BGR images.

Deviations: no gradients (require_grad=True raises NotImplementedError); inputs are CUDA float32 (B, 3, H, W); the means,
variances and covariances are float64 sums (the reference's covariance is float32 E[xy] - E[x]E[y]); the weights come from local
files (weights_path, then Metric/DISTS/DISTS_pytorch/weights.pt under the working directory; never a download).
"""
from __future__ import annotations

import os

import torch
from torch import nn

from . import _pmetric, ops
from .perceptual import _conv

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
CHNS = (3, 64, 128, 256, 512, 512)
STAGES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))  # torchvision indices of stage1 .. stage5; 4 / 9 / 16 / 23 are L2pooling
TAPS = (0.25, 0.5, 0.25)  # L2pooling's filter is their outer product: hanning(5)[1:-1], normalised
DEFAULT_WEIGHTS = os.path.join("Metric", "DISTS", "DISTS_pytorch", "weights.pt")


class L2pooling(nn.Module):
    """The reference's L2 pooling state: a depthwise 3 x 3 `filter` buffer, outer(TAPS, TAPS) per channel.  The kernels apply
    sqrt(conv2d(x^2, filter, stride 2, padding 1) + 1e-12) with these taps."""

    def __init__(self, filter_size=5, stride=2, channels=None, pad_off=0):
        super().__init__()
        if filter_size != 5 or stride != 2:
            raise NotImplementedError("L2pooling: only the reference's filter_size=5, stride=2")
        self.padding, self.stride, self.channels = 1, stride, channels
        t = torch.tensor(TAPS)
        self.register_buffer("filter", (t[:, None] * t[None, :]).expand(channels, 1, 3, 3).contiguous())


def _weights_file(weights_path):
    if weights_path is not None and os.path.isfile(weights_path):
        return weights_path
    if weights_path is None and os.path.isfile(DEFAULT_WEIGHTS):
        return DEFAULT_WEIGHTS
    raise FileNotFoundError(f"DISTS: no alpha / beta weights: weights_path {weights_path!r} is not a file, and the recipes' "
                            f"{DEFAULT_WEIGHTS} is not under {os.getcwd()}; pass weights_path=<weights.pt>, or load_weights=False")


class DISTS(nn.Module):
    """RealSR/Metric/dists.py's DISTS.

    Args:
        load_weights (bool): read `alpha` and `beta` from weights_path, or without one from Metric/DISTS/DISTS_pytorch/weights.pt
            under the working directory (FileNotFoundError naming both).  False: the reference's random N(0.1, 0.01) draws.
        weights_path (str): the DISTS weights file (a dict with 'alpha' and 'beta').
        vgg_weights: the VGG16 trunk, as PerceptualLoss's `weights`: 'auto' (experiments/pretrained_models/vgg16-397923af.pth, then
            the torch hub cache; never downloaded), the path of a torchvision VGG16 state_dict, or None (torchvision's random one).

    forward(x, y, require_grad=False, batch_average=False) -> 1 - the weighted similarity, (B,) fp32 squeezed (0-dim at B = 1), or
    its mean with batch_average.  x, y: CUDA float32 (B, 3, H, W) of one shape, in [0, 1]."""

    def __init__(self, load_weights=True, weights_path=None, vgg_weights="auto"):
        super().__init__()
        import torchvision
        features = torchvision.models.vgg16(weights=None).features  # first, so that a seeded construction draws the reference's alpha / beta
        for k, (lo, hi) in enumerate(STAGES, 1):
            s = nn.Sequential()
            for i in range(lo, hi):
                s.add_module(str(i), L2pooling(channels=CHNS[k - 1]) if k > 1 and i == lo else features[i])
            setattr(self, f"stage{k}", s)
        for p in self.parameters():
            p.requires_grad = False
        self.register_buffer("mean", torch.tensor(MEAN).view(1, -1, 1, 1))
        self.register_buffer("std", torch.tensor(STD).view(1, -1, 1, 1))
        self.chns = list(CHNS)
        self.register_parameter("alpha", nn.Parameter(torch.randn(1, sum(CHNS), 1, 1)))
        self.register_parameter("beta", nn.Parameter(torch.randn(1, sum(CHNS), 1, 1)))
        self.alpha.data.normal_(0.1, 0.01)
        self.beta.data.normal_(0.1, 0.01)
        if vgg_weights is not None:
            loaded = _pmetric.vgg16_features(vgg_weights, "DISTS")
            with torch.no_grad():
                for i in _pmetric.CONVS:
                    self._module(i).weight.copy_(loaded[i].weight)
                    self._module(i).bias.copy_(loaded[i].bias)
        if load_weights:
            w = torch.load(_weights_file(weights_path), map_location="cpu", weights_only=True)
            self.alpha.data = w["alpha"]
            self.beta.data = w["beta"]

    def _module(self, i):
        k = next(k for k, (lo, hi) in enumerate(STAGES, 1) if lo <= i < hi)
        return getattr(self, f"stage{k}")[i - STAGES[k - 1][0]]

    def _device(self):
        return self.stage1[0].weight.device

    def _score(self, t, src0, src1, B, H, W, batch_average):
        """-> (scores (B,), mean or None) of the pair sources; t: a tensor on their device"""
        if self.alpha.numel() != sum(CHNS) or self.beta.numel() != sum(CHNS):
            raise ValueError(f"DISTS: alpha and beta must have {sum(CHNS)} elements")
        with torch.no_grad(), torch.autocast("cuda", enabled=False):
            sizes = [(H, W), (H, W)]  # feature k's plane: the input, relu1_2 at H x W, then ceil halves
            for _ in range(4):
                h, w = sizes[-1]
                sizes.append(((h + 1) // 2, (w + 1) // 2))
            tiles = [ops.pmetric_tiles(B * c, h * w if k == 0 else ((h + 1) // 2) * ((w + 1) // 2))
                     for k, (c, (h, w)) in enumerate(zip(CHNS, sizes))]
            offsets = [0]
            for c, t_k in zip(CHNS, tiles):
                offsets.append(offsets[-1] + B * c * t_k)
            stats = torch.empty(offsets[-1] * 5, dtype=torch.float64, device=t.device)
            view = lambda k: stats[offsets[k] * 5:offsets[k + 1] * 5]
            alpha, beta = self.alpha.detach().reshape(-1).contiguous(), self.beta.detach().reshape(-1).contiguous()
            h = ops.pmetric_prep(t, src0, src1, B, H, W, "dists", self.mean, self.std, stats=view(0))
            for w, b, feat in _pmetric.conv_plan(self._module):
                y = _conv(h, w, b)
                if feat is None:
                    ops.percep_stage(y, True, False, [0, 0, 0], [None] * 3, "l1", False)
                    h = y
                else:
                    h = ops.dists_layer(y, view(feat + 1), pool=feat + 1 < len(CHNS) - 1)
            return ops.dists_final(stats, alpha, beta, offsets[:-1], CHNS, tiles, [h * w for h, w in sizes], B, batch_average)

    def forward(self, x, y, require_grad=False, batch_average=False):
        if require_grad:
            raise NotImplementedError("DISTS: require_grad=True is not implemented (no gradients through the metric)")
        _pmetric.check_no_grad("DISTS", x, y)
        src0, src1, B, H, W = _pmetric.float_sources(x, y, self._device(), "DISTS", 1)
        score, mean = self._score(x, src0, src1, B, H, W, batch_average)
        return mean if batch_average else score.squeeze()


def calculate_dists(img_restored, img_gt, model):
    """Metric/dists.py's per-image score, model(ref, dist) with ref the ground truth, after the script's ToTensor (/ 255), done on
    the GPU in the preparation kernel.

    img_restored, img_gt: (H, W, 3) uint8 BGR numpy images as cv2.imread returns them -> a Python float; or (B, H, W, 3) uint8 BGR
    CUDA tensors -> a (B,) float32 CUDA tensor, without a host synchronisation.  model: a DISTS on the GPU."""
    keep, src_gt, src_out, B, H, W, host = _pmetric.u8_sources(img_gt, img_restored, model._device(), "calculate_dists", 1)
    score, _ = model._score(keep[0], src_gt, src_out, B, H, W, False)
    return float(score[0].item()) if host else score


__all__ = ["DISTS", "calculate_dists"]
