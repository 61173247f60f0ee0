"""LPIPS with the VGG trunk, the metric both recipes' metric.sh score with first (RealSR/Metric/LPIPS.py): a drop-in for
`lpips.LPIPS(net='vgg')` (lpips 0.1.x, version '0.1') on deterministic sm_90a kernels (csrc/percep_metrics.cu).

The module holds lpips's state (`scaling_layer.shift|scale`, torchvision's VGG16 features up to relu5_3 as `net.slice1..5`, the
lin weights `lin0..4.model.1.weight` and their `lins.0..4` aliases) and its forward never calls the sub-modules.  Both images of
each pair run as one 2B batch: one launch prepares it (the optional 2 v - 1 and the scaling layer), each convolution is one cuDNN
call (torch's TF32 flag applies), the ReLUs and max-pools run on vmb_percep_stage, and at each of the five feature layers one kernel
reads the conv output once and writes the per-CTA partials of sum_c w_c (f0 / |f0| - f1 / |f1|)^2; one CTA adds them up.  No host
synchronisation, no atomics: a call is bitwise reproducible and can be captured in a CUDA graph.

`calculate_lpips(img_restored, img_gt, model)` is Metric/LPIPS.py's loop body, batched: uint8 BGR images go to the GPU as they
are, and the script's conversion (/ 255., BGR to RGB, normalize(.5, .5)) happens in the preparation kernel.

Deviations: there is no backward (an input that requires grad raises NotImplementedError); inputs are CUDA float32 (N, 3, H, W)
with H, W >= 16; net='alex' / 'squeeze', lpips=False, spatial=True, version='0.0' and pnet_tune=True raise NotImplementedError.
"""
from __future__ import annotations

import importlib.util
import os

import torch
from torch import nn

from . import _pmetric, ops
from .perceptual import _conv

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))  # torchvision indices of net.slice1 .. slice5
MIN_HW = 16  # four 2 x 2 max-pools before relu5_3


class ScalingLayer(nn.Module):
    """lpips's input scaling, (v - shift) / scale per channel (buffers only; the kernels apply it)"""

    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.Tensor(SHIFT)[None, :, None, None])
        self.register_buffer("scale", torch.Tensor(SCALE)[None, :, None, None])


class VGG16Slices(nn.Module):
    """lpips's pretrained_networks.vgg16 state: torchvision's vgg16 features 0..29 in five Sequentials under their indices"""

    def __init__(self, features):
        super().__init__()
        for k, (lo, hi) in enumerate(SLICES, 1):
            s = nn.Sequential()
            for i in range(lo, hi):
                s.add_module(str(i), features[i])
            setattr(self, f"slice{k}", s)

    def module(self, i):
        k = next(k for k, (lo, hi) in enumerate(SLICES, 1) if lo <= i < hi)
        return getattr(self, f"slice{k}")[i - SLICES[k - 1][0]]


class NetLinLayer(nn.Module):
    """lpips's lin layer: Dropout (the identity in eval mode) and a bias-free 1 x 1 convolution C -> 1"""

    def __init__(self, chn_in, use_dropout=True):
        super().__init__()
        layers = ([nn.Dropout()] if use_dropout else []) + [nn.Conv2d(chn_in, 1, 1, stride=1, padding=0, bias=False)]
        self.model = nn.Sequential(*layers)


def lpips_package_weights(version="0.1", net="vgg"):
    """weights/v<version>/<net>.pth of an installed lpips package (found without importing it), or None"""
    spec = importlib.util.find_spec("lpips")
    if spec is None or spec.origin is None:
        return None
    return os.path.join(os.path.dirname(spec.origin), "weights", f"v{version}", f"{net}.pth")


def lin_weights_path(model_path):
    """the file the lin weights are read from: model_path, else the lpips package's weights/v0.1/vgg.pth; never downloaded"""
    pkg = lpips_package_weights()
    if model_path is not None and os.path.isfile(model_path):
        return model_path
    if model_path is None and pkg is not None and os.path.isfile(pkg):
        return pkg
    where = pkg if pkg is not None else "<lpips package>/weights/v0.1/vgg.pth (lpips is not installed)"
    raise FileNotFoundError(f"LPIPS: no lin weights: model_path {model_path!r} is not a file, and the default is the lpips package's "
                            f"{where}; pass model_path=<vgg.pth>, or pretrained=False (nothing is downloaded)")


class LPIPS(nn.Module):
    """lpips.LPIPS(net='vgg') (version 0.1).

    Args (lpips's):
        pretrained (bool): load the lin weights from model_path, or without one from the installed lpips package's
            weights/v0.1/vgg.pth (FileNotFoundError naming both when neither exists; never downloaded).  False: lpips's random lins.
        net (str): 'vgg' or 'vgg16'.  version (str): '0.1'.  lpips (bool): True.  spatial (bool): False.
        pnet_rand (bool): False loads the VGG16 trunk through perceptual.find_weights('vgg16'); True keeps torchvision's random one.
        pnet_tune (bool): False.  use_dropout (bool): lpips's lin layout (model.0 Dropout, model.1 conv; False: model.0 conv).
        model_path (str): the lin weights file.  eval_mode (bool), verbose (bool): as lpips.

    forward(in0, in1, retPerLayer=False, normalize=False) -> (N, 1, 1, 1) fp32, and with retPerLayer (val, [res_k]).  in0, in1:
    CUDA float32 (N, 3, H, W) of one shape, H, W >= 16, in [-1, 1] (normalize=True: in [0, 1])."""

    def __init__(self, pretrained=True, net="vgg", version="0.1", lpips=True, spatial=False, pnet_rand=False, pnet_tune=False,
                 use_dropout=True, model_path=None, eval_mode=True, verbose=True):
        super().__init__()
        if net not in ("vgg", "vgg16"):
            raise NotImplementedError(f"LPIPS: net={net!r} is not implemented; only the VGG trunk (net='vgg') is")
        for bad, what in ((not lpips, "lpips=False (the unweighted baseline)"), (spatial, "spatial=True"),
                          (version != "0.1", f"version={version!r}"), (pnet_tune, "pnet_tune=True (no gradients)")):
            if bad:
                raise NotImplementedError(f"LPIPS: {what} is not implemented")
        self.pnet_type, self.pnet_tune, self.pnet_rand = net, pnet_tune, pnet_rand
        self.spatial, self.lpips, self.version = spatial, lpips, version
        self.scaling_layer = ScalingLayer()
        self.chns = list(_pmetric.CHANNELS)
        self.L = len(self.chns)
        self.net = VGG16Slices(_pmetric.vgg16_features(None if pnet_rand else "auto", "LPIPS"))
        for p in self.net.parameters():
            p.requires_grad = False
        for k, c in enumerate(self.chns):
            setattr(self, f"lin{k}", NetLinLayer(c, use_dropout=use_dropout))
        self.lins = nn.ModuleList([getattr(self, f"lin{k}") for k in range(self.L)])
        if pretrained:
            path = lin_weights_path(model_path)
            if verbose:
                print(f"Loading model from: {path}")
            self.load_state_dict(torch.load(path, map_location="cpu", weights_only=True), strict=False)
        if eval_mode:
            self.eval()

    def _score(self, t, src0, src1, B, H, W, normalize):
        """-> (val (B,), per-layer values (5, B)) of the prepared pair sources; t: a tensor on their device"""
        with torch.no_grad(), torch.autocast("cuda", enabled=False):
            sl = self.scaling_layer
            h = ops.pmetric_prep(t, src0, src1, B, H, W, "lpips", sl.shift, sl.scale, normalize=normalize)
            ctas, hws, offsets, hh, ww = [], [], [], H, W
            for _ in range(self.L):
                offsets.append(B * sum(ctas))
                ctas.append(ops.lpips_layer_ctas(B, hh, ww))
                hws.append(hh * ww)
                hh, ww = hh // 2, ww // 2
            partial = torch.empty(B * sum(ctas), dtype=torch.float32, device=t.device)
            for w, b, feat in _pmetric.conv_plan(self.net.module):
                y = _conv(h, w, b)
                if feat is None:
                    ops.percep_stage(y, True, False, [0, 0, 0], [None] * 3, "l1", False)
                    h = y
                    continue
                lin = self.lins[feat].model[-1].weight
                ops.lpips_layer(y, lin, partial[offsets[feat]:offsets[feat] + B * ctas[feat]])
                if feat + 1 < self.L:
                    h = ops.percep_stage(y, True, True, [0, 0, 0], [None] * 3, "l1", False)[0]
            return ops.lpips_final(partial, offsets, ctas, hws, B)

    def _device(self):
        return self.net.slice1[0].weight.device

    def forward(self, in0, in1, retPerLayer=False, normalize=False):
        _pmetric.check_no_grad("LPIPS", in0, in1)
        src0, src1, B, H, W = _pmetric.float_sources(in0, in1, self._device(), "LPIPS", MIN_HW)
        val, res = self._score(in0, src0, src1, B, H, W, normalize)
        val = val.view(B, 1, 1, 1)
        if retPerLayer:
            return val, [r.view(B, 1, 1, 1) for r in res]
        return val


def calculate_lpips(img_restored, img_gt, model):
    """Metric/LPIPS.py's per-image value, lpips(img_restored, img_gt) after the script's conversion (/ 255., BGR -> RGB,
    normalize(mean=.5, std=.5)), done on the GPU in the preparation kernel.

    img_restored, img_gt: (H, W, 3) uint8 BGR numpy images as cv2.imread returns them -> a Python float; or (B, H, W, 3) uint8 BGR
    CUDA tensors -> a (B,) float32 CUDA tensor, without a host synchronisation.  model: an LPIPS on the GPU."""
    keep, src0, src1, B, H, W, host = _pmetric.u8_sources(img_restored, img_gt, model._device(), "calculate_lpips", MIN_HW)
    val, _ = model._score(keep[0], src0, src1, B, H, W, False)
    return float(val[0].item()) if host else val


__all__ = ["LPIPS", "calculate_lpips"]
