"""What LPIPS (lpips.py) and DISTS (dists.py) share: torchvision's VGG16 `features` with their weights, the convolution plan of the
trunk up to relu5_3, and the checks and device views of their two kinds of input (float32 NCHW, uint8 BGR images)."""
from __future__ import annotations

import numpy as np
import torch

from . import ops
from .perceptual import find_weights

# torchvision vgg16().features: index of each convolution, and of the ReLU after conv1_2, conv2_2, conv3_3, conv4_3, conv5_3 (the
# features both metrics read); a layer's slice ends after its ReLU
CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
FEATURE_RELUS = (3, 8, 15, 22, 29)
CHANNELS = (64, 128, 256, 512, 512)


def vgg16_features(weights, who):
    """torchvision's vgg16(weights=None).features, with `weights` loaded: 'auto' (perceptual.find_weights; never downloaded), the
    path of a torchvision VGG16 state_dict, or None (torchvision's random initialisation)"""
    import torchvision
    features = torchvision.models.vgg16(weights=None).features
    if weights == "auto":
        weights = find_weights("vgg16", who)
    if weights is not None:
        sd = torch.load(weights, map_location="cpu", weights_only=True)
        missing = [f"features.{k}" for k in features.state_dict() if f"features.{k}" not in sd]
        if missing:
            raise KeyError(f"{who}: {weights} lacks {', '.join(missing)}")
        features.load_state_dict({k: sd[f"features.{k}"] for k in features.state_dict()})
    return features


def conv_plan(module_of):
    """the trunk's 13 convolutions in order: (weight, bias, feature layer index or None); module_of(i) is the module at
    torchvision index i"""
    plan = []
    for i in CONVS:
        m = module_of(i)
        feat = FEATURE_RELUS.index(i + 1) if i + 1 in FEATURE_RELUS else None
        plan.append((m.weight, m.bias, feat))
    return plan


def float_sources(x, y, dev, who, min_hw):
    """checks a pair of (B, 3, H, W) float32 CUDA tensors on `dev` -> (src0, src1, B, H, W)"""
    for name, t in (("first input", x), ("second input", y)):
        if not isinstance(t, torch.Tensor) or t.dim() != 4 or t.shape[1] != 3:
            raise ValueError(f"{who}: the {name} must be a (B, 3, H, W) tensor, got {getattr(t, 'shape', type(t))}")
        if t.dtype != torch.float32:
            raise ValueError(f"{who}: the {name} must be float32, got {t.dtype}")
    if x.shape != y.shape:
        raise ValueError(f"{who}: the inputs' shapes differ: {tuple(x.shape)} and {tuple(y.shape)}")
    B, _, H, W = x.shape
    if B < 1 or H < min_hw or W < min_hw:
        raise ValueError(f"{who}: H and W must be at least {min_hw} (and B at least 1), got {tuple(x.shape)}")
    if not x.is_cuda or x.device != y.device or x.device != dev:
        raise ValueError(f"{who} runs on CUDA: the inputs are on {x.device} and {y.device}, the network on {dev}")
    return ops.pmetric_src(x, 0, x.stride()), ops.pmetric_src(y, 0, y.stride()), B, H, W


def _device_u8(img, dev, who):
    """a uint8 BGR image as cv2.imread returns it ((H, W, 3) numpy) or a (B, H, W, 3) uint8 CUDA tensor -> (B, H, W, 3) on dev"""
    if isinstance(img, np.ndarray):
        if img.ndim != 3 or img.shape[2] != 3 or img.dtype != np.uint8:
            raise ValueError(f"{who}: a numpy image must be (H, W, 3) uint8 BGR, got {img.shape} {img.dtype}")
        staged = torch.empty(img.shape, dtype=torch.uint8, pin_memory=True)
        staged.numpy()[...] = img
        return staged.to(dev, non_blocking=True).unsqueeze(0)
    if isinstance(img, torch.Tensor):
        if img.dim() != 4 or img.shape[3] != 3 or img.dtype != torch.uint8 or not img.is_cuda:
            raise ValueError(f"{who}: a tensor image batch must be (B, H, W, 3) uint8 BGR on CUDA, got {tuple(img.shape)} {img.dtype} "
                             f"on {img.device}")
        if img.device != dev:
            raise ValueError(f"{who}: the images are on {img.device}, the network on {dev}")
        return img
    raise TypeError(f"{who}: expected a numpy array or a torch tensor, got {type(img).__name__}")


def u8_sources(a, b, dev, who, min_hw):
    """-> (keep-alive tensors, src0, src1, B, H, W, both numpy) for two uint8 BGR images or batches (the RGB planes are read from
    channel 2 down)"""
    if isinstance(a, np.ndarray) != isinstance(b, np.ndarray):
        raise TypeError(f"{who}: pass two numpy images or two tensors")
    ta, tb = _device_u8(a, dev, who), _device_u8(b, dev, who)
    if ta.shape != tb.shape:
        raise ValueError(f"{who}: image shapes differ: {tuple(ta.shape)} and {tuple(tb.shape)}")
    B, H, W, _ = ta.shape
    if B < 1 or H < min_hw or W < min_hw:
        raise ValueError(f"{who}: H and W must be at least {min_hw} (and B at least 1), got {tuple(ta.shape)}")
    srcs = [ops.pmetric_src(t, 2 * t.stride(3), (t.stride(0), -t.stride(3), t.stride(1), t.stride(2))) for t in (ta, tb)]
    return (ta, tb), srcs[0], srcs[1], B, H, W, isinstance(a, np.ndarray)


def check_no_grad(who, *ts):
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in ts):
        raise NotImplementedError(f"{who} has no backward: score under torch.no_grad(), or pass inputs that do not require grad")
