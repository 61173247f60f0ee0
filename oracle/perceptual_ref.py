"""Torch restatement of basicsr's PerceptualLoss (test infrastructure), in any dtype and on any device, for vmambair_b200.perceptual
to be checked against.

The network is torchvision's VGG `features` (in-place ReLUs, MaxPool2d(2, 2)) cut after the deepest requested layer, with the weights
of a vmambair_b200 PerceptualLoss state_dict.  The loss restates basicsr's VGGFeatureExtractor.forward and PerceptualLoss.forward:
(x + 1) / 2 when range_norm, (x - mean) / std when use_input_norm, each requested layer's output clone()d as it is produced, then
perceptual_weight * sum over the features in network order of criterion(x_k, gt_k) * w_k, with gt detached; l1 / l2 are
F.l1_loss / F.mse_loss (means), fro is torch.norm(x_k - gt_k, p='fro').
"""
from __future__ import annotations

import copy

import torch
import torch.nn.functional as F
import torchvision

from vmambair_b200.perceptual import layer_names

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def features_from_state_dict(sd, vgg_type, layer_weights):
    """torchvision's VGG `features` cut after the deepest layer of layer_weights, with the convolutions of a PerceptualLoss state_dict"""
    names = layer_names(vgg_type)
    cut = max(names.index(k) for k in layer_weights)
    feats = getattr(torchvision.models, vgg_type)(weights=None).features[:cut + 1]
    with torch.no_grad():
        for i, n in enumerate(names[:cut + 1]):
            if n.startswith("conv"):
                feats[i].weight.copy_(sd[f"vgg.vgg_net.{n}.weight"])
                feats[i].bias.copy_(sd[f"vgg.vgg_net.{n}.bias"])
    for p in feats.parameters():
        p.requires_grad_(False)
    return feats.eval()


def extract(feats, names, wanted, x, use_input_norm, range_norm):
    if range_norm:
        x = (x + 1) / 2
    if use_input_norm:
        mean = torch.tensor(MEAN, dtype=torch.float32).view(1, 3, 1, 1).to(x.device)
        std = torch.tensor(STD, dtype=torch.float32).view(1, 3, 1, 1).to(x.device)
        x = (x - mean) / std
    out = {}
    for key, layer in zip(names, feats):
        x = layer(x)
        if key in wanted:
            out[key] = x.clone()
    return out


def perceptual_loss(feats, vgg_type, layer_weights, x, gt, use_input_norm=True, range_norm=False, perceptual_weight=1.0,
                    criterion="l1"):
    """basicsr's PerceptualLoss(...)(x, gt)[0] on `feats` (features_from_state_dict), in x's dtype"""
    names = layer_names(vgg_type)
    fx = extract(feats, names, layer_weights, x, use_input_norm, range_norm)
    fg = extract(feats, names, layer_weights, gt.detach(), use_input_norm, range_norm)
    if perceptual_weight == 0:
        return None
    loss = 0
    for k in fx:
        if criterion == "fro":
            loss = loss + torch.norm(fx[k] - fg[k], p="fro") * layer_weights[k]
        elif criterion == "l1":
            loss = loss + F.l1_loss(fx[k], fg[k]) * layer_weights[k]
        else:
            loss = loss + F.mse_loss(fx[k], fg[k]) * layer_weights[k]
    return loss * perceptual_weight


def copy_to(feats, dtype):
    """a copy of `feats` in `dtype`"""
    return copy.deepcopy(feats).to(dtype)
