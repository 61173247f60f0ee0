"""Torch restatement of DISTS (RealSR/Metric/dists.py's class) as written out in vmambair_b200.dists (test infrastructure), in any
dtype and on any device, for the drop-in to be checked against.

  features of x: x itself, then relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 of (x - mean) / std through VGG16, with L2 pooling
  between the blocks (sqrt(depthwise 3 x 3 [.25 .5 .25]^T [.25 .5 .25] conv of f^2, stride 2, padding 1, + 1e-12));
  per image and channel mu, var = mean((f - mu)^2), cov = mean(f0 f1) - mu0 mu1, S1 = (2 mu0 mu1 + 1e-6) / (mu0^2 + mu1^2 + 1e-6),
  S2 = (2 cov + 1e-6) / (var0 + var1 + 1e-6); score = 1 - sum_c (alpha_c S1_c + beta_c S2_c) / (sum alpha + sum beta).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.lpips_ref import convs_from_state_dict, vgg16_features

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
TAPS = (0.25, 0.5, 0.25)


def l2pool(f):
    t = torch.tensor(TAPS, dtype=f.dtype, device=f.device)
    k = (t[:, None] * t[None, :]).expand(f.shape[1], 1, 3, 3)
    return torch.sqrt(F.conv2d(f * f, k, stride=2, padding=1, groups=f.shape[1]) + 1e-12)


def features(convs, x):
    mean = torch.tensor(MEAN).to(x.device, x.dtype).view(1, 3, 1, 1)  # the module's float32 buffers
    std = torch.tensor(STD).to(x.device, x.dtype).view(1, 3, 1, 1)
    return [x] + vgg16_features(convs, (x - mean) / std, l2pool)


def dists(convs, alpha, beta, x, y, batch_average=False):
    """-> the (B,) scores (0-dim at B = 1; their mean with batch_average) in x's dtype; alpha, beta: 1475 weights"""
    alpha = alpha.reshape(-1).to(x.device, x.dtype)
    beta = beta.reshape(-1).to(x.device, x.dtype)
    s1, s2 = [], []
    for a, b in zip(features(convs, x), features(convs, y)):
        m0, m1 = a.mean([2, 3]), b.mean([2, 3])
        v0 = ((a - m0[..., None, None]) ** 2).mean([2, 3])
        v1 = ((b - m1[..., None, None]) ** 2).mean([2, 3])
        cov = (a * b).mean([2, 3]) - m0 * m1
        s1.append((2 * m0 * m1 + 1e-6) / (m0 ** 2 + m1 ** 2 + 1e-6))
        s2.append((2 * cov + 1e-6) / (v0 + v1 + 1e-6))
    s1, s2 = torch.cat(s1, 1), torch.cat(s2, 1)
    score = 1 - ((s1 * alpha).sum(1) + (s2 * beta).sum(1)) / (alpha.sum() + beta.sum())
    return score.mean() if batch_average else score.squeeze()


def dists_from_state_dict(sd, x, y, batch_average=False):
    """dists() with the convolutions, alpha and beta of a DISTS state_dict, in x's dtype and on its device"""
    convs = convs_from_state_dict(sd, "stage{slice}.{index}", x.dtype, x.device)
    return dists(convs, sd["alpha"], sd["beta"], x, y, batch_average)


def feature_sums(convs, x):
    """per feature of x: (sum, sum of squares), a (6, 2) tensor in x's dtype"""
    return torch.stack([torch.stack([f.sum(), (f * f).sum()]) for f in features(convs, x)])
