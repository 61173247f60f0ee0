"""Torch restatement of LPIPS with the VGG trunk (lpips.LPIPS(net='vgg'), version 0.1) as written out in vmambair_b200.lpips
(test infrastructure), in any dtype and on any device, for the drop-in to be checked against.

  in0, in1 -> (2 v - 1 when normalize) -> (v - shift) / scale -> VGG16 features relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
  (3 x 3 convolutions with padding 1, ReLU, floor 2 x 2 max-pools between the blocks); per layer k f / (sqrt(sum_c f^2) + 1e-10),
  the squared difference, the bias-free 1 x 1 convolution C_k -> 1 with lin{k}'s weight and the mean over H x W; the sum over k.

Also the seeded VGG16 trunk the tests and tests/golden/make_golden_dists.py use (seeded_vgg16_convs).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

BLOCKS = (2, 2, 3, 3, 3)            # convolutions per VGG16 block; a feature after each block's last ReLU
CHANNELS = (64, 128, 256, 512, 512)
CONV_INDEX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)  # torchvision features index of each convolution
SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))


def seeded_vgg16_convs(seed):
    """the 13 (weight, bias) float32 pairs of a random VGG16 trunk: torch.randn in parameter order from a Generator seeded with
    `seed`, weights scaled by 1 / sqrt(fan_in), biases by 0.1 (non-zero)"""
    g = torch.Generator().manual_seed(seed)
    out, cin = [], 3
    for n, c in zip(BLOCKS, CHANNELS):
        for _ in range(n):
            w = torch.randn(c, cin, 3, 3, generator=g) / (cin * 9) ** 0.5
            b = 0.1 * torch.randn(c, generator=g)
            out.append((w, b))
            cin = c
    return out


def checksums(convs):
    """(sum, sum of squares) in float64 of every tensor of `convs`, weight then bias: a (26, 2) tensor"""
    return torch.tensor([[t.double().sum().item(), t.double().square().sum().item()] for wb in convs for t in wb], dtype=torch.float64)


def vgg16_features(convs, x, pool):
    """the five block features (after each block's last ReLU) of x through `convs`; pool(f) sits between the blocks"""
    feats, i = [], 0
    for k, n in enumerate(BLOCKS):
        if k > 0:
            x = pool(x)
        for _ in range(n):
            w, b = convs[i]
            x = F.relu(F.conv2d(x, w, b, padding=1))
            i += 1
        feats.append(x)
    return feats


def convs_from_state_dict(sd, fmt, dtype=torch.float64, device="cpu"):
    """the 13 (weight, bias) of a state_dict whose convolution i (torchvision index) is fmt.format(slice=k, index=i)"""
    out = []
    for i in CONV_INDEX:
        k = next(k for k, (lo, hi) in enumerate(SLICES, 1) if lo <= i < hi)
        key = fmt.format(slice=k, index=i)
        out.append((sd[key + ".weight"].to(device, dtype), sd[key + ".bias"].to(device, dtype)))
    return out


def lpips(convs, lins, shift, scale, in0, in1, normalize=False):
    """-> (val (N, 1, 1, 1), [res_k (N, 1, 1, 1)]) in in0's dtype; lins: the five (1, C_k, 1, 1) lin weights"""
    if normalize:
        in0, in1 = 2 * in0 - 1, 2 * in1 - 1
    dt = in0.dtype
    shift, scale = shift.to(in0.device, dt), scale.to(in0.device, dt)
    maxpool = lambda f: F.max_pool2d(f, 2, 2)
    f0 = vgg16_features(convs, (in0 - shift) / scale, maxpool)
    f1 = vgg16_features(convs, (in1 - shift) / scale, maxpool)
    res = []
    for a, b, w in zip(f0, f1, lins):
        a = a / (torch.sqrt(torch.sum(a ** 2, dim=1, keepdim=True)) + 1e-10)
        b = b / (torch.sqrt(torch.sum(b ** 2, dim=1, keepdim=True)) + 1e-10)
        res.append(F.conv2d((a - b) ** 2, w.to(in0.device, dt)).mean([2, 3], keepdim=True))
    val = res[0]
    for r in res[1:]:
        val = val + r
    return val, res


def lpips_from_state_dict(sd, in0, in1, normalize=False):
    """lpips() with the convolutions, lins and scaling of an LPIPS state_dict, in in0's dtype and on its device"""
    dt, dev = in0.dtype, in0.device
    convs = convs_from_state_dict(sd, "net.slice{slice}.{index}", dt, dev)
    lins = [next(v for k, v in sd.items() if k.startswith(f"lin{k_}.model.") and k.endswith(".weight")) for k_ in range(5)]
    return lpips(convs, lins, sd["scaling_layer.shift"], sd["scaling_layer.scale"], in0, in1, normalize)
