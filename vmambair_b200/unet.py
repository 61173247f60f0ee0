"""Inference path of the U-Net around the OSS blocks on this library's kernels (SURVEY.md 8f rank 1).

Reference forward: MambaSISR6.forward, SRGAN/VmambaIR/archs/MambaSISR6_arch.py:610-642 (OverlapPatchEmbed :520-528, Downsample
:533-541, Upsample :544-553, reduce_chan_level* :590-600, SR tail :607,640 with Upsampler from archs/common.py:45-60) and the
Deraining / RealSR twins.  What the reference evaluates as conv -> PixelUnshuffle / PixelShuffle -> torch.cat -> 1x1 conv, each a
separate pass over HBM (and, on cuDNN, an NCHW<->NHWC transform either side of every conv), runs here as

  * vmb_conv3x3 with the (un)shuffle folded into the store, writing straight into its half of the decoder's concatenation buffer;
  * the last OSS block of each encoder level storing its result into the other half (fused.block_forward(out=...)), so no torch.cat;
  * reduce_chan_level* = vmb_pixlin over the concatenation buffer;
  * the SR tail's last conv reading the NHWC tensor the tail runs on, adding the nearest-upsampled input image and writing NCHW
    (the reference's conv + F.interpolate + add; here also the NHWC -> NCHW copy) in one kernel; Mamber32's output conv + inp_img
    the same way.

The two middle convs of the SR tail (96 -> 384 at 64x64 and 128x128: 22 + 87 GFLOP per 8-image batch, compute-bound) stay on the
library convolution (cuDNN's sm_90 kernels, NHWC) with this library's NHWC PixelShuffle between them.

Inference only: with gradients enabled the modules' nn.Conv2d / torch.cat path (autograd) is used.  set_mode("torch") restores that
path for inference as well (cross-checks, tests).
"""
from __future__ import annotations


import torch
import torch.nn as nn

from . import fused, ops

_MODE = "native"


def set_mode(mode: str) -> None:
    """'native' (default): this library's kernels; 'torch': nn.Conv2d / torch.cat (the round-1 path), for cross-checks"""
    global _MODE
    assert mode in ("native", "torch")
    _MODE = mode


def enabled(x: torch.Tensor) -> bool:
    return _MODE == "native" and x.is_cuda and not torch.is_grad_enabled() and x.dtype in fused._DTYPES and x.dim() == 4


def _dense_planes(x):
    return x if (x.stride(3) == 1 and x.stride(2) == x.shape[3]) else x.contiguous()


def _cached(conv: nn.Conv2d, dtype, kind):
    """kernel-layout weight (+ fp32 bias) of one nn.Conv2d, rebuilt when the parameter changes"""
    w = conv.weight
    ver = (dtype, w.device, w._version, w.data_ptr(), None if conv.bias is None else (conv.bias._version, conv.bias.data_ptr()))
    c = getattr(conv, "_vmb_conv", None)
    if c is None or c[0] != ver or c[1] != kind:
        if kind == "3x3":
            wp = ops.pack_conv3x3_weight(w, dtype)
        else:
            wp = ops.pad_weight(w.detach().reshape(w.shape[0], w.shape[1]).to(dtype))
        c = (ver, kind, wp, fused._f32(conv.bias))
        conv._vmb_conv = c
    return c[2], c[3]


def conv3x3(conv: nn.Conv2d, x, mode=ops.CONV_PLAIN, out=None, add=None, add_scale=1, nhwc=False):
    assert conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.padding == (1, 1) and conv.groups == 1 and \
        conv.dilation == (1, 1) and conv.padding_mode == "zeros"
    wp, bias = _cached(conv, x.dtype, "3x3")
    if not nhwc:
        x = _dense_planes(x)
    return ops.conv3x3(x, wp, bias, conv.out_channels, mode, out=out, add=add, add_scale=add_scale, nhwc=nhwc)


def conv1x1(conv: nn.Conv2d, x):
    """reduce_chan_level*: 1x1 conv over the (contiguous) concatenation buffer"""
    w, bias = _cached(conv, x.dtype, "1x1")
    B, K, H, W = x.shape
    return ops.pixlin(x.contiguous().view(B, K, H * W), w, bias).view(B, conv.out_channels, H, W)


def run_stage(stage: nn.Sequential, x, out=None):
    """a level's OSS blocks; the last one stores into `out` (a channel slice of a concatenation buffer) when given"""
    n = len(stage)
    for i, blk in enumerate(stage):
        x = blk(x, out=out) if (out is not None and i == n - 1) else blk(x)
    if out is not None and n == 0:
        out.copy_(x)
        return out
    return x


def lowres(net, e1, up_out=None):
    """everything below full resolution: e1 -> up2_1(d2)  (reference forward :612-633), e1 possibly a strided channel slice"""
    B, C1, H, W = e1.shape
    dt, dev = e1.dtype, e1.device
    cat2 = torch.empty((B, 4 * C1, H // 2, W // 2), dtype=dt, device=dev)   # [up3_2(d3) | e2]
    cat3 = torch.empty((B, 8 * C1, H // 4, W // 4), dtype=dt, device=dev)   # [up4_3(lat) | e3]
    x2 = conv3x3(net.down1_2.body[0], e1, ops.CONV_UNSHUFFLE2)
    e2 = run_stage(net.encoder_level2, x2, out=cat2[:, 2 * C1:])
    x3 = conv3x3(net.down2_3.body[0], e2, ops.CONV_UNSHUFFLE2)
    e3 = run_stage(net.encoder_level3, x3, out=cat3[:, 4 * C1:])
    x4 = conv3x3(net.down3_4.body[0], e3, ops.CONV_UNSHUFFLE2)
    lat = run_stage(net.latent, x4)
    conv3x3(net.up4_3.body[0], lat, ops.CONV_SHUFFLE2, out=cat3[:, :4 * C1])
    d3 = run_stage(net.decoder_level3, conv1x1(net.reduce_chan_level3, cat3))
    conv3x3(net.up3_2.body[0], d3, ops.CONV_SHUFFLE2, out=cat2[:, :2 * C1])
    d2 = run_stage(net.decoder_level2, conv1x1(net.reduce_chan_level2, cat2))
    return conv3x3(net.up2_1.body[0], d2, ops.CONV_SHUFFLE2, out=up_out)


def trunk(net, inp_img):
    """patch_embed ... refinement (reference forward :610-638) -> (features, patch-embed output)"""
    B, _, H, W = inp_img.shape
    assert H % 8 == 0 and W % 8 == 0, "the U-Net needs H, W multiples of 8 (tiling.padded_inference pads)"
    e1_in = conv3x3(net.patch_embed.proj, inp_img)
    C1 = e1_in.shape[1]
    cat1 = torch.empty((B, 2 * C1, H, W), dtype=e1_in.dtype, device=e1_in.device)  # [up2_1(d2) | e1]
    e1 = run_stage(net.encoder_level1, e1_in, out=cat1[:, C1:])
    if net._lowres_chains > 1 and B % net._lowres_chains == 0:
        from .engine import fork_join_batch
        cat1[:, :C1].copy_(fork_join_batch(lambda t: lowres(net, t), e1, net._lowres_chains, net._lowres_streams))
    else:
        lowres(net, e1, up_out=cat1[:, :C1])
    return run_stage(net.refinement, run_stage(net.decoder_level1, cat1)), e1_in
