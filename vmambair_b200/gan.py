"""The GAN stage of the RealSR / SRGAN recipes: drop-in `UNetDiscriminatorSN` and vanilla `GANLoss`.

`UNetDiscriminatorSN` (RealSR/VmambaIR/archs/discriminator_arch.py:19-67; the SRGAN copy is identical) builds its layers exactly as the
reference does (nn.Conv2d, torch.nn.utils.spectral_norm on conv1..conv8), so the state_dict, its keys and a seeded initialisation are
the reference's, and its `net_d_*.pth` files load with strict=True.  The forward never calls the sub-modules: the whole network is one
autograd Function.  The ten convolutions run on cuDNN (aten.convolution / convolution_backward with an output mask, so the G step
computes no parameter gradient and the D step no input gradient); everything between them is csrc/gan.cu:
  spectral norm of conv1..conv8 in one call (4 launches in train mode, 2 in eval), the decoder junctions up2(leaky(pre) [+ skip]),
  the encoder's in-place leaky ReLU, and on the way back the junctions' adjoint as a gather, the activation backward that adds the
  skip gradient on the fly, and dW_orig of all spectral-normalised weights in two launches.
No atomics and no host synchronisation: the forward and backward are bitwise reproducible, also under
torch.use_deterministic_algorithms(True), where the reference's bilinear backward raises.

Spectral norm follows torch.nn.utils.spectral_norm (dim 0, one power iteration, eps 1e-12): in train mode every forward advances
weight_u and weight_v in place, in eval mode sigma = u . (W v) with the stored u, v; the gradient treats u and v as constants.
"""
from __future__ import annotations

import torch
from torch import nn
from torch.nn.utils import spectral_norm

from . import fused_train, ops

_SN_LAYERS = [f"conv{k}" for k in range(1, 9)]
_STRIDE = {1: 2, 2: 2, 3: 2}  # conv1..conv3: 4 x 4, stride 2, padding 1; the others 3 x 3, stride 1, padding 1


def _conv(x, w, b, k):
    s = _STRIDE.get(k, 1)
    return torch.ops.aten.convolution(x, w, b, [s, s], [1, 1], [1, 1], False, [0, 0], 1).contiguous()


def _conv_bwd(g, x, w, k, mask, bias):
    s = _STRIDE.get(k, 1)
    return torch.ops.aten.convolution_backward(g, x, w, [w.shape[0]] if bias else None, [s, s], [1, 1], [1, 1], False, [0, 0], 1,
                                               mask)


def _dense(t):
    return None if t is None else t.contiguous()


class _Discriminator(torch.autograd.Function):
    """(cfg, x, conv0.weight, conv0.bias, conv9.weight, conv9.bias, conv1..8.weight_orig) -> logits (B, 1, H, W)"""

    @staticmethod
    def forward(ctx, cfg, x, w0, b0, w9, b9, *sn_w):
        dt, skip = cfg["dtype"], cfg["skip"]
        with torch.autocast("cuda", enabled=False):
            xin = x.to(dt).contiguous()
            w0c, b0c, w9c, b9c = (t.to(dt) for t in (w0, b0, w9, b9))
            wns, sigma, us, vs = ops.spectral_norm(list(sn_w), cfg["u"], cfg["v"], cfg["train"], dt)
            x0 = ops.gan_act(_conv(xin, w0c, b0c, 0))
            x1 = ops.gan_act(_conv(x0, wns[0], None, 1))
            x2 = ops.gan_act(_conv(x1, wns[1], None, 2))
            p3 = _conv(x2, wns[2], None, 3)
            u3 = ops.gan_up(p3)
            p4 = _conv(u3, wns[3], None, 4)
            u4 = ops.gan_up(p4, x2 if skip else None)
            p5 = _conv(u4, wns[4], None, 5)
            u5 = ops.gan_up(p5, x1 if skip else None)
            p6 = _conv(u5, wns[5], None, 6)
            x6 = ops.gan_act(p6, x0, out=torch.empty_like(p6)) if skip else ops.gan_act(p6)
            x7 = ops.gan_act(_conv(x6, wns[6], None, 7))
            x8 = ops.gan_act(_conv(x7, wns[7], None, 8))
            out = _conv(x8, w9c, b9c, 9)
        ctx.cfg = cfg
        ctx.sn_params = sn_w
        ctx.x_dtype = x.dtype
        ctx.save_for_backward(xin, w0c, w9c, x0, x1, x2, p3, u3, p4, u4, p5, u5, p6 if skip else x6, x6, x7, x8, sigma,
                              *wns, *us, *vs)
        return out

    @staticmethod
    def backward(ctx, go):
        cfg = ctx.cfg
        dt, skip = cfg["dtype"], cfg["skip"]
        need = ctx.needs_input_grad
        need_x = need[1]
        need_w0, need_b0, need_w9, need_b9 = need[2], need[3], need[4], need[5]
        need_sn = any(need[6:])
        saved = ctx.saved_tensors
        xin, w0c, w9c, x0, x1, x2, p3, u3, p4, u4, p5, u5, ref6, x6, x7, x8, sigma = saved[:17]
        wns, us, vs = saved[17:25], saved[25:33], saved[33:41]
        dwn = [None] * 8
        with torch.autocast("cuda", enabled=False):
            go = go.to(dt).contiguous()
            dx8, dw9, db9 = _conv_bwd(go, x8, w9c, 9, [True, need_w9, need_b9], True)
            g = ops.gan_act_bwd(_dense(dx8), x8)
            dx7, dwn[7], _ = _conv_bwd(g, x7, wns[7], 8, [True, need_sn, False], False)
            g = ops.gan_act_bwd(_dense(dx7), x7)
            dx6, dwn[6], _ = _conv_bwd(g, x6, wns[6], 7, [True, need_sn, False], False)
            dx6 = _dense(dx6)
            g = ops.gan_act_bwd(dx6, ref6, out=torch.empty_like(dx6) if skip else None)  # with skip, dx6 is also x0's skip gradient
            du5, dwn[5], _ = _conv_bwd(g, u5, wns[5], 6, [True, need_sn, False], False)
            g, dx1s = ops.gan_up_bwd(_dense(du5), p5, skip)
            du4, dwn[4], _ = _conv_bwd(g, u4, wns[4], 5, [True, need_sn, False], False)
            g, dx2s = ops.gan_up_bwd(_dense(du4), p4, skip)
            du3, dwn[3], _ = _conv_bwd(g, u3, wns[3], 4, [True, need_sn, False], False)
            g, _ = ops.gan_up_bwd(_dense(du3), p3, False)
            dx2, dwn[2], _ = _conv_bwd(g, x2, wns[2], 3, [True, need_sn, False], False)
            g = ops.gan_act_bwd(_dense(dx2), x2, dx2s)
            dx1, dwn[1], _ = _conv_bwd(g, x1, wns[1], 2, [True, need_sn, False], False)
            g = ops.gan_act_bwd(_dense(dx1), x1, dx1s)
            dx0, dwn[0], _ = _conv_bwd(g, x0, wns[0], 1, [True, need_sn, False], False)
            g = ops.gan_act_bwd(_dense(dx0), x0, dx6 if skip else None)
            dx, dw0, db0 = _conv_bwd(g, xin, w0c, 0, [need_x, need_w0, need_b0], True)
            sn_grads = [None] * 8
            if need_sn:
                bufs, direct = zip(*(fused_train._acc(p, torch.empty(p.shape, dtype=torch.float32, device=p.device))
                                     for p in ctx.sn_params))
                ops.spectral_norm_bwd([_dense(d) for d in dwn], list(ctx.sn_params), us, vs, sigma, bufs, direct)
                sn_grads = [None if d else b for b, d in zip(bufs, direct)]
        f32 = lambda t: None if t is None else t.float()
        return (None, None if dx is None else dx.to(ctx.x_dtype), f32(dw0), f32(db0), f32(dw9), f32(db9), *sn_grads)


class UNetDiscriminatorSN(nn.Module):
    """U-Net discriminator with spectral normalisation (Real-ESRGAN); drop-in for the reference class of the same name.

    Args:
        num_in_ch (int): channels of the input images.
        num_feat (int): channels of the first feature map. Default: 64.
        skip_connection (bool): add the encoder features to the decoder's. Default: True.

    The input must be a CUDA tensor of H, W multiples of 8; float32, or any dtype under torch.autocast("cuda", torch.bfloat16), where
    the activations are bf16 and spectral norm stays fp32."""

    def __init__(self, num_in_ch, num_feat=64, skip_connection=True):
        super().__init__()
        self.skip_connection = skip_connection
        norm = spectral_norm
        # the reference's construction order, so that a seeded initialisation draws the same values
        self.conv0 = nn.Conv2d(num_in_ch, num_feat, kernel_size=3, stride=1, padding=1)
        self.conv1 = norm(nn.Conv2d(num_feat, num_feat * 2, 4, 2, 1, bias=False))
        self.conv2 = norm(nn.Conv2d(num_feat * 2, num_feat * 4, 4, 2, 1, bias=False))
        self.conv3 = norm(nn.Conv2d(num_feat * 4, num_feat * 8, 4, 2, 1, bias=False))
        self.conv4 = norm(nn.Conv2d(num_feat * 8, num_feat * 4, 3, 1, 1, bias=False))
        self.conv5 = norm(nn.Conv2d(num_feat * 4, num_feat * 2, 3, 1, 1, bias=False))
        self.conv6 = norm(nn.Conv2d(num_feat * 2, num_feat, 3, 1, 1, bias=False))
        self.conv7 = norm(nn.Conv2d(num_feat, num_feat, 3, 1, 1, bias=False))
        self.conv8 = norm(nn.Conv2d(num_feat, num_feat, 3, 1, 1, bias=False))
        self.conv9 = nn.Conv2d(num_feat, 1, 3, 1, 1)

    def forward(self, x):
        if not x.is_cuda:
            raise ValueError("UNetDiscriminatorSN runs on CUDA tensors only")
        if x.dim() != 4 or x.shape[2] % 8 or x.shape[3] % 8:
            raise ValueError(f"UNetDiscriminatorSN needs a (B, C, H, W) input with H and W multiples of 8, got {tuple(x.shape)}")
        sn = [getattr(self, n) for n in _SN_LAYERS]
        ws = [m.weight_orig for m in sn]
        if not all(w.dtype == torch.float32 and w.is_contiguous() and w.is_cuda for w in ws):
            raise ValueError("UNetDiscriminatorSN's spectral-normalised weights must be contiguous float32 CUDA tensors")
        dt = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float32
        if dt != torch.float32 and dt != torch.bfloat16:
            raise ValueError(f"UNetDiscriminatorSN runs in float32 or under bfloat16 autocast, not {dt}")
        cfg = {"dtype": dt, "skip": self.skip_connection, "train": self.training,
               "u": [m.weight_u for m in sn], "v": [m.weight_v for m in sn]}
        return _Discriminator.apply(cfg, x, self.conv0.weight, self.conv0.bias, self.conv9.weight, self.conv9.bias, *ws)


class _BceLogits(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, target, weight):
        x = x.contiguous()
        ctx.save_for_backward(x)
        ctx.target, ctx.weight = target, weight
        return ops.bce_logits(x, target, weight)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return ops.bce_logits_bwd(x, g.float().contiguous(), ctx.target, ctx.weight), None, None


class GANLoss(nn.Module):
    """basicsr's GANLoss for gan_type='vanilla': BCEWithLogits(input, full_like(input, label)).mean(), times loss_weight for the
    generator's loss (is_disc=False).  Other gan_types raise NotImplementedError."""

    def __init__(self, gan_type, real_label_val=1.0, fake_label_val=0.0, loss_weight=1.0):
        super().__init__()
        if gan_type != "vanilla":
            raise NotImplementedError(f"GAN type {gan_type} is not implemented.")
        self.gan_type = gan_type
        self.real_label_val, self.fake_label_val = real_label_val, fake_label_val
        self.loss_weight = loss_weight

    def forward(self, input, target_is_real, is_disc=False):
        if not input.is_cuda:
            raise ValueError("GANLoss runs on CUDA tensors only")
        target = self.real_label_val if target_is_real else self.fake_label_val
        return _BceLogits.apply(input, float(target), 1.0 if is_disc else float(self.loss_weight))


__all__ = ["UNetDiscriminatorSN", "GANLoss"]
