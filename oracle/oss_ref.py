"""CPU oracle of the OSS block / network, forward and (under autograd) backward.  TEST INFRASTRUCTURE ONLY.

A functional (state_dict-driven) restatement in plain torch of the reference modules
  LayerNorm          SRGAN/VmambaIR/archs/MambaSISR6_arch.py:166-195
  FeedForward        MambaSISR6_arch.py:201-218
  SS2D_1.forward     MambaSISR6_arch.py:395-498 (and the Mamber32/33, RealSR variants, SURVEY.md 0.2)
  MamberBlock        MambaSISR6_arch.py:502-515
  MambaSISR6.forward MambaSISR6_arch.py:610-643 (Mamber32: mamber32_arch.py:611-649)
with the scan evaluated by the sequential C oracle (oracle/cscan.py).  Pinned against outputs of the
real reference modules by tests/test_oracle_modules.py (fixtures from tests/golden/make_golden.py).
Used by tests, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg; the product
(vmambair_b200) never imports it.

The torch ops run in the dtype and on the device of their inputs (the GPU tests evaluate the oracle in float64 on CUDA); the scan
always runs on the CPU.  With grad enabled and an input that requires grad, the scan is cscan.Scan (the C oracle's analytic backward),
so the whole block / net is differentiable: tests/test_oracle_grad_cpu.py pins that backward against the real reference's autograd.

Storage-precision emulation (STORE_DTYPE, test infrastructure): when set to a dtype (torch.bfloat16), every tensor the fused pipeline
keeps in that dtype between kernels is rounded to it here as well and back to its own dtype (arithmetic stays in the input dtype, like
the kernels' fp32 accumulators), and GEMM / conv weights are rounded once.  Gives the error a "bf16 storage, fp32 accumulate" evaluation
of the SAME network is expected to have against the unrounded oracle -- the yardstick for the bf16 bounds of
tests/test_bench_parity_gpu.py (inference) and tests/test_train_net_gpu.py (training).  Under autograd the rounding points act on the
backward too, as the training path (vmambair_b200.fused_train) stores them:
  _q    an activation the forward stores AND whose gradient the backward stores in the compute dtype: value and gradient rounded
        -- xz's x half (_Front.forward pixlin -> xz / backward dxz[:, :C] from the flipped dwconv), xc (dwconv3x3 + SiLU / sum4_add
        -> dxc), delta, B, C (dbl4 / ddbl), the scan outputs (ys / dys = the gathered merge gradient dm), y2 (merge_norm_gate / the
        dy2 _Tail hands back), the FFN's t (_Tail.forward pixlin + norm2 / dt) and gg (dwconv3x3 GELU gate / dgg);
  _qs   the residual stream, likewise: x1 (out_conv + residual / dx1 = layernorm_bwd(add=dout)) and the block output (/ dout);
  _qg   a gradient the backward stores with no stored forward value behind it: gradient only -- the scan's du per direction
        (selective_scan_bwd), dv in front of both depthwise convs (dwconv3x3_bwd phase "data"), dxn / dx1n at the norm1 / norm2
        outputs (pixlin with WinT / WpinT), norm1's dx (layernorm_bwd, before autograd adds the residual's), z_pre's gradient
        (merge_norm_gate_bwd dz_out), and dyg in front of the channel gate (_out_conv_bwd pixlin with WoutT);
  _qw   GEMM weights (prepare_block's kernel-layout copies): forward only -- parameter gradients are fp32 accumulators, never rounded.
Not emulated: z_pre's stored value (the training path keeps z_pre and applies SiLU in fp32; the inference path, emulated here, stores
SiLU(z)), and the single rounding of the x_proj data gradient summed over the four directions (pixlin with WbigT).
With STORE_DTYPE unset, or without grad, the oracle computes exactly what it computes without these rules.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import cscan

STORE_DTYPE = None
STREAM_FP32 = False  # with STORE_DTYPE set: keep the residual stream (block inputs / outputs) un-rounded


class _Store(torch.autograd.Function):
    """value and / or incoming gradient rounded to STORE_DTYPE and back to their own dtype"""

    @staticmethod
    def forward(ctx, t, value, grad):
        ctx.grad = grad
        return t.to(STORE_DTYPE).to(t.dtype) if value else t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return (g.to(STORE_DTYPE).to(g.dtype) if ctx.grad else g), None, None


def _store(t, value=True, grad=True):
    if STORE_DTYPE is None:
        return t
    if torch.is_grad_enabled() and t.requires_grad:
        return _Store.apply(t, value, grad)
    return t.to(STORE_DTYPE).to(t.dtype) if value else t


def _q(t):
    return _store(t)


def _qs(t):  # residual stream
    return t if STREAM_FP32 else _store(t)


def _qg(t):
    return _store(t, value=False)


def _qw(w):
    return w if (w is None or w.dim() < 2) else _store(w, grad=False)


def _ln(x, w, b):  # per-pixel LayerNorm over channels of (B,C,H,W)
    mu = x.mean(1, keepdim=True)
    var = x.var(1, keepdim=True, unbiased=False)
    y = (x - mu) / torch.sqrt(var + 1e-5) if b is not None else x / torch.sqrt(var + 1e-5)
    y = y * w.view(1, -1, 1, 1)
    return y + b.view(1, -1, 1, 1) if b is not None else y


def _scan(u, dt, A, B, C, D, bias):
    ins = (u, dt, A, B, C, D, bias)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ins):
        return cscan.Scan.apply(*ins, True)
    return cscan.scan_fwd(*ins, True, fp64=u.dtype == torch.float64).to(device=u.device, dtype=u.dtype)


def ss2d(sd, pre, x, gate):
    g = lambda k: sd[pre + k]
    B_, C, H, W = x.shape
    L = H * W
    xz = F.conv2d(x, _qw(g("in_conv.weight")), g("in_conv.bias"))
    xi, z = xz.chunk(2, 1)
    z = _store(F.silu(_qg(z)), grad=False)
    xi = _q(F.silu(_qg(F.conv2d(_q(xi), g("conv2d.weight"), g("conv2d.bias"), padding=1, groups=C))))
    # four spatial directions: row-major, column-major, and their reversals (:401-404)
    rows = xi.flatten(2)
    cols = xi.transpose(2, 3).flatten(2)
    xs = torch.stack([rows, cols, rows.flip(-1), cols.flip(-1)], 1)  # (B,4,C,L)
    xw = g("x_proj_weight")
    R = g("dt_projs_weight").shape[2]
    N = g("A_logs").shape[1]
    x_dbl = torch.einsum("bkdl,kcd->bkcl", xs, xw)
    dts = torch.einsum("bkrl,kdr->bkdl", x_dbl[:, :, :R], g("dt_projs_weight"))
    Bs, Cs = x_dbl[:, :, R:R + N], x_dbl[:, :, R + N:]
    if STORE_DTYPE is not None:  # the fused path folds W_dt W_x into one low-precision weight and stores delta, B, C
        big = _qw(torch.einsum("kdr,krc->kdc", g("dt_projs_weight"), xw[:, :R]))
        dts = _q(torch.einsum("bkcl,kdc->bkdl", xs, big))
        xq = torch.einsum("bkdl,kcd->bkcl", xs, _qw(xw))
        Bs, Cs = _q(xq[:, :, R:R + N]), _q(xq[:, :, R + N:])
    oy = _scan(_qg(xs).reshape(B_, 4 * C, L), dts.reshape(B_, 4 * C, L), -torch.exp(g("A_logs")), Bs, Cs, g("Ds"),
               g("dt_projs_bias").reshape(-1)).view(B_, 4, C, L)
    oy = _q(oy)
    y = oy[:, 0] + oy[:, 2].flip(-1)
    ycol = oy[:, 1] + oy[:, 3].flip(-1)
    y = y + ycol.view(B_, C, W, H).transpose(2, 3).reshape(B_, C, L)
    y1 = _ln(y.view(B_, C, H, W), g("out_norm.body.weight"), g("out_norm.body.bias"))
    y2 = _q(y1 * z)
    c = channel(sd, pre, y2.mean((2, 3)))[:, :, None, None]  # (B,C,1,1)
    y2 = _qg(y2 * c + y2 if gate == "mul" else y2 + c)
    return F.conv2d(y2, _qw(g("out_conv.weight")), g("out_conv.bias"))


def channel(sd, pre, pooled):
    """channel direction (forward + backward scan over the pooled channel descriptor, :438-483): pooled (B, C) channel means ->
    channel_norm output (B, C)"""
    g = lambda k: sd[pre + k]
    B_, C = pooled.shape
    if pre + "conv_cin.weight" in sd:
        seq = pooled[:, None, :] * g("conv_cin.weight").view(1, -1, 1) + g("conv_cin.bias").view(1, -1, 1)
    else:
        seq = pooled[:, None, :]
    dc = seq.shape[1]
    xsc = torch.stack([seq, seq.flip(-1)], 1)  # (B,2,dc,C)
    Rc = g("dtc_projs_weight").shape[2]
    Nc = g("Ac_logs").shape[1]
    xc_dbl = torch.einsum("bkdl,kcd->bkcl", xsc, g("xc_proj_weight"))
    dtc = torch.einsum("bkrl,kdr->bkdl", xc_dbl[:, :, :Rc], g("dtc_projs_weight"))
    oc = _scan(xsc.reshape(B_, 2 * dc, C), dtc.reshape(B_, 2 * dc, C), -torch.exp(g("Ac_logs")), xc_dbl[:, :, Rc:Rc + Nc],
               xc_dbl[:, :, Rc + Nc:], g("Dsc"), g("dtc_projs_bias").reshape(-1)).view(B_, 2, dc, C)
    yc = oc[:, 0] + oc[:, 1].flip(-1)  # (B, dc, C)
    if pre + "conv_cout.weight" in sd:
        yc = (yc * g("conv_cout.weight").view(1, -1, 1)).sum(1, keepdim=True) + g("conv_cout.bias").view(1, 1, 1)
    return _ln(yc.transpose(1, 2).unsqueeze(-1), g("channel_norm.body.weight"), g("channel_norm.body.bias")).view(B_, C)


def ffn(sd, pre, x):
    t = _q(F.conv2d(x, _qw(sd[pre + "project_in.weight"]), sd.get(pre + "project_in.bias")))
    t = _qg(F.conv2d(t, sd[pre + "dwconv.weight"], sd.get(pre + "dwconv.bias"), padding=1, groups=t.shape[1]))
    a, b = t.chunk(2, 1)
    return F.conv2d(_q(F.gelu(a) * b), _qw(sd[pre + "project_out.weight"]), sd.get(pre + "project_out.bias"))


def block(sd, pre, x, gate="mul"):
    x = _qs(x + ss2d(sd, pre + "attn.", _qg(_ln(_qg(x), sd[pre + "norm1.body.weight"], sd.get(pre + "norm1.body.bias"))), gate))
    return _qs(x + ffn(sd, pre + "ffn.", _qg(_ln(x, sd[pre + "norm2.body.weight"], sd.get(pre + "norm2.body.bias")))))


def _stage(sd, name, x, gate):
    i = 0
    while f"{name}.{i}.norm1.body.weight" in sd:
        x = block(sd, f"{name}.{i}.", x, gate)
        i += 1
    return x


def net_forward(sd, x, kind="sisr", scale=4):
    """kind: 'sisr' / 'realsr' (SR tail + nearest-upsampled input) or 'mamber32' / 'mamber33' (conv + input)."""
    gate = "add" if kind == "mamber32" else "mul"
    conv = lambda k, t, **kw: _q(F.conv2d(t, _qw(sd[k + ".weight"]), sd.get(k + ".bias"), **kw))
    e1 = _stage(sd, "encoder_level1", conv("patch_embed.proj", x, padding=1), gate)
    e2 = _stage(sd, "encoder_level2", F.pixel_unshuffle(conv("down1_2.body.0", e1, padding=1), 2), gate)
    e3 = _stage(sd, "encoder_level3", F.pixel_unshuffle(conv("down2_3.body.0", e2, padding=1), 2), gate)
    lat = _stage(sd, "latent", F.pixel_unshuffle(conv("down3_4.body.0", e3, padding=1), 2), gate)
    d3 = torch.cat([F.pixel_shuffle(conv("up4_3.body.0", lat, padding=1), 2), e3], 1)
    d3 = _stage(sd, "decoder_level3", conv("reduce_chan_level3", d3), gate)
    d2 = torch.cat([F.pixel_shuffle(conv("up3_2.body.0", d3, padding=1), 2), e2], 1)
    d2 = _stage(sd, "decoder_level2", conv("reduce_chan_level2", d2), gate)
    d1 = torch.cat([F.pixel_shuffle(conv("up2_1.body.0", d2, padding=1), 2), e1], 1)
    f = _stage(sd, "refinement", _stage(sd, "decoder_level1", d1, gate), gate)
    if kind in ("sisr", "realsr"):
        f = F.pixel_shuffle(conv("tail.0.0", f, padding=1), 2)
        f = F.pixel_shuffle(conv("tail.0.2", f, padding=1), 2)
        return conv("tail.1", f, padding=1) + F.interpolate(x, scale_factor=scale, mode="nearest")
    return conv("output", f, padding=1) + x
