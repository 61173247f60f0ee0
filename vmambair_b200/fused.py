"""Fused inference pipeline of one OSS block: 15 launches of this library's kernels instead of the ~85
un-fused PyTorch ops of the reference MamberBlock.forward (SRGAN/VmambaIR/archs/MambaSISR6_arch.py:486-515).

   norm1+in_conv(+SiLU z) -> dwconv3x3+SiLU -> transpose (the (W,H) copy of x) -> x_proj (+dt_proj folded: W_dt W_x is a
   CxC map, so delta, B, C of directions 0/2 come out of ONE GEMM on x and of 1/3 out of one GEMM on x^T) ->
   direction-aware selective scan (reversal inside the kernel, no gathered operands) -> 4-way sum in the reference's
   order + out_norm + gate + pooling -> channel-direction OSS (1 CTA/image) -> channel gate + out_conv + residual ->
   norm2+project_in -> dwconv3x3 + GELU gate -> project_out + residual
   (shapes with L % 8 != 0 take the explicit cross_scan gather instead of the direction-aware scan)

A standalone SS2D_1 (ss2d_forward) runs the same chain from in_conv (no norm1 prologue) to out_conv (no residual), with d_model and the
expanded width E = d_inner carried separately.

No CPU path, no silent fallback: every stage goes through the C-ABI and raises on failure.
"""
from __future__ import annotations

import torch

from . import ops

_DTYPES = (torch.float32, torch.bfloat16, torch.float16)


_warned = set()


def unsupported_reason(mod, x: torch.Tensor):
    """None when the fused kernels cover this call of `mod` (a MamberBlock, or a standalone SS2D_1), else the first kernel limit it
    violates.  Mirrors the checks of the launchers: LayerNorm / gate prologues keep the whole K resident (csrc/pixlin.cu pixlin_launch:
    K <= 384), the depthwise conv indexes (batch, channel) planes on gridDim.y (csrc/api.cu vmb_dwconv3x3: batch * channels <= 65535),
    the channel branch holds its (dc, E) problem in one CTA's shared memory (csrc/oss_ops.cu channel_launch), dstate <= 16."""
    if not (x.is_cuda and x.dim() == 4):
        return "not a CUDA (B,C,H,W) tensor"
    if x.dtype not in _DTYPES:
        return f"dtype {x.dtype}"
    a = getattr(mod, "attn", mod)
    if a.d_state > 16 or a.dc_state > 16:
        return f"d_state {a.d_state} / dc_state {a.dc_state} > 16"
    B, C = x.shape[0], x.shape[1]
    if mod is a:  # standalone SS2D_1: in_conv has no LayerNorm prologue; out_conv's gate prologue keeps the E inputs resident
        E = a.d_inner
        if C != a.d_model:
            return f"x has {C} channels, the module d_model = {a.d_model}"
        if type(a.act) is not torch.nn.SiLU:
            return f"act_layer {type(a.act).__name__} (the kernels apply SiLU)"
        if E > 384:
            return f"E = {E} > 384 (gate prologue keeps K resident)"
        if B * E > 65535:
            return f"batch * channels = {B * E} > 65535 (depthwise-conv grid)"
    else:
        E = C
        h2 = mod.ffn.project_in.weight.shape[0]
        if C > 384:
            return f"C = {C} > 384 (LayerNorm / gate prologue keeps K resident)"
        if B * max(C, h2 // 2) > 65535 or B > 65535:
            return f"batch * channels = {B * max(C, h2 // 2)} > 65535 (depthwise-conv grid)"
    RN = a.dtc_rank + 2 * a.dc_state
    dc = a.dc_inner
    smem = 4 * (dc * E + 2 * RN * (E | 1) + 4 * dc * E + E + 64 + 2 * RN * dc + 2 * dc * a.dtc_rank + 5 * dc + 1)
    if smem > 227 * 1024:
        return f"channel branch needs {smem} B of shared memory"
    return None


def available(mod, x: torch.Tensor) -> bool:
    why = unsupported_reason(mod, x)
    if why is not None and x.is_cuda:
        what = "SS2D_1" if getattr(mod, "attn", None) is None else "OSS block"
        key = (what, why, tuple(x.shape[1:]))
        if key not in _warned:  # once per (module kind, reason, shape): the composed torch + scan-operator path takes over, loudly
            _warned.add(key)
            import warnings
            warnings.warn(f"vmambair_b200: fused {what} not available ({why}); using the composed path for x{tuple(x.shape)}")
    return why is None


def _f32(t):
    """fp32 kernel parameter; prefers the un-rounded fp32 master kept by engine.cast_for_inference"""
    if t is None:
        return None
    m = getattr(t, "_vmb_master", None)
    if m is not None and m.shape == t.shape and m.device == t.device:
        return m.contiguous()
    return t.detach().float().contiguous()


def _prepare(mod, dtype, device):
    """Weights in kernel layout (cached per module; rebuilt when any parameter changed).  mod: a MamberBlock (attn + norms + FFN) or a
    standalone SS2D_1 (attn weights only).  D = d_model (in_conv's input, out_conv's output), E = d_inner (the scanned width)."""
    ver = (dtype, device, sum(p._version for p in mod.parameters()), tuple(p.data_ptr() for p in mod.parameters()))
    cache = getattr(mod, "_vmb_cache", None)
    if cache is not None and cache["ver"] == ver:
        return cache
    a = getattr(mod, "attn", mod)
    D, C, R, N = a.d_model, a.d_inner, a.dt_rank, a.d_state
    w = lambda t: ops.pad_weight(t.detach().to(dtype))
    ln = lambda m: (1 if hasattr(m.body, "bias") else 2, _f32(m.body.weight), _f32(getattr(m.body, "bias", None)))
    xw, dtw = a.x_proj_weight.detach().float(), a.dt_projs_weight.detach().float()
    big = torch.cat([torch.cat([dtw[k] @ xw[k, :R], xw[k, R:]], 0) for k in range(4)], 0)  # (4(C+2N), C)
    has_cio = hasattr(a, "conv_cin")
    c = dict(
        ver=ver, C=C, N=N, R=R,
        w_in=w(a.in_conv.weight.view(2 * C, D)), b_in=_f32(a.in_conv.bias),
        dw=_f32(a.conv2d.weight.view(C, 9)), dw_b=_f32(a.conv2d.bias),
        w_big=w(big),
        w_big02=w(torch.cat([big[0:C + 2 * N], big[2 * (C + 2 * N):3 * (C + 2 * N)]], 0)),
        w_big13=w(torch.cat([big[(C + 2 * N):2 * (C + 2 * N)], big[3 * (C + 2 * N):]], 0)),
        A=(-torch.exp(a.A_logs.detach().float())).contiguous(), Ds=_f32(a.Ds), dt_bias=_f32(a.dt_projs_bias.view(-1)),
        on_w=_f32(a.out_norm.body.weight), on_b=_f32(a.out_norm.body.bias),
        ch=dict(cin_w=_f32(a.conv_cin.weight.view(-1)) if has_cio else None, cin_b=_f32(a.conv_cin.bias) if has_cio else None,
                xc_proj=_f32(a.xc_proj_weight), dtc_w=_f32(a.dtc_projs_weight), dtc_b=_f32(a.dtc_projs_bias),
                Ac_logs=_f32(a.Ac_logs), Dsc=_f32(a.Dsc),
                cout_w=_f32(a.conv_cout.weight.view(-1)) if has_cio else None, cout_b=_f32(a.conv_cout.bias) if has_cio else None,
                cn_w=_f32(a.channel_norm.body.weight), cn_b=_f32(a.channel_norm.body.bias),
                dc=a.dc_inner, Rc=a.dtc_rank, N=a.dc_state),
        gate_mode=1 if a.gate == "mul" else 2,
        w_out=w(a.out_conv.weight.view(D, C)), b_out=_f32(a.out_conv.bias),
    )
    if a is not mod:
        f = mod.ffn
        c.update(
            h=f.project_out.weight.shape[1], ln1=ln(mod.norm1), ln2=ln(mod.norm2),
            w_pin=w(f.project_in.weight.view(-1, C)), b_pin=_f32(f.project_in.bias),
            fdw=_f32(f.dwconv.weight.view(-1, 9)), fdw_b=_f32(f.dwconv.bias),
            w_pout=w(f.project_out.weight.view(C, -1)), b_pout=_f32(f.project_out.bias),
        )
    mod._vmb_cache = c
    return c


def _ss2d_core(c, x3, H, W, ln=None):
    """in_conv (ln: the norm1 prologue of a block) -> ... -> merge + out_norm + gate: x3 (B,D,L) -> (y2 (B,E,L), pooled sums (B,E))"""
    B, L = x3.shape[0], H * W
    C, N = c["C"], c["N"]
    # in_conv; SiLU on the z half
    xz = ops.pixlin(x3, c["w_in"], c["b_in"], ln=ln, act=(C, 2 * C))
    if L % 8 == 0:
        xc, xt = ops.dwconv3x3_t(xz[:, :C], c["dw"], c["dw_b"], C, H, W)  # x and its (W,H) copy from one launch
        # direction-aware scan: directions 0/2 read x and the GEMM on x, 1/3 read the transposed copies; reversed
        # directions walk the same memory backwards -- no gathered / flipped (B,4C,L) operands exist
        d02 = ops.pixlin(xc, c["w_big02"]).view(B, 2, C + 2 * N, L)
        d13 = ops.pixlin(xt, c["w_big13"]).view(B, 2, C + 2 * N, L)
        src = [(xc, d02[:, 0]), (xt, d13[:, 0]), (xc, d02[:, 1]), (xt, d13[:, 1])]
        ys = ops.selective_scan_fwd_grouped([s[0] for s in src], [s[1][:, :C] for s in src], [s[1][:, C:C + N] for s in src],
                                            [s[1][:, C + N:] for s in src], [0, 0, 1, 1], c["A"], c["Ds"], c["dt_bias"], True)
        return ops.merge_norm_gate(ys, xz[:, C:], c["on_w"], c["on_b"], C, H, W, in_place_order=True)
    # L % 8 != 0: the gathered path
    xc = ops.dwconv3x3(xz[:, :C], c["dw"], c["dw_b"], C, H, W, 0)
    # delta (dt_proj o x_proj), B, C of the four directions from one GEMM on the un-permuted x
    dbl = ops.pixlin(xc, c["w_big"])  # (B, 4*(C+2N), L)
    dbl4 = dbl.view(B, 4, C + 2 * N, L)
    xs = ops.cross_scan([xc] * 4, C, H, W)
    dts = ops.cross_scan([dbl4[:, k, :C] for k in range(4)], C, H, W)
    bc = ops.cross_scan([dbl4[:, k, C:] for k in range(4)], 2 * N, H, W)
    ys, _ = ops.selective_scan_fwd(xs.view(B, 4 * C, L), dts.view(B, 4 * C, L), c["A"], bc[:, :, :N], bc[:, :, N:], c["Ds"],
                                   c["dt_bias"], True, need_ckpt=False)
    return ops.merge_norm_gate(ys.view(B, 4, C, L), xz[:, C:], c["on_w"], c["on_b"], C, H, W)


def _gate_out_conv(c, y2, pooled, L, residual=None):
    """channel-direction OSS on the pooled sums -> channel gate + out_conv (+ residual): (B,E,L) -> (B,D,L)"""
    cg = ops.channel_branch(pooled, 1.0 / L, c["ch"], c["C"])
    return ops.pixlin(y2, c["w_out"], c["b_out"], residual=residual, gate=cg, gate_mode=c["gate_mode"])


@torch.no_grad()
def ss2d_forward(mod, x: torch.Tensor) -> torch.Tensor:
    """SS2D_1.forward of a standalone module (no norm in front, no residual behind): x (B,D,H,W) -> (B,D,H,W)"""
    B, D, H, W = x.shape
    L = H * W
    c = _prepare(mod, x.dtype, x.device)
    y2, pooled = _ss2d_core(c, x.contiguous().view(B, D, L), H, W)
    return _gate_out_conv(c, y2, pooled, L).view(B, D, H, W)


@torch.no_grad()
def block_forward(block, x: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """out: optional (B,C,H,W) destination with dense planes -- e.g. a channel slice of the decoder's concatenation buffer
    (unet.py): the block's last kernel stores there and torch.cat never runs."""
    B, C, H, W = x.shape
    L = H * W
    c = _prepare(block, x.dtype, x.device)
    x3 = x.contiguous().view(B, C, L)
    y2, pooled = _ss2d_core(c, x3, H, W, ln=c["ln1"])  # norm1 as in_conv's prologue
    x1 = _gate_out_conv(c, y2, pooled, L, residual=x3)
    t = ops.pixlin(x1, c["w_pin"], c["b_pin"], ln=c["ln2"])
    g = ops.dwconv3x3(t, c["fdw"], c["fdw_b"], c["h"], H, W, 1)
    if out is not None:
        assert out.shape == (B, C, H, W) and out.stride(3) == 1 and out.stride(2) == W and out.stride(1) == L
        ops.pixlin(g, c["w_pout"], c["b_pout"], residual=x1, out=out.view(B, C, L))
        return out
    return ops.pixlin(g, c["w_pout"], c["b_pout"], residual=x1).view(B, C, H, W)
