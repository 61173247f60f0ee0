"""`selective_scan_fn` -- drop-in for the reference's SelectiveScanFn / selective_scan_fn_v1
(SRGAN/VmambaIR/archs/MambaSISR6_arch.py:24-96, same in the Deraining / RealSR archs): same
argument order, same contiguity / dim fix-ups, same returned gradients; the kernels underneath are
the sm_90a ones of this repository (through the C-ABI).
"""
from __future__ import annotations

import torch

from . import ops


class SelectiveScanFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
        if u.stride(-1) != 1:
            u = u.contiguous()
        if delta.stride(-1) != 1:
            delta = delta.contiguous()
        if D is not None:
            D = D.contiguous()
        if B.stride(-1) != 1:
            B = B.contiguous()
        if C.stride(-1) != 1:
            C = C.contiguous()
        ctx.squeeze_B = B.dim() == 3
        ctx.squeeze_C = C.dim() == 3
        if ctx.squeeze_B:
            B = B.unsqueeze(1)
        if ctx.squeeze_C:
            C = C.unsqueeze(1)
        ctx._d_dtype = None if D is None else D.dtype
        ctx._b_dtype = None if delta_bias is None else delta_bias.dtype
        if D is not None and D.dtype != torch.float32:
            D = D.float()
        if delta_bias is not None and delta_bias.dtype != torch.float32:
            delta_bias = delta_bias.float()
        if u.shape[1] % (B.shape[1] * nrows) != 0 or nrows not in (1, 2, 3, 4):
            raise AssertionError("dim must be divisible by n_groups * nrows; nrows in 1..4")
        need_grad = any(t is not None and t.requires_grad for t in (u, delta, A, B, C, D, delta_bias))
        A = A.contiguous()
        out, ckpt = ops.selective_scan_fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, need_ckpt=need_grad)
        ctx.delta_softplus = delta_softplus
        ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, ckpt)
        return out

    @staticmethod
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, delta_bias, ckpt = ctx.saved_tensors
        if dout.stride(-1) != 1:
            dout = dout.contiguous()
        du, ddelta, dA, dB, dC, dD, dbias = ops.selective_scan_bwd(
            u, delta, A, B, C, D, delta_bias, dout, ckpt, ctx.delta_softplus)
        if ctx.squeeze_B:
            dB = dB.squeeze(1)
        if ctx.squeeze_C:
            dC = dC.squeeze(1)
        if dD is not None and ctx._d_dtype not in (None, dD.dtype):
            dD = dD.to(ctx._d_dtype)
        if dbias is not None and ctx._b_dtype not in (None, dbias.dtype):
            dbias = dbias.to(ctx._b_dtype)
        return du, ddelta, dA, dB, dC, dD, dbias, None, None


def selective_scan_fn(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
    """out = selective_scan(u, delta, A, B, C, D, delta_bias, delta_softplus) with autograd.
    Mixed input dtypes (autocast regions) are promoted to fp32, like the RealSR reference's
    custom_fwd(cast_inputs=torch.float32) (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:269-270)."""
    if not (u.dtype == delta.dtype == B.dtype == C.dtype):
        u, delta, B, C = u.float(), delta.float(), B.float(), C.float()
    if A.dtype != torch.float32:
        A = A.float()
    return SelectiveScanFn.apply(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows)


selective_scan_fn_v1 = selective_scan_fn
