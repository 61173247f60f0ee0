"""`selective_scan_fn` -- drop-in for the reference's SelectiveScanFn / selective_scan_fn_v1
(SRGAN/VmambaIR/archs/MambaSISR6_arch.py:24-96, same in the Deraining / RealSR archs): same
argument order, same contiguity / dim fix-ups, same returned gradients; the kernels underneath are
the sm_90a ones of this repository (through the C-ABI).
"""
from __future__ import annotations

import torch

from . import ops, selective_scan_cuda


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
    custom_fwd(cast_inputs=torch.float32) (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:269-270).
    Under torch.use_deterministic_algorithms(True) the backward runs the library's deterministic kernels (fixed-order sums of
    per-CTA partials instead of fp32 atomics), so its gradients are bitwise reproducible."""
    if not (u.dtype == delta.dtype == B.dtype == C.dtype):
        u, delta, B, C = u.float(), delta.float(), B.float(), C.float()
    if A.dtype != torch.float32:
        A = A.float()
    return SelectiveScanFn.apply(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows)


selective_scan_fn_v1 = selective_scan_fn


class MambaSelectiveScanFn(torch.autograd.Function):
    """mamba_ssm's SelectiveScanFn over selective_scan_cuda (the reference's wrapper, Mamba/kernels/selective_scan/
    test_selective_scan.py:18-165, MODE "mamba_ssm")"""

    @staticmethod
    def forward(ctx, u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, return_last_state=False):
        u, delta, B, C = (t if t.stride(-1) == 1 else t.contiguous() for t in (u, delta, B, C))
        if z is not None and z.stride(-1) != 1:
            z = z.contiguous()
        ctx._d_dtype = None if D is None else D.dtype
        ctx._b_dtype = None if delta_bias is None else delta_bias.dtype
        if D is not None:
            D = D.contiguous().float()
        if delta_bias is not None:
            delta_bias = delta_bias.float()
        A = A.contiguous()
        out, x, *rest = selective_scan_cuda.fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus)
        ctx.delta_softplus = delta_softplus
        ctx.has_z = z is not None
        ctx.save_for_backward(u, delta, A, B, C, D, z, delta_bias, x, out if z is not None else None)
        y = rest[0] if z is not None else out
        if not return_last_state:
            return y
        last_state = x[:, :, -1, 1::2]
        ctx.mark_non_differentiable(last_state)
        return y, last_state

    @staticmethod
    def backward(ctx, dout, *args):
        u, delta, A, B, C, D, z, delta_bias, x, out = ctx.saved_tensors
        du, ddelta, dA, dB, dC, dD, dbias, *rest = selective_scan_cuda.bwd(
            u, delta, A, B, C, D, z, delta_bias, dout, x, out, None, ctx.delta_softplus, False)
        dz = rest[0] if ctx.has_z else None
        if dD is not None and ctx._d_dtype not in (None, dD.dtype):
            dD = dD.to(ctx._d_dtype)
        if dbias is not None and ctx._b_dtype not in (None, dbias.dtype):
            dbias = dbias.to(ctx._b_dtype)
        return du, ddelta, dA, dB, dC, dD, dz, dbias, None, None


def mamba_selective_scan_fn(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False, return_last_state=False):
    """mamba_ssm's selective_scan_fn: out = selective_scan(u, delta, A, B, C, D, delta_bias, delta_softplus), times SiLU(z) when z
    is given, with autograd (dz included).  Its 7th positional argument is z, where selective_scan_fn's is delta_bias.
    return_last_state: also return the state after the last position, (batch, dim, dstate) fp32, which has no gradient.
    B, C: (batch, dstate, L) or (batch, G, dstate, L); A real.  Mixed input dtypes are promoted to fp32 as in selective_scan_fn.
    Under torch.use_deterministic_algorithms(True) the gradients are bitwise reproducible."""
    ts = (u, delta, B, C) + ((z,) if z is not None else ())
    if any(t.dtype != u.dtype for t in ts):
        u, delta, B, C = u.float(), delta.float(), B.float(), C.float()
        z = z.float() if z is not None else None
    return MambaSelectiveScanFn.apply(u, delta, A, B, C, D, z, delta_bias, delta_softplus, return_last_state)
