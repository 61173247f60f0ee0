"""Module-level stand-in for mamba_ssm's pybind extension `selective_scan_cuda`, the fourth module the reference reaches the scan
through (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:21-29,294-313 when `selective_scan_cuda_core` is missing; the ground truth of
Mamba/kernels/selective_scan/test_selective_scan.py:321-359, wrapper at :18-165).  Same arity and return order:

    fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus) -> [out, x]  or  [out, x, out_z] with z
    bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, dz, delta_softplus, recompute_out_z)
        -> [du, ddelta, dA, dB, dC, dD, ddelta_bias]  + [dz] with z  + [out_z] with recompute_out_z

    import sys, vmambair_b200.selective_scan_cuda as m
    sys.modules["selective_scan_cuda"] = m          # before importing code that imports it

The z gate: out_z = out * SiLU(z), written by the forward launch next to the ungated `out` (which bwd needs back).  bwd runs the
gate's backward (vmb_scan_gate_bwd: dz into `dz` when given, and dout * SiLU(z) in fp32) and then the scan backward on that fp32
gradient, so 16-bit inputs lose no precision in between.
`x` is fp32 (batch, dim, ceil(L/64), 2 dstate): checkpoints of the state every 64 positions in the odd slots, zeros in the even
ones, and its last row is the state after position L-1 for every L, so the reference wrapper's `x[:, :, -1, 1::2]` (:79) is the
last state.  bwd hands the backward the dense copy x[..., 1::2].
B and C must be variable, (batch, dstate, L) or (batch, G, dstate, L), and A real: the forms the reference test runs
(:373,384-386).  dB / dC come back in B / C's shape and dtype; dA, dD, ddelta_bias in fp32.
Under torch.use_deterministic_algorithms(True) the scan backward runs the library's deterministic kernels: gradients are bitwise
reproducible.
"""
import torch

from . import ops


def _prepare(u, A, B, C, who):
    if A.is_complex():
        raise RuntimeError(f"{who}: complex A is not supported (real A only)")
    if B.dim() not in (3, 4) or C.dim() not in (3, 4):
        raise RuntimeError(f"{who}: B and C must be variable, (batch, dstate, L) or (batch, G, dstate, L); "
                           f"got B {tuple(B.shape)}, C {tuple(C.shape)}")
    return (B.unsqueeze(1) if B.dim() == 3 else B), (C.unsqueeze(1) if C.dim() == 3 else C)


def fwd(u, delta, A, B, C, D=None, z=None, delta_bias=None, delta_softplus=False):
    B4, C4 = _prepare(u, A, B, C, "selective_scan_cuda.fwd")
    out, x, out_z = ops.selective_scan_fwd_z(u, delta, A, B4, C4, D, z, delta_bias, bool(delta_softplus))
    return [out, x] if z is None else [out, x, out_z]


def bwd(u, delta, A, B, C, D, z, delta_bias, dout, x, out, dz, delta_softplus, recompute_out_z):
    B4, C4 = _prepare(u, A, B, C, "selective_scan_cuda.bwd")
    if dout.stride(-1) != 1:
        dout = dout.contiguous()
    ckpt = x[..., 1::2].contiguous()
    if z is None:
        grads = list(ops.selective_scan_bwd(u, delta, A, B4, C4, D, delta_bias, dout, ckpt, bool(delta_softplus)))
        extra = []
    else:
        if out is None:
            raise RuntimeError("selective_scan_cuda.bwd: with z, the forward's `out` is needed")
        dout_eff, dz, out_z = ops.scan_gate_bwd(dout, out, z, dz, bool(recompute_out_z))
        grads = list(ops.selective_scan_bwd(u, delta, A, B4, C4, D, delta_bias, dout_eff, ckpt, bool(delta_softplus),
                                            dout_float=True))
        extra = [dz] + ([out_z] if recompute_out_z else [])
    if B.dim() == 3:
        grads[3] = grads[3].squeeze(1)
    if C.dim() == 3:
        grads[4] = grads[4].squeeze(1)
    return grads + extra
