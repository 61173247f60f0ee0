"""Module-level stand-in for the reference's pybind extension `selective_scan_cuda_core`
(Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan.cpp:351-354): exposes
`fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows) -> [out, x]` and
`bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus, nrows) -> [du, ddelta, dA, dB, dC, dD, ddelta_bias]`
with the same arity / return order, so the UNMODIFIED reference archs run on the sm_90a kernels:

    import sys, vmambair_b200.selective_scan_cuda_core as m
    sys.modules["selective_scan_cuda_core"] = m          # before importing the reference arch

`x` is opaque to the callers (they only hand it back to bwd): here it is the fp32 checkpoint tensor
(batch, dim, ceil(L/64), dstate).  `nrows` is accepted and ignored, as in the reference (cpp:235,345).
Under torch.use_deterministic_algorithms(True) the backward runs the library's deterministic kernels (fixed-order sums
of per-CTA partials instead of fp32 atomics): gradients are bitwise reproducible.
"""
from . import ops


def fwd(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
    out, ckpt = ops.selective_scan_fwd(u, delta, A, B, C, D, delta_bias, bool(delta_softplus), need_ckpt=True)
    return [out, ckpt]


def bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus=False, nrows=1):
    return list(ops.selective_scan_bwd(u, delta, A, B, C, D, delta_bias, dout, x, bool(delta_softplus)))
