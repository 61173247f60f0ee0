"""Module-level stand-in for the reference's pybind extension `selective_scan_cuda_oflex`
(Mamba/kernels/selective_scan/csrc/selective_scan/cusoflex/selective_scan_oflex.cpp:360-363): exposes
`fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows, out_float) -> [out, x]` and
`bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus, nrows) -> [du, ddelta, dA, dB, dC, dD, ddelta_bias]`
with the same arity / return order, on the sm_90a kernels:

    import sys, vmambair_b200.selective_scan_cuda_oflex as m
    sys.modules["selective_scan_cuda_oflex"] = m          # before importing code that imports it

out_float=True gives an fp32 `out` from bf16 / fp16 inputs: the fp32 accumulator, stored without rounding (cpp:219,235-239).
bwd accepts that fp32 `dout` against 16-bit inputs (cpp:257-260,349-355); du, ddelta, dB, dC come back in the input dtype and
dA, dD, ddelta_bias in fp32, as in the reference (cpp:324-356).  With fp32 inputs out_float changes nothing.
`x` is opaque to the callers (they only hand it back to bwd): here it is the fp32 checkpoint tensor
(batch, dim, ceil(L/64), dstate), as in selective_scan_cuda_core.  `nrows` is accepted and ignored.
Under torch.use_deterministic_algorithms(True) the backward runs the library's deterministic kernels (fixed-order sums
of per-CTA partials instead of fp32 atomics): gradients are bitwise reproducible.
"""
from . import ops


def fwd(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1, out_float=False):
    out, ckpt = ops.selective_scan_fwd(u, delta, A, B, C, D, delta_bias, bool(delta_softplus), need_ckpt=True,
                                       out_float=bool(out_float))
    return [out, ckpt]


def bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus=False, nrows=1):
    return list(ops.selective_scan_bwd(u, delta, A, B, C, D, delta_bias, dout, x, bool(delta_softplus), dout_float=True))
