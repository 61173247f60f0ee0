"""Module-level stand-in for the reference's pybind extension `selective_scan_cuda_ndstate`
(Mamba/kernels/selective_scan/csrc/selective_scan/cusndstate/selective_scan_ndstate.cpp:338-341), the state-dimension-1
layout: A is (dim,), B and C are (batch, ngroups, seqlen).  Exposes
`fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows) -> [out, x]` (cpp:148-228) and
`bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus, nrows) -> [du, ddelta, dA, dB, dC, dD, ddelta_bias]`
(cpp:230-336) with the same arity / return order:

    import sys, vmambair_b200.selective_scan_cuda_ndstate as m
    sys.modules["selective_scan_cuda_ndstate"] = m

It runs the dstate = 1 case of the flat operator through views (A -> (dim, 1), B / C -> (batch, ngroups, 1, seqlen)): no copies
and no kernel of its own.  Gradients come back in the ndstate shapes: dA (dim,), dB / dC (batch, ngroups, seqlen).  `out` has the
input dtype (cpp:207).  `x` is opaque (the fp32 checkpoint tensor (batch, dim, ceil(L/64), 1)); `nrows` is ignored.
Under torch.use_deterministic_algorithms(True) the backward runs the library's deterministic kernels (fixed-order sums
of per-CTA partials instead of fp32 atomics): gradients are bitwise reproducible.
"""
from . import ops


def _views(A, B, C, who):
    if A.dim() != 1 or B.dim() != 3 or C.dim() != 3:
        raise RuntimeError(f"{who}: expected A (D,), B / C (B, G, L) (state dimension 1)")
    return A.unsqueeze(1), B.unsqueeze(2), C.unsqueeze(2)


def fwd(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
    A2, B2, C2 = _views(A, B, C, "selective_scan_fwd")
    out, ckpt = ops.selective_scan_fwd(u, delta, A2, B2, C2, D, delta_bias, bool(delta_softplus), need_ckpt=True)
    return [out, ckpt]


def bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus=False, nrows=1):
    A2, B2, C2 = _views(A, B, C, "selective_scan_bwd")
    if dout.dtype != u.dtype:  # cpp:248: no fp32 dout in this module
        raise RuntimeError(f"selective_scan_bwd: dout.dtype {dout.dtype} != u.dtype {u.dtype}")
    du, ddelta, dA, dB, dC, dD, dbias = ops.selective_scan_bwd(u, delta, A2, B2, C2, D, delta_bias, dout, x, bool(delta_softplus))
    return [du, ddelta, dA.view(A.shape), dB.squeeze(2), dC.squeeze(2), dD, dbias]
