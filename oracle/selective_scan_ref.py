"""CPU oracle for the selective-scan operator.  TEST INFRASTRUCTURE ONLY.

This file is a from-scratch restatement (torch, CPU) of the math the reference
states in ``Mamba/kernels/selective_scan/test_selective_scan.py:168-234``
(``selective_scan_ref``) and of the analytic backward the reference CUDA
kernel implements in
``Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan_bwd_kernel.cuh:139-241``.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` leg may import it.  The product path
(``vmambair_b200``) never does.

Parity pinning: ``tests/golden/make_golden.py`` runs the *real* reference
function (AST-extracted from the reference project, not copied) on seeded inputs and
commits its outputs under ``tests/golden/``; ``tests/test_oracle.py`` checks
this restatement against those vectors.

Math (per batch b, channel d, state n, position l), all in fp32 (or fp64):
    dt   = delta + delta_bias[d];  dt = softplus(dt) if delta_softplus
    h_l  = exp(dt_l * A[d,n]) * h_{l-1} + dt_l * u_l * B[b,g(d),n,l]
    y_l  = sum_n C[b,g(d),n,l] * h_l  + D[d] * u_l
with g(d) = d // (D/G)  (group-shared B/C,  reference fwd kernel :82).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _prep(u, delta, A, B, C, D, delta_bias, delta_softplus, dtype):
    u = u.to(dtype)
    dt = delta.to(dtype)
    if delta_bias is not None:
        dt = dt + delta_bias.to(dtype)[None, :, None]
    if delta_softplus:
        dt = F.softplus(dt)  # threshold 20, same as the reference kernel (:117)
    if B.dim() == 3:
        B = B[:, None]
    if C.dim() == 3:
        C = C[:, None]
    Dm = A.shape[0]
    G = B.shape[1]
    assert Dm % G == 0
    rep = Dm // G
    Bf = B.to(dtype).repeat_interleave(rep, dim=1)  # (b, D, N, L)
    Cf = C.to(dtype).repeat_interleave(rep, dim=1)
    return u, dt, A.to(dtype), Bf, Cf, (None if D is None else D.to(dtype))


def selective_scan_oracle(u, delta, A, B, C, D=None, delta_bias=None,
                          delta_softplus=False, return_last_state=False,
                          dtype=torch.float32):
    """Sequential recurrence; returns out in u.dtype (like the reference :232)."""
    dtype_in = u.dtype
    u_, dt, A_, Bf, Cf, D_ = _prep(u, delta, A, B, C, D, delta_bias, delta_softplus, dtype)
    b, Dm, L = u_.shape
    N = A_.shape[1]
    h = torch.zeros(b, Dm, N, dtype=dtype)
    ys = torch.empty(b, Dm, L, dtype=dtype)
    dtu = dt * u_
    for l in range(L):
        a = torch.exp(dt[:, :, l, None] * A_[None])              # (b, D, N)
        h = a * h + dtu[:, :, l, None] * Bf[:, :, :, l]
        ys[:, :, l] = (h * Cf[:, :, :, l]).sum(-1)
    out = ys if D_ is None else ys + u_ * D_[None, :, None]
    out = out.to(dtype_in)
    return (out, h) if return_last_state else out


def selective_scan_oracle_bwd(u, delta, A, B, C, D, delta_bias, dout,
                              delta_softplus=False, dtype=torch.float64):
    """Analytic backward, restated from the formulas the reference bwd kernel
    evaluates (:198-241):  dh_l = C_l*dout_l + a_{l+1}*dh_{l+1};
    du = D*dout + sum_n dh*dt*B;  ddt = sum_n dh*(u*B + A*(h - dt*u*B));
    dA = sum_l dh*dt*(h - dt*u*B);  dB = sum_{d in g} dh*dt*u;
    dC = sum_{d in g} dout*h;  dD = sum dout*u;  ddelta = ddt*sigmoid(x) if softplus;
    dbias = sum ddelta.  Returns fp64 (or `dtype`) tensors.
    """
    u_, dt, A_, Bf, Cf, D_ = _prep(u, delta, A, B, C, D, delta_bias, delta_softplus, dtype)
    dout = dout.to(dtype)
    b, Dm, L = u_.shape
    N = A_.shape[1]
    G = B.shape[1] if B.dim() == 4 else 1
    rep = Dm // G
    # forward states
    hs = torch.empty(b, Dm, N, L, dtype=dtype)
    h = torch.zeros(b, Dm, N, dtype=dtype)
    dtu = dt * u_
    for l in range(L):
        a = torch.exp(dt[:, :, l, None] * A_[None])
        h = a * h + dtu[:, :, l, None] * Bf[:, :, :, l]
        hs[:, :, :, l] = h
    du = torch.zeros_like(u_) if D_ is None else dout * D_[None, :, None]
    ddt = torch.zeros_like(u_)
    dA = torch.zeros_like(A_)
    dBf = torch.zeros_like(Bf)
    dCf = torch.zeros_like(Cf)
    dh = torch.zeros(b, Dm, N, dtype=dtype)
    for l in range(L - 1, -1, -1):
        if l + 1 < L:
            a_next = torch.exp(dt[:, :, l + 1, None] * A_[None])
            dh = a_next * dh
        dh = dh + Cf[:, :, :, l] * dout[:, :, l, None]
        hl = hs[:, :, :, l]
        bl = dtu[:, :, l, None] * Bf[:, :, :, l]
        du[:, :, l] += (dh * Bf[:, :, :, l]).sum(-1) * dt[:, :, l]
        ddt[:, :, l] = (dh * (u_[:, :, l, None] * Bf[:, :, :, l] + A_[None] * (hl - bl))).sum(-1)
        dA += (dh * dt[:, :, l, None] * (hl - bl)).sum(0)
        dBf[:, :, :, l] = dh * dtu[:, :, l, None]
        dCf[:, :, :, l] = hl * dout[:, :, l, None]
    dB = dBf.view(b, G, rep, N, L).sum(2)
    dC = dCf.view(b, G, rep, N, L).sum(2)
    dD = None if D is None else (dout * u_).sum((0, 2))
    if delta_softplus:
        x = delta.to(dtype)
        if delta_bias is not None:
            x = x + delta_bias.to(dtype)[None, :, None]
        ddelta = torch.where(x <= 20.0, ddt * torch.sigmoid(x), ddt)
    else:
        ddelta = ddt
    dbias = None if delta_bias is None else ddelta.sum((0, 2))
    return du, ddelta, dA, dB, dC, dD, dbias
