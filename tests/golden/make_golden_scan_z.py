#!/usr/bin/env python
"""Golden vectors of the z-gated selective scan from the REAL reference function (a checkout of the reference project next to this
repository, ../reference, or $VMB_REFERENCE_DIR), like make_golden.py: `selective_scan_ref`
(Mamba/kernels/selective_scan/test_selective_scan.py:168-234, which takes z and return_last_state) is AST-extracted at run time and
run on seeded inputs; only numbers are written.

  python tests/golden/make_golden_scan_z.py      # -> tests/golden/scan_z_ref.npz

Per case <name>/: the inputs (u, delta, A, B, C, z, and D / bias when present), the gated `out`, `last_state`, the incoming gradient
`dout` and all eight gradients (du, ddelta, dA, dB, dC, dz, dD, dbias), fp32 throughout."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import load_ref_scan  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
REF_SCAN = load_ref_scan()

SPECS = [  # (name, b, D, L, N, G, has_D, has_bias, softplus)
    ("a", 2, 8, 64, 16, 2, True, True, True),
    ("b", 1, 12, 100, 16, 1, True, False, True),     # ragged L
    ("c", 2, 6, 129, 8, 2, False, True, False),      # ragged L, one past two checkpoint intervals
    ("d", 1, 8, 33, 4, 1, False, False, False),
]


def gen():
    cases = {}
    for name, b, Dm, L, N, G, hD, hb, sp in SPECS:
        torch.manual_seed(300 + ord(name))
        # distributions of the reference test (test_selective_scan.py:411-441)
        A = -0.5 * torch.rand(Dm, N)
        Bm = torch.randn(b, G, N, L)
        Cm = torch.randn(b, G, N, L)
        Dv = torch.randn(Dm) if hD else None
        bias = 0.5 * torch.rand(Dm) if hb else None
        z = torch.randn(b, Dm, L)
        u = torch.randn(b, Dm, L)
        delta = 0.5 * torch.rand(b, Dm, L)
        ins = [t.clone().requires_grad_() if t is not None else None for t in (u, delta, A, Bm, Cm, Dv, z, bias)]
        out, last = REF_SCAN(*ins, sp, True)
        g = torch.randn_like(out)
        grads = torch.autograd.grad(out, [t for t in ins if t is not None], g)
        it = iter(grads)
        gl = [next(it) if t is not None else None for t in ins]
        rec = dict(u=u, delta=delta, A=A, B=Bm, C=Cm, z=z, out=out.detach(), last_state=last.detach(), dout=g,
                   du=gl[0], ddelta=gl[1], dA=gl[2], dB=gl[3], dC=gl[4], dz=gl[6])
        if hD:
            rec.update(D=Dv, dD=gl[5])
        if hb:
            rec.update(bias=bias, dbias=gl[7])
        for k, v in rec.items():
            cases[f"{name}/{k}"] = v.float().numpy()
        cases[f"{name}/softplus"] = np.array(int(sp))
    np.savez(f"{OUT}/scan_z_ref.npz", **cases)
    print("scan_z_ref.npz", sum(v.nbytes for v in cases.values()) // 1024, "KiB")


if __name__ == "__main__":
    gen()
