#!/usr/bin/env python
"""Generate tests/golden/cross_selective_scan_c.npz from the REAL reference's cross_selective_scanC
(RealSR/VmambaIR/archs/MambaRealSR11_arch.py:438-534), with the reference's own selective_scan_ref as the scan.

Same conventions as make_golden.py, whose helpers it uses (the stubbed `selective_scan_cuda_core` import, the reference
checkout next to this repository or in $VMB_REFERENCE_DIR); nothing is copied from the reference, only the numeric inputs and
outputs of its function are written.  The other fixtures are left untouched.

  python tests/golden/make_golden_cross_scan_c.py        # needs the reference checkout
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, REF, install_stubs, load_file  # noqa: E402

# (name, B, D, L, R, N, with x_proj_bias): the RealSR channel call at C = 48 (D = 1, R = ceil(C/16)), and a general shape
CASES = [("realsr", 3, 1, 48, 3, 16, True), ("general", 2, 2, 40, 4, 8, False)]


def gen_case(realsr, name, B, D, L, R, N, with_bias, seed):
    """output and every gradient of cross_selective_scanC with the arch's WithBias LayerNorm(L) (random affine) as out_norm"""
    torch.manual_seed(seed)
    ins = dict(x=torch.randn(B, D, L), x_proj_weight=0.3 * torch.randn(2, R + 2 * N, D),
               dt_projs_weight=0.5 * torch.randn(2, D, R), dt_projs_bias=-4.0 + 0.5 * torch.rand(2, D),
               A_logs=torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(2 * D, 1) + 0.1 * torch.randn(2 * D, N),
               Ds=1.0 + 0.2 * torch.randn(2 * D))
    if with_bias:
        ins["x_proj_bias"] = 0.1 * torch.randn(2, R + 2 * N)
    ins = {k: v.clone().requires_grad_() for k, v in ins.items()}
    norm = realsr.LayerNorm(L, "WithBias")  # y is (B, L, 1, D): the norm runs over L, as channel_norm does in SS2D_1
    with torch.no_grad():
        norm.body.weight.copy_(1.0 + 0.2 * torch.randn(L))
        norm.body.bias.copy_(0.1 * torch.randn(L))
    y = realsr.cross_selective_scanC(ins["x"], ins["x_proj_weight"], ins.get("x_proj_bias"), ins["dt_projs_weight"],
                                     ins["dt_projs_bias"], ins["A_logs"], ins["Ds"], norm, nrows=-1, delta_softplus=True)
    g = torch.randn_like(y)
    y.backward(g)
    rec = {f"{name}/{k}": v.detach().numpy() for k, v in ins.items()}
    rec.update({f"{name}/grad/{k}": v.grad.numpy() for k, v in ins.items()})
    rec.update({f"{name}/norm_w": norm.body.weight.detach().numpy(), f"{name}/norm_b": norm.body.bias.detach().numpy(),
                f"{name}/grad/norm_w": norm.body.weight.grad.numpy(), f"{name}/grad/norm_b": norm.body.bias.grad.numpy(),
                f"{name}/y": y.detach().numpy(), f"{name}/dout": g.numpy()})
    return rec


if __name__ == "__main__":
    torch.set_num_threads(8)
    install_stubs()
    load_file("VmambaIR.archs.common", f"{REF}/SRGAN/VmambaIR/archs/common.py")
    realsr = load_file("ref_realsr", f"{REF}/RealSR/VmambaIR/archs/MambaRealSR11_arch.py")
    rec = {}
    for i, case in enumerate(CASES):
        rec.update(gen_case(realsr, *case, seed=31 + i))
    np.savez_compressed(f"{OUT}/cross_selective_scan_c.npz", **rec)
    print("cross_selective_scan_c.npz", sum(v.nbytes for v in rec.values()) // 1024, "KiB")
