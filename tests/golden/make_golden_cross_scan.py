#!/usr/bin/env python
"""Generate tests/golden/cross_selective_scan.npz from the REAL reference's cross_selective_scan
(RealSR/VmambaIR/archs/MambaRealSR11_arch.py:371-434), with the reference's own selective_scan_ref as the scan.

Same conventions as make_golden.py, whose helpers it uses (the stubbed `selective_scan_cuda_core` import, the reference
checkout next to this repository or in $VMB_REFERENCE_DIR); nothing is copied from the reference, only the numeric inputs and
outputs of its function are written.  The other fixtures are left untouched.

  python tests/golden/make_golden_cross_scan.py        # needs the reference checkout
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, REF, install_stubs, load_file  # noqa: E402


def gen_cross_selective_scan(realsr):
    """output and every gradient of cross_selective_scan with x_proj_bias and the arch's WithBias LayerNorm as out_norm,
    non-square (H, W) = (8, 12)"""
    torch.manual_seed(21)
    B, D, H, W, N, R = 2, 16, 8, 12, 16, 4
    ins = dict(x=torch.randn(B, D, H, W), x_proj_weight=0.3 * torch.randn(4, R + 2 * N, D), x_proj_bias=0.1 * torch.randn(4, R + 2 * N),
               dt_projs_weight=0.5 * torch.randn(4, D, R), dt_projs_bias=-4.0 + 0.5 * torch.rand(4, D),
               A_logs=torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(4 * D, 1) + 0.1 * torch.randn(4 * D, N),
               Ds=1.0 + 0.2 * torch.randn(4 * D))
    ins = {k: v.clone().requires_grad_() for k, v in ins.items()}
    norm = realsr.LayerNorm(D, "WithBias")
    with torch.no_grad():
        norm.body.weight.copy_(1.0 + 0.2 * torch.randn(D))
        norm.body.bias.copy_(0.1 * torch.randn(D))
    y = realsr.cross_selective_scan(ins["x"], ins["x_proj_weight"], ins["x_proj_bias"], ins["dt_projs_weight"], ins["dt_projs_bias"],
                                    ins["A_logs"], ins["Ds"], norm, nrows=-1, delta_softplus=True)
    g = torch.randn_like(y)
    y.backward(g)
    rec = {k: v.detach().numpy() for k, v in ins.items()}
    rec.update({f"grad/{k}": v.grad.numpy() for k, v in ins.items()})
    rec.update({"norm_w": norm.body.weight.detach().numpy(), "norm_b": norm.body.bias.detach().numpy(),
                "grad/norm_w": norm.body.weight.grad.numpy(), "grad/norm_b": norm.body.bias.grad.numpy(),
                "y": y.detach().numpy(), "dout": g.numpy()})
    np.savez_compressed(f"{OUT}/cross_selective_scan.npz", **rec)
    print("cross_selective_scan.npz", sum(v.nbytes for v in rec.values()) // 1024, "KiB")


if __name__ == "__main__":
    torch.set_num_threads(8)
    install_stubs()
    load_file("VmambaIR.archs.common", f"{REF}/SRGAN/VmambaIR/archs/common.py")
    gen_cross_selective_scan(load_file("ref_realsr", f"{REF}/RealSR/VmambaIR/archs/MambaRealSR11_arch.py"))
