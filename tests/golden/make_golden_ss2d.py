#!/usr/bin/env python
"""Generate the standalone-SS2D_1 golden fixtures from the REAL reference (see make_golden.py for where the checkout is found).

Nothing here is copied from the reference: its SS2D_1 classes are imported at run time, with the scan stubbed to the reference's
own selective_scan_ref (make_golden.install_stubs), run on the CPU on seeded inputs, and only their numeric inputs / outputs are
written to tests/golden/ss2d_<variant>_r<ssm_ratio>_<H>x<W>.npz.

  python tests/golden/make_golden_ss2d.py       # needs the reference checkout

Classes exercised (SS2D_1 on its own: no norm1 in front, no residual or FFN behind, expanded width E = ssm_ratio * d_model):
  * sisr       SRGAN/VmambaIR/archs/MambaSISR6_arch.py:222-498
  * mamber32   Deraining/basicsr/models/archs/mamber32_arch.py (additive channel gate)
  * mamber33   Deraining/basicsr/models/archs/mamber33_arch.py (dc_inner = 2)
  * realsr     RealSR/VmambaIR/archs/MambaRealSR11_arch.py:540-832
Each file holds the state_dict ("sd/<key>"), x, y, a seeded dout, dx and every parameter gradient ("grad/<name>").
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402

OUT = mg.OUT

# (ssm_ratio, d_model): E = 32 at ssm_ratio 2 (d_model != E), E = d_model = 24 at ssm_ratio 1
MODELS = [(1, 24), (2, 16)]
GEOMS = [(8, 12), (7, 9)]  # L = 96 (L % 8 == 0: direction-aware scan) and L = 63 (the gathered path)


def gen_ss2d(variant, mod, ratio, d_model, H, W):
    torch.manual_seed(1000 * ratio + 10 * H + W)
    m = mod.SS2D_1(d_model=d_model, ssm_ratio=ratio)
    # randomise the params that init to constants so every term is exercised (as make_golden.gen_block)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("body.weight") or n.endswith("Ds") or n.endswith("Dsc"):
                p.data = p.data.clone() + 0.2 * torch.randn(p.shape)
            if n.endswith("body.bias"):
                p.data = p.data.clone() + 0.1 * torch.randn(p.shape)
            if n.endswith("A_logs") or n.endswith("Ac_logs"):
                p.data = p.data.clone() + 0.1 * torch.randn(p.shape)
    x = torch.randn(2, d_model, H, W)
    xi = x.clone().requires_grad_()
    y = m(xi)
    g = torch.randn_like(y)
    y.backward(g)
    rec = {"x": x.numpy(), "y": y.detach().numpy(), "dout": g.numpy(), "dx": xi.grad.numpy(),
           "d_model": np.array(d_model), "ssm_ratio": np.array(ratio)}
    for n, p in m.named_parameters():
        rec[f"grad/{n}"] = p.grad.numpy()
    for k, v in mg.np_state(m.state_dict()).items():
        rec[f"sd/{k}"] = v
    name = f"ss2d_{variant}_r{ratio}_{H}x{W}.npz"
    np.savez_compressed(f"{OUT}/{name}", **rec)
    print(name, sum(v.nbytes for v in rec.values()) // 1024, "KiB")


if __name__ == "__main__":
    torch.set_num_threads(8)
    mg.install_stubs()
    mg.load_file("VmambaIR.archs.common", f"{mg.REF}/SRGAN/VmambaIR/archs/common.py")
    mods = {
        "sisr": mg.load_file("ref_sisr", f"{mg.REF}/SRGAN/VmambaIR/archs/MambaSISR6_arch.py"),
        "mamber32": mg.load_file("ref_m32", f"{mg.REF}/Deraining/basicsr/models/archs/mamber32_arch.py"),
        "mamber33": mg.load_file("ref_m33", f"{mg.REF}/Deraining/basicsr/models/archs/mamber33_arch.py"),
        "realsr": mg.load_file("ref_realsr", f"{mg.REF}/RealSR/VmambaIR/archs/MambaRealSR11_arch.py"),
    }
    for variant, mod in mods.items():
        for ratio, d_model in MODELS:
            for H, W in GEOMS:
                gen_ss2d(variant, mod, ratio, d_model, H, W)
