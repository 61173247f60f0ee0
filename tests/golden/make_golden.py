#!/usr/bin/env python
"""Generate golden fixtures from the REAL reference (a checkout of the reference project next to this repository,
../reference, or $VMB_REFERENCE_DIR).

Nothing here is copied from the reference: its functions are
AST-extracted / imported at run time, executed on seeded inputs, and only
their numeric inputs/outputs are written to tests/golden/*.npz|json.

  python tests/golden/make_golden.py            # needs the reference checkout

Sources exercised:
  * selective_scan_ref         Mamba/kernels/selective_scan/test_selective_scan.py:168-234
  * MamberBlock / SS2D_1 (SISR)   SRGAN/VmambaIR/archs/MambaSISR6_arch.py:222-515
  * MamberBlock (Mamber32/33)   Deraining/basicsr/models/archs/mamber32_arch.py, mamber33_arch.py
  * MamberBlock (RealSR)        RealSR/VmambaIR/archs/MambaRealSR11_arch.py
  * MambaSISR6 (tiny config)    SRGAN/VmambaIR/archs/MambaSISR6_arch.py:557-643
The reference archs import `selective_scan_cuda_core`; we give them a stub whose
fwd/bwd are the reference's own selective_scan_ref (+ autograd through it).
"""
import ast
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F
from einops import rearrange, repeat

OUT = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("VMB_REFERENCE_DIR") or os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(OUT))), "reference")


def load_ref_scan():
    path = f"{REF}/Mamba/kernels/selective_scan/test_selective_scan.py"
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "selective_scan_ref"][0]
    ns = {"torch": torch, "F": F, "rearrange": rearrange, "repeat": repeat}
    exec(compile(ast.Module([fn], []), path, "exec"), ns)
    return ns["selective_scan_ref"]


REF_SCAN = load_ref_scan()


def install_stubs():
    """sys.modules stubs so the reference arch files import on CPU."""
    reg = types.ModuleType("basicsr.utils.registry")

    class _Reg:
        def register(self, *a, **k):
            return lambda c: c
    reg.ARCH_REGISTRY = _Reg()
    for name in ("basicsr", "basicsr.utils"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["basicsr.utils.registry"] = reg
    fv = types.ModuleType("fvcore.nn")
    fv.flop_count = fv.parameter_count = lambda *a, **k: None
    sys.modules.setdefault("fvcore", types.ModuleType("fvcore"))
    sys.modules["fvcore.nn"] = fv
    timm = types.ModuleType("timm.models.layers")
    timm.DropPath = torch.nn.Identity
    timm.trunc_normal_ = torch.nn.init.trunc_normal_
    timm.to_2tuple = lambda x: (x, x)
    sys.modules.setdefault("timm", types.ModuleType("timm"))
    sys.modules.setdefault("timm.models", types.ModuleType("timm.models"))
    sys.modules["timm.models.layers"] = timm

    core = types.ModuleType("selective_scan_cuda_core")

    def fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, nrows):
        out = REF_SCAN(u, delta, A, B, C, D, None, delta_bias, delta_softplus)
        return [out, torch.zeros(1)]

    def bwd(u, delta, A, B, C, D, delta_bias, dout, x, delta_softplus, nrows):
        ins = [t.detach().clone().requires_grad_() if t is not None else None
               for t in (u, delta, A, B, C, D, delta_bias)]
        with torch.enable_grad():
            out = REF_SCAN(ins[0], ins[1], ins[2], ins[3], ins[4], ins[5], None, ins[6], delta_softplus)
        grads = torch.autograd.grad(out, [t for t in ins if t is not None], dout)
        it = iter(grads)
        return [next(it) if t is not None else None for t in ins]
    core.fwd, core.bwd = fwd, bwd
    sys.modules["selective_scan_cuda_core"] = core
    sys.modules["selective_scan_cuda_oflex"] = core
    sys.modules["selective_scan_cuda"] = core
    # VmambaIR.archs.common -> the real file
    for name in ("VmambaIR", "VmambaIR.archs"):
        sys.modules.setdefault(name, types.ModuleType(name))


def load_file(modname, path):
    spec = importlib.util.spec_from_file_location(modname, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[modname] = mod
    spec.loader.exec_module(mod)
    return mod


def np_state(sd):
    return {k: v.detach().numpy() for k, v in sd.items()}


def gen_scan_cases():
    cases = {}
    specs = [  # (name, b, D, L, N, G, has_D, has_bias, softplus)
        ("a", 2, 8, 64, 16, 2, True, True, True),
        ("b", 1, 12, 100, 16, 4, True, True, True),
        ("c", 2, 6, 257, 8, 1, False, False, False),
        ("d", 1, 8, 48, 16, 2, True, False, True),
        ("e", 1, 4, 1, 16, 1, True, True, True),
    ]
    for name, b, Dm, L, N, G, hD, hb, sp in specs:
        torch.manual_seed(100 + ord(name))
        # distributions of the reference test (test_selective_scan.py:406-441)
        A = -0.5 * torch.rand(Dm, N)
        Bm = torch.randn(b, G, N, L)
        Cm = torch.randn(b, G, N, L)
        Dv = torch.randn(Dm) if hD else None
        bias = 0.5 * torch.rand(Dm) if hb else None
        u = torch.randn(b, Dm, L)
        delta = 0.5 * torch.rand(b, Dm, L)
        ins = [t.clone().requires_grad_() if t is not None else None for t in (u, delta, A, Bm, Cm, Dv, bias)]
        out, last = REF_SCAN(ins[0], ins[1], ins[2], ins[3], ins[4], ins[5], None, ins[6], sp, True)
        g = torch.randn_like(out)
        grads = torch.autograd.grad(out, [t for t in ins if t is not None], g)
        it = iter(grads)
        gl = [next(it) if t is not None else None for t in ins]
        rec = dict(u=u, delta=delta, A=A, B=Bm, C=Cm, out=out.detach(), last_state=last.detach(), dout=g,
                   du=gl[0], ddelta=gl[1], dA=gl[2], dB=gl[3], dC=gl[4])
        if hD:
            rec.update(D=Dv, dD=gl[5])
        if hb:
            rec.update(bias=bias, dbias=gl[6])
        for k, v in rec.items():
            cases[f"{name}/{k}"] = v.numpy()
        cases[f"{name}/softplus"] = np.array(int(sp))
    np.savez(f"{OUT}/scan_cases.npz", **cases)
    print("scan_cases.npz", sum(v.nbytes for v in cases.values()) // 1024, "KiB")


def gen_block(tag, mod, dim, H, W, with_grad):
    torch.manual_seed(7)
    blk = mod.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias")
    # randomise the params that init to constants so every term is exercised
    with torch.no_grad():
        for n, p in blk.named_parameters():
            # (.data = ...: some reference params are expanded views and cannot be updated in place)
            if n.endswith("body.weight") or n.endswith("Ds") or n.endswith("Dsc"):
                p.data = p.data.clone() + 0.2 * torch.randn(p.shape)
            if n.endswith("body.bias"):
                p.data = p.data.clone() + 0.1 * torch.randn(p.shape)
            if n.endswith("A_logs") or n.endswith("Ac_logs"):
                p.data = p.data.clone() + 0.1 * torch.randn(p.shape)
    x = torch.randn(2, dim, H, W)
    rec = {}
    if with_grad:
        xi = x.clone().requires_grad_()
        y = blk(xi)
        g = torch.randn_like(y)
        y.backward(g)
        rec["dout"] = g.numpy()
        rec["dx"] = xi.grad.numpy()
        for n, p in blk.named_parameters():
            rec[f"grad/{n}"] = p.grad.numpy()
    else:
        with torch.no_grad():
            y = blk(x)
    # intermediate: SS2D output alone
    with torch.no_grad():
        rec["attn_out"] = blk.attn(blk.norm1(x)).numpy()
    rec["x"] = x.numpy()
    rec["y"] = y.detach().numpy()
    for k, v in np_state(blk.state_dict()).items():
        rec[f"sd/{k}"] = v
    np.savez_compressed(f"{OUT}/block_{tag}.npz", **rec)
    print(f"block_{tag}.npz", sum(v.nbytes for v in rec.values()) // 1024, "KiB")


def gen_net(sisr):
    torch.manual_seed(11)
    net = sisr.MambaSISR6(dim=8, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).eval()
    x = torch.rand(1, 3, 16, 24)
    with torch.no_grad():
        y = net(x)
    rec = {"x": x.numpy(), "y": y.numpy()}
    for k, v in np_state(net.state_dict()).items():
        rec[f"sd/{k}"] = v.astype(np.float32)
    # two compressed files, neither above 1 MB (tests/conftest.py::net_sisr_tiny merges them)
    big = "sd/up4_3.body.0.weight"
    np.savez_compressed(f"{OUT}/net_sisr_tiny.npz", **{k: v for k, v in rec.items() if k != big})
    np.savez_compressed(f"{OUT}/net_sisr_tiny_up4_3.npz", **{big: rec[big]})
    print("net_sisr_tiny.npz", sum(v.nbytes for v in rec.values()) // 1024, "KiB")


def gen_manifests(mods):
    man = {}
    ctor = {
        "MambaSISR6_default": lambda: mods["sisr"].MambaSISR6(),
        "MambaSISR6_full": lambda: mods["sisr"].MambaSISR6(num_blocks=[15, 1, 1, 1], num_refinement_blocks=15),
        "MambaRealSR11_default": lambda: mods["realsr"].MambaRealSR11(),
        "Mamber32_derain": lambda: mods["m32"].Mamber32(num_blocks=[3, 5, 7, 9], num_refinement_blocks=2),
        "Mamber33_default": lambda: mods["m33"].Mamber33(num_blocks=[1, 1, 1, 1], num_refinement_blocks=1),
    }
    for name, fn in ctor.items():
        net = fn()
        man[name] = {k: list(v.shape) for k, v in net.state_dict().items()}
        print(name, len(man[name]), "keys", sum(int(np.prod(s)) for s in man[name].values()), "params")
    json.dump(man, open(f"{OUT}/state_dict_manifest.json", "w"))


def gen_cross_scan(realsr):
    """bit-exact gather maps (CrossScan / CrossMerge, MambaRealSR11_arch.py:325-355)."""
    torch.manual_seed(3)
    x = torch.randn(1, 2, 3, 5)
    xs = realsr.CrossScan.apply(x)
    ys = torch.randn(1, 4, 2, 3, 5)
    y = realsr.CrossMerge.apply(ys)
    np.savez(f"{OUT}/cross_scan.npz", x=x.numpy(), xs=xs.numpy(), ys=ys.numpy(), y=y.numpy())


if __name__ == "__main__":
    torch.set_num_threads(8)
    install_stubs()
    load_file("VmambaIR.archs.common", f"{REF}/SRGAN/VmambaIR/archs/common.py")
    mods = {
        "sisr": load_file("ref_sisr", f"{REF}/SRGAN/VmambaIR/archs/MambaSISR6_arch.py"),
        "m32": load_file("ref_m32", f"{REF}/Deraining/basicsr/models/archs/mamber32_arch.py"),
        "m33": load_file("ref_m33", f"{REF}/Deraining/basicsr/models/archs/mamber33_arch.py"),
        "realsr": load_file("ref_realsr", f"{REF}/RealSR/VmambaIR/archs/MambaRealSR11_arch.py"),
    }
    gen_scan_cases()
    gen_cross_scan(mods["realsr"])
    gen_block("sisr_c48", mods["sisr"], 48, 16, 24, with_grad=True)
    gen_block("m32_c32", mods["m32"], 32, 12, 8, with_grad=False)
    gen_block("m33_c32", mods["m33"], 32, 12, 8, with_grad=False)
    gen_block("realsr_c32", mods["realsr"], 32, 12, 8, with_grad=True)
    gen_net(mods["sisr"])
    gen_manifests(mods)
