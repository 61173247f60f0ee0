"""Stored outputs of the reference's own `selective_scan_cuda_oflex` and `selective_scan_cuda_ndstate` CUDA kernels.
TEST INFRASTRUCTURE ONLY.

tests/test_scan_oflex_gpu.py compares this library's stand-in modules with the reference modules on the same seeded inputs:
  * oflex: bf16 and fp16 inputs, out_float=True (fp32 `out`), backward with an fp32 dout;
  * ndstate: fp32 and bf16 inputs, state dimension 1 (A (D,), B / C (B, G, L)).
The reference extensions are not part of this repository, so their outputs are kept in tests/golden/scan_ref_kernel_oflex.npz in the
layout of oracle/ref_kernel_golden.py: inputs regenerated from fixed seeds on the CPU, the large outputs at 4096 seeded sample points
each, the per-channel reductions (dA, dD, ddelta_bias) whole.

Regenerate on a GPU after building oracle/_ref/ (oracle/build_ref_oflex.py, needs a checkout of the reference project):
  python -m oracle.ref_kernel_golden_oflex [out.npz]
"""
import os
import sys

import numpy as np
import torch

from oracle.ref_kernel_golden import NAMES, WHOLE, sample  # noqa: F401  (same stored layout)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
GOLDEN = os.path.join(ROOT, "tests", "golden", "scan_ref_kernel_oflex.npz")
CASES = [("oflex", torch.bfloat16), ("oflex", torch.float16), ("ndstate", torch.float32), ("ndstate", torch.bfloat16)]
SHAPE = dict(b=2, dim=192, L=4096, G=4)  # L = 4096: two of the reference's 2048-position chunks, so bwd reads its `x`


def tag(kind, itype):
    return f"{kind}_{str(itype).split('.')[-1]}"


def inputs(kind, itype):
    """the reference test's distributions (test_selective_scan.py:406-441), seeded CPU draws -> (u, delta, A, B, C, D, bias), dout.
    oflex: N = 16, dout fp32;  ndstate: A (D,), B / C (b, G, L), dout in the input dtype."""
    b, dim, L, G = SHAPE["b"], SHAPE["dim"], SHAPE["L"], SHAPE["G"]
    g = torch.Generator().manual_seed(2000 + CASES.index((kind, itype)))
    if kind == "oflex":
        N = 16
        A = -0.5 * torch.rand(dim, N, generator=g)
        Bm = torch.randn(b, G, N, L, generator=g).to(itype)
        Cm = torch.randn(b, G, N, L, generator=g).to(itype)
    else:
        A = -0.5 * torch.rand(dim, generator=g)
        Bm = torch.randn(b, G, L, generator=g).to(itype)
        Cm = torch.randn(b, G, L, generator=g).to(itype)
    D = torch.randn(dim, generator=g)
    bias = 0.5 * torch.rand(dim, generator=g)
    u = torch.randn(b, dim, L, generator=g).to(itype)
    delta = (0.5 * torch.rand(b, dim, L, generator=g)).to(itype)
    dout = torch.randn(b, dim, L, generator=g)
    return (u, delta, A, Bm, Cm, D, bias), (dout if kind == "oflex" else dout.to(itype))


def load():
    """numeric entries as torch tensors; the `<name>_dtype` / `<name>_shape` records of the reference's outputs as numpy arrays"""
    z = np.load(GOLDEN)
    return {k: (torch.from_numpy(z[k]) if z[k].dtype.kind == "f" else z[k]) for k in z.files}


def _module(name):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF_DIR, name + ".so"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def main(out=GOLDEN):
    mods = {"oflex": _module("selective_scan_cuda_oflex"), "ndstate": _module("selective_scan_cuda_ndstate")}
    store = {}
    for kind, itype in CASES:
        args, dout = inputs(kind, itype)
        args = [t.cuda() for t in args]
        ref = mods[kind]
        if kind == "oflex":
            out_r, x_r = ref.fwd(*args, True, 1, True)
        else:
            out_r, x_r = ref.fwd(*args, True, 1)
        grads = ref.bwd(*args, dout.cuda(), x_r, True, 1)
        for n, t in zip(NAMES, (out_r,) + tuple(grads)):
            store[f"{tag(kind, itype)}/{n}"] = sample(n, t).numpy()
            store[f"{tag(kind, itype)}/{n}_dtype"] = np.array(str(t.dtype))
            store[f"{tag(kind, itype)}/{n}_shape"] = np.array(tuple(t.shape))
    np.savez_compressed(out, **store)
    print("wrote", out, os.path.getsize(out), "bytes,", torch.cuda.get_device_name())


if __name__ == "__main__":
    main(*sys.argv[1:])
