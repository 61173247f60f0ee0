"""Stored outputs of the reference's own selective-scan CUDA kernel.  TEST INFRASTRUCTURE ONLY.

tests/test_bench_parity_gpu.py compares this library's scan with selective_scan_cuda_core.fwd / .bwd of the reference at
u (b, 4*96, 4096).  The reference extension is not part of this repository, so its outputs are kept in
tests/golden/scan_ref_kernel.npz: the inputs are regenerated from fixed seeds on the CPU, the large outputs are kept at
4096 seeded sample points each, the per-channel reductions (dA, dD, ddelta_bias) whole.

Regenerate on a GPU after building oracle/_ref/ (oracle/build_ref.py, needs a checkout of the reference project):
  python -m oracle.ref_kernel_golden [out.npz]
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "selective_scan_cuda_core.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "scan_ref_kernel.npz")
CASES = [(b, itype) for b in (8, 4, 1) for itype in (torch.float32, torch.bfloat16)]
NAMES = ("out", "du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias")
WHOLE = ("dA", "dD", "ddelta_bias")
NSAMPLE = 4096


def tag(b, itype):
    return f"b{b}_{str(itype).split('.')[-1]}"


def inputs(b, itype, dim=384, L=4096, G=4, N=16):
    """distributions of the reference test (test_selective_scan.py:406-441), seeded CPU draws -> (u, delta, A, B, C, D, bias), dout"""
    g = torch.Generator().manual_seed(1000 * b + (1 if itype == torch.bfloat16 else 0))
    A = -0.5 * torch.rand(dim, N, generator=g)
    Bm = torch.randn(b, G, N, L, generator=g).to(itype)
    Cm = torch.randn(b, G, N, L, generator=g).to(itype)
    D = torch.randn(dim, generator=g)
    bias = 0.5 * torch.rand(dim, generator=g)
    u = torch.randn(b, dim, L, generator=g).to(itype)
    delta = (0.5 * torch.rand(b, dim, L, generator=g)).to(itype)
    dout = torch.randn(b, dim, L, generator=g).to(itype)
    return (u, delta, A, Bm, Cm, D, bias), dout


def sample(name, t):
    """the stored view of output `name`: whole for the per-channel reductions, else NSAMPLE seeded flat positions (fp32)"""
    t = t.detach().float().cpu().reshape(-1)
    if name in WHOLE:
        return t
    idx = torch.randint(0, t.numel(), (NSAMPLE,), generator=torch.Generator().manual_seed(7 + NAMES.index(name)))
    return t[idx]


def load():
    z = np.load(GOLDEN)
    return {k: torch.from_numpy(z[k]) for k in z.files}


def main(out=GOLDEN):
    import importlib.util
    spec = importlib.util.spec_from_file_location("selective_scan_cuda_core", REF_SO)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    store = {}
    for b, itype in CASES:
        args, dout = inputs(b, itype)
        args = [t.cuda() for t in args]
        out_r, x_r = ref.fwd(*args, True, 1)
        grads = ref.bwd(*args, dout.cuda(), x_r, True, 1)
        for n, t in zip(NAMES, (out_r,) + tuple(grads)):
            store[f"{tag(b, itype)}/{n}"] = sample(n, t).numpy()
    np.savez_compressed(out, **store)
    print("wrote", out, os.path.getsize(out), "bytes,", torch.cuda.get_device_name())


if __name__ == "__main__":
    main(*sys.argv[1:])
