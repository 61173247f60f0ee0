"""The differentiable CPU oracle: cscan.Scan (the C oracle's analytic backward as an autograd Function) against a plain float64 torch
recurrence under autograd, and the float64 oracle block (oracle/oss_ref.block under autograd) against the autograd goldens of the real
reference MamberBlock (tests/golden/block_*.npz).  This is the reference tests/test_train_net_gpu.py holds the training path to."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cscan, oss_ref

NAMES = ("du", "ddelta", "dA", "dB", "dC", "dD", "ddelta_bias")


def _recurrence(u, delta, A, B, C, D, bias, softplus):
    """selective_scan_ref (reference test_selective_scan.py:168-234) as a sequential torch loop: u, delta (b,d,L), A (d,N),
    B / C (b,G,N,L) or (b,N,L)"""
    b, d, L = u.shape
    if bias is not None:
        delta = delta + bias[:, None]
    if softplus:
        delta = F.softplus(delta)
    B4 = B if B.dim() == 4 else B[:, None]
    C4 = C if C.dim() == 4 else C[:, None]
    rep = d // B4.shape[1]
    Bd, Cd = B4.repeat_interleave(rep, 1), C4.repeat_interleave(rep, 1)  # (b,d,N,L)
    x = u.new_zeros(b, d, A.shape[1])
    ys = []
    for i in range(L):
        x = torch.exp(delta[:, :, i, None] * A) * x + (delta[:, :, i] * u[:, :, i])[..., None] * Bd[..., i]
        ys.append((x * Cd[..., i]).sum(-1))
    y = torch.stack(ys, -1)
    return y if D is None else y + u * D[:, None]


def _inputs(G, has_D, has_bias, L, seed):
    g = torch.Generator().manual_seed(seed)
    b, d, N = 2, 8, 5
    r = lambda *s: torch.randn(*s, generator=g)
    Bshape = (b, N, L) if G == 1 else (b, G, N, L)  # G = 1 as the 3-d layout (cscan._shapes)
    ins = [r(b, d, L), 0.5 * r(b, d, L), -0.5 - torch.rand(d, N, generator=g), r(*Bshape), r(*Bshape),
           r(d) if has_D else None, 0.5 * torch.rand(d, generator=g) if has_bias else None]
    return [None if t is None else t.float().double() for t in ins], r(b, d, L).float().double()  # fp32-rounded, as the C oracle reads


def _run(fn, ins, dout, dtype):
    leaves = [None if t is None else t.to(dtype).detach().requires_grad_() for t in ins]
    y = fn(*leaves)
    y.backward(dout.to(dtype))
    return y.detach(), [None if t is None else t.grad for t in leaves]


@pytest.mark.parametrize("L", [1, 7, 33])
@pytest.mark.parametrize("has_D,has_bias", [(True, True), (False, True), (True, False), (False, False)])
@pytest.mark.parametrize("G", [1, 2, 4])
def test_scan_function_matches_float64_autograd_recurrence(G, has_D, has_bias, L):
    cscan.use_host_threads()
    ins, dout = _inputs(G, has_D, has_bias, L, seed=G * 100 + L + 10 * has_D + 20 * has_bias)
    y, got = _run(lambda *t: cscan.Scan.apply(*t, True), ins, dout, torch.float64)
    yr, ref = _run(lambda *t: _recurrence(*t, True), ins, dout, torch.float64)
    assert y.dtype == torch.float64
    assert float((y - yr).abs().max()) <= 1e-10 * float(yr.abs().max())
    for n, a, r, t in zip(NAMES, got, ref, ins):
        if t is None:
            assert a is None, n
            continue
        assert a.dtype == torch.float64 and a.shape == t.shape, n
        err, scale = float((a - r).abs().max()), float(r.abs().max())
        assert (scale > 0 or (n == "dA" and L == 1)) and err <= 1e-10 * scale, (n, err, scale)  # L = 1: A never acts, dA = 0
    # float32 mode: the same recurrence and analytic backward evaluated sequentially in fp32.  Bound: at most 33 sequential steps of
    # a few fp32 roundings each on O(1) values, with the dA / dD / ddelta_bias sums over b * L = 66 terms: 5e-6 of the largest value
    # (5.5e-7 measured)
    y32, got32 = _run(lambda *t: cscan.Scan.apply(*t, True), ins, dout, torch.float32)
    assert y32.dtype == torch.float32
    assert float((y32.double() - y).abs().max()) <= 5e-6 * float(y.abs().max())
    for n, a, r in zip(NAMES, got32, got):
        if r is None:
            continue
        assert a.dtype == torch.float32
        err, scale = float((a.double() - r).abs().max()), float(r.abs().max())
        assert err <= 5e-6 * scale, (n, err, scale)


@pytest.mark.parametrize("tag", ["sisr_c48", "realsr_c32"])
def test_float64_oracle_block_matches_reference_autograd(golden_dir, tag):
    """y, dx and every parameter gradient of oss_ref.block in float64 autograd vs the real reference block's (fp32 autograd):
    within 1e-4 of each tensor's max |golden| (3.4e-5 measured)"""
    cscan.use_host_threads()
    z = np.load(os.path.join(golden_dir, f"block_{tag}.npz"))
    sd = {k[3:]: torch.from_numpy(z[k]).double().requires_grad_() for k in z.files if k.startswith("sd/")}
    x = torch.from_numpy(z["x"]).double().requires_grad_()
    y = oss_ref.block(sd, "", x, "mul")
    y.backward(torch.from_numpy(z["dout"]).double())
    checks = [("y", y.detach()), ("dx", x.grad)] + [(f"grad/{n}", p.grad) for n, p in sd.items()]
    assert {k for k, _ in checks} == {k for k in z.files if not k.startswith("sd/") and k not in ("x", "dout", "attn_out")}
    for k, got in checks:
        ref = torch.from_numpy(z[k]).double()
        assert got is not None and got.shape == ref.shape, k
        err = float((got - ref).abs().max())
        if k.endswith("conv_cout.bias"):
            # the true gradient is 0: a constant added in front of channel_norm.  The golden holds the reference's fp32 round-off
            assert float(got.abs().max()) < 1e-9, (k, float(got.abs().max()))
            continue
        assert err <= 1e-4 * float(ref.abs().max()), (k, err, float(ref.abs().max()))


@pytest.mark.parametrize("store", [None, torch.bfloat16])
def test_grad_enabled_forward_is_bit_identical(golden_dir, store):
    """the oracle under autograd (cscan.Scan, the _Store rounding Function) computes the same forward, bit for bit, as without grad --
    with STORE_DTYPE unset (the fp32 oracle of the inference parity tests), and with the bf16-storage emulation"""
    cscan.use_host_threads()
    z = np.load(os.path.join(golden_dir, "block_sisr_c48.npz"))
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}
    x = torch.from_numpy(z["x"])
    oss_ref.STORE_DTYPE = store
    try:
        with torch.no_grad():
            y0 = oss_ref.block(sd, "", x, "mul")
        sdg = {k: v.clone().requires_grad_() for k, v in sd.items()}
        y1 = oss_ref.block(sdg, "", x.clone().requires_grad_(), "mul")
        y1.sum().backward()
    finally:
        oss_ref.STORE_DTYPE = None
    assert y1.dtype == torch.float32 and torch.equal(y1.detach(), y0)
    assert all(p.grad is not None for p in sdg.values())
