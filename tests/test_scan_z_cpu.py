"""The z-gated selective scan's oracle (the library's scan oracle composed with the gate out * SiLU(z) and its analytic backward)
against golden vectors of the reference's own `selective_scan_ref` with z and return_last_state (tests/golden/make_golden_scan_z.py).
test_scan_z_gpu.py checks the `selective_scan_cuda` stand-in against the same composition."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.selective_scan_ref import selective_scan_oracle, selective_scan_oracle_bwd

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scan_z_ref.npz")
GRADS = ("du", "ddelta", "dA", "dB", "dC", "dz", "dD", "dbias")


def oracle_z_fwd(u, delta, A, B, C, D, z, bias, softplus, dtype=torch.float64):
    """-> (out_z, out, last_state) in `dtype`: the scan oracle on the inputs as given (cast to `dtype`), then out * SiLU(z)"""
    cast = lambda t: None if t is None else t.to(dtype)
    out, last = selective_scan_oracle(*map(cast, (u, delta, A, B, C, D, bias)), softplus, return_last_state=True, dtype=dtype)
    return out * F.silu(cast(z)), out, last


def oracle_z_bwd(u, delta, A, B, C, D, z, bias, dout, softplus, dtype=torch.float64):
    """-> (du, ddelta, dA, dB, dC, dz, dD, dbias): dz = dout * out * s * (1 + z (1 - s)), s = sigmoid(z); the scan's gradients from
    dout * SiLU(z)"""
    _, out, _ = oracle_z_fwd(u, delta, A, B, C, D, z, bias, softplus, dtype)
    z, dout = z.to(dtype), dout.to(dtype)
    s = torch.sigmoid(z)
    dz = dout * out * s * (1 + z * (1 - s))
    du, ddelta, dA, dB, dC, dD, dbias = selective_scan_oracle_bwd(u, delta, A, B, C, D, bias, dout * z * s, softplus, dtype=dtype)
    return du, ddelta, dA, dB, dC, dz, dD, dbias


def golden_cases():
    with np.load(GOLDEN) as f:
        data = {k: torch.from_numpy(f[k]) for k in f.files}
    names = sorted({k.split("/")[0] for k in data})
    return {n: {k.split("/", 1)[1]: v for k, v in data.items() if k.startswith(n + "/")} for n in names}


CASES = golden_cases()


def case_inputs(c):
    return c["u"], c["delta"], c["A"], c["B"], c["C"], c.get("D"), c["z"], c.get("bias")


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_z_matches_reference_function(name):
    c = CASES[name]
    ins = case_inputs(c)
    sp = bool(int(c["softplus"]))
    out_z, _, last = oracle_z_fwd(*ins, sp)
    torch.testing.assert_close(out_z.float(), c["out"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(last.float(), c["last_state"], rtol=1e-4, atol=1e-5)
    grads = oracle_z_bwd(*ins, c["dout"], sp)
    for gname, g in zip(GRADS, grads):
        if gname in c:
            torch.testing.assert_close(g.float(), c[gname], rtol=1e-4, atol=1e-4, msg=f"{name}/{gname}")
        else:
            assert g is None, gname


def test_golden_covers_ragged_lengths_and_groups():
    Ls = {c["u"].shape[-1] for c in CASES.values()}
    assert any(L % 64 for L in Ls) and any(L > 128 for L in Ls)
    assert any(c["B"].shape[1] == 2 for c in CASES.values())
    assert all({"out", "last_state", "dz", "du", "ddelta", "dA", "dB", "dC"} <= set(c) for c in CASES.values())
