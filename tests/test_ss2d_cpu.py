"""CPU tests of the standalone OSS module: SS2D_1.forward_compose (scan routed to the CPU oracle) against the real reference SS2D_1
classes at ssm_ratio 1 and 2 (expanded width E != d_model), on an L % 8 == 0 and an L % 8 != 0 geometry
(tests/golden/make_golden_ss2d.py)."""
import glob
import os

import numpy as np
import pytest
import torch

import vmambair_b200.archs as archs
from oracle.selective_scan_ref import selective_scan_oracle

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = sorted(os.path.basename(p)[5:-4] for p in glob.glob(os.path.join(_GOLDEN, "ss2d_*.npz")))


@pytest.fixture
def oracle_scan(monkeypatch):
    def fn(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
        return selective_scan_oracle(u, delta, A, B, C, D, delta_bias, delta_softplus)
    monkeypatch.setattr(archs, "selective_scan_fn", fn)


def load_ss2d(golden_dir, case):
    """-> (SS2D_1 with the fixture's state_dict, the fixture's arrays)"""
    z = np.load(os.path.join(golden_dir, f"ss2d_{case}.npz"))
    variant = case.split("_r")[0]
    m = archs.SS2D_1(d_model=int(z["d_model"]), ssm_ratio=float(z["ssm_ratio"]), variant=variant)
    m.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}, strict=True)
    return m, z


def test_fixtures_cover_both_ratios_and_geometries():
    assert len(CASES) == 16
    for v in archs.VARIANTS:
        for r in (1, 2):
            assert {f"{v}_r{r}_8x12", f"{v}_r{r}_7x9"} <= set(CASES)


@pytest.mark.parametrize("case", CASES)
def test_ss2d_forward_matches_reference_golden(golden_dir, oracle_scan, case):
    m, z = load_ss2d(golden_dir, case)
    assert m.d_inner == int(float(z["ssm_ratio"]) * int(z["d_model"]))
    with torch.no_grad():
        y = m.forward_compose(torch.from_numpy(z["x"]))
    torch.testing.assert_close(y, torch.from_numpy(z["y"]), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("case", CASES)
def test_ss2d_backward_matches_reference_golden(golden_dir, oracle_scan, case):
    m, z = load_ss2d(golden_dir, case)
    x = torch.from_numpy(z["x"]).requires_grad_()
    m.forward_compose(x).backward(torch.from_numpy(z["dout"]))
    torch.testing.assert_close(x.grad, torch.from_numpy(z["dx"]), rtol=1e-3, atol=1e-4)
    for n, p in m.named_parameters():
        ref = torch.from_numpy(z[f"grad/{n}"])
        if n.endswith("conv_cout.bias"):  # true gradient exactly 0 (a constant added before channel_norm): both sides round-off
            assert (p.grad - ref).abs().max() < 1e-3, n
            continue
        scale = ref.abs().max().clamp_min(1e-6)
        assert (p.grad - ref).abs().max() <= 2e-3 * scale + 1e-5, n
