"""Pins the module-level CPU oracle (oracle/oss_ref.py) against outputs of the REAL reference modules
(fixtures written by tests/golden/make_golden.py from the reference project)."""
import os

import numpy as np
import pytest
import torch

from oracle import oss_ref


def _sd(z):
    return {k[3:]: torch.from_numpy(z[k]) for k in z if k.startswith("sd/")}


@pytest.mark.parametrize("tag,gate", [("sisr_c48", "mul"), ("m32_c32", "add"), ("m33_c32", "mul"), ("realsr_c32", "mul")])
def test_block_oracle_matches_reference(golden_dir, tag, gate):
    z = np.load(os.path.join(golden_dir, f"block_{tag}.npz"))
    sd = _sd(z)
    x = torch.from_numpy(z["x"])
    ln = oss_ref._ln(x, sd["norm1.body.weight"], sd["norm1.body.bias"])
    a = oss_ref.ss2d(sd, "attn.", ln, gate)
    torch.testing.assert_close(a, torch.from_numpy(z["attn_out"]), rtol=1e-4, atol=2e-5)
    y = oss_ref.block(sd, "", x, gate)
    torch.testing.assert_close(y, torch.from_numpy(z["y"]), rtol=1e-4, atol=2e-5)


def test_net_oracle_matches_reference(net_sisr_tiny):
    z = net_sisr_tiny
    y = oss_ref.net_forward(_sd(z), torch.from_numpy(z["x"]), "sisr")
    torch.testing.assert_close(y, torch.from_numpy(z["y"]), rtol=1e-4, atol=2e-5)


def test_cross_scan_gather_bit_exact(golden_dir):
    """the four direction orders used by the oracle are exactly the reference's CrossScan / CrossMerge maps."""
    z = np.load(os.path.join(golden_dir, "cross_scan.npz"))
    x = torch.from_numpy(z["x"])
    rows = x.flatten(2)
    cols = x.transpose(2, 3).flatten(2)
    xs = torch.stack([rows, cols, rows.flip(-1), cols.flip(-1)], 1)
    assert torch.equal(xs, torch.from_numpy(z["xs"]))
    ys = torch.from_numpy(z["ys"]).flatten(3)
    B, K, D, L = ys.shape
    H, W = x.shape[2:]
    y = ys[:, 0] + ys[:, 2].flip(-1) + (ys[:, 1] + ys[:, 3].flip(-1)).view(B, D, W, H).transpose(2, 3).reshape(B, D, L)
    assert torch.equal(y, torch.from_numpy(z["y"]))
