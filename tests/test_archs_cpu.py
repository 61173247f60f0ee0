"""CPU tests of the drop-in modules: state_dict identity with the reference archs (manifest produced from
the real reference classes by tests/golden/make_golden.py) and module math against golden block outputs, with
the scan operator routed to the CPU oracle (the product path itself has no CPU fallback)."""
import json
import os

import numpy as np
import pytest
import torch

import vmambair_b200.archs as archs
from oracle.selective_scan_ref import selective_scan_oracle


def _manifest(golden_dir):
    return json.load(open(os.path.join(golden_dir, "state_dict_manifest.json")))


CTORS = {
    "MambaSISR6_default": lambda: archs.MambaSISR6(),
    "MambaSISR6_full": lambda: archs.MambaSISR6(num_blocks=[15, 1, 1, 1], num_refinement_blocks=15),
    "MambaRealSR11_default": lambda: archs.MambaRealSR11(),
    "Mamber32_derain": lambda: archs.Mamber32(num_blocks=[3, 5, 7, 9], num_refinement_blocks=2),
    "Mamber33_default": lambda: archs.Mamber33(num_blocks=[1, 1, 1, 1], num_refinement_blocks=1),
}


@pytest.mark.parametrize("name", list(CTORS))
def test_state_dict_keys_and_shapes_match_reference(golden_dir, name):
    ref = _manifest(golden_dir)[name]
    net = CTORS[name]()
    ours = {k: list(v.shape) for k, v in net.state_dict().items()}
    assert set(ours) == set(ref), (sorted(set(ours) - set(ref))[:5], sorted(set(ref) - set(ours))[:5])
    bad = {k: (ours[k], ref[k]) for k in ref if ours[k] != ref[k]}
    assert not bad, list(bad.items())[:5]
    assert all(v.dtype == torch.float32 for v in net.state_dict().values())


@pytest.fixture
def oracle_scan(monkeypatch):
    def fn(u, delta, A, B, C, D=None, delta_bias=None, delta_softplus=False, nrows=1):
        return selective_scan_oracle(u, delta, A, B, C, D, delta_bias, delta_softplus)
    monkeypatch.setattr(archs, "selective_scan_fn", fn)


def _load_block(golden_dir, tag, variant, dim):
    z = np.load(os.path.join(golden_dir, f"block_{tag}.npz"))
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias",
                            variant=variant)
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}
    blk.load_state_dict(sd, strict=True)
    return blk, z


@pytest.mark.parametrize("tag,variant,dim", [("sisr_c48", "sisr", 48), ("m32_c32", "mamber32", 32),
                                             ("m33_c32", "mamber33", 32), ("realsr_c32", "realsr", 32)])
def test_block_forward_matches_reference_golden(golden_dir, oracle_scan, tag, variant, dim):
    blk, z = _load_block(golden_dir, tag, variant, dim)
    x = torch.from_numpy(z["x"])
    with torch.no_grad():
        y = blk.forward_compose(x)
        a = blk.attn.forward_compose(blk.norm1(x))
    torch.testing.assert_close(a, torch.from_numpy(z["attn_out"]), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(y, torch.from_numpy(z["y"]), rtol=1e-4, atol=1e-5)


def test_block_backward_matches_reference_golden(golden_dir, oracle_scan):
    blk, z = _load_block(golden_dir, "realsr_c32", "realsr", 32)
    x = torch.from_numpy(z["x"]).requires_grad_()
    y = blk.forward_compose(x)
    y.backward(torch.from_numpy(z["dout"]))
    torch.testing.assert_close(x.grad, torch.from_numpy(z["dx"]), rtol=1e-3, atol=1e-4)
    for n, p in blk.named_parameters():
        ref = torch.from_numpy(z[f"grad/{n}"])
        scale = ref.abs().max().clamp_min(1e-6)
        assert (p.grad - ref).abs().max() <= 2e-3 * scale + 1e-5, n


def test_tiny_net_matches_reference_golden(net_sisr_tiny, oracle_scan):
    z = net_sisr_tiny
    net = archs.MambaSISR6(dim=8, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).eval()
    net.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z if k.startswith("sd/")}, strict=True)
    with torch.no_grad():
        y = net(torch.from_numpy(z["x"]))
    torch.testing.assert_close(y, torch.from_numpy(z["y"]), rtol=1e-4, atol=1e-5)


def test_init_statistics_follow_reference_inits():
    torch.manual_seed(0)
    m = archs.SS2D_1(d_model=48, ssm_ratio=1)
    A = -torch.exp(m.A_logs)
    torch.testing.assert_close(A[0], -torch.arange(1, 17, dtype=torch.float32), rtol=1e-6, atol=1e-6)
    assert torch.all(m.Ds == 1)
    dt = torch.nn.functional.softplus(m.dt_projs_bias)
    assert dt.min() >= 1e-4 - 1e-7 and dt.max() <= 0.1 + 1e-6
    assert m.dt_projs_weight.abs().max() <= 3 ** -0.5 + 1e-6
    assert getattr(m.A_logs, "_no_weight_decay", False) and getattr(m.Ds, "_no_weight_decay", False)


def test_c_abi_exports_every_declared_symbol():
    import re
    from vmambair_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "vmambair_b200.h")).read()
    declared = set(re.findall(r"\b(vmb_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    lib = _lib.lib()  # loads, resolves every symbol
    assert lib.vmb_version().decode().startswith("vmambair_b200")
    assert lib.vmb_scan_ckpt_interval() == 64


def test_product_path_has_no_cpu_fallback():
    from vmambair_b200 import ops
    with pytest.raises(RuntimeError):
        t = torch.zeros(1, 4, 8)
        ops.selective_scan_fwd(t, t, torch.zeros(4, 16), torch.zeros(1, 1, 16, 8), torch.zeros(1, 1, 16, 8))


def test_pack_conv3x3_weight_layout():
    """[tap = 3 ky + kx][Cout -> x64][Cin -> x16], zero padded: a conv evaluated tap by tap from the packed tensor = F.conv2d"""
    import torch.nn.functional as F
    from vmambair_b200 import ops
    torch.manual_seed(0)
    w = torch.randn(5, 7, 3, 3)
    x = torch.randn(2, 7, 6, 9)
    wp = ops.pack_conv3x3_weight(w, torch.float32)
    assert wp.shape == (9, 64, 16) and float(wp[:, 5:].abs().max()) == 0 and float(wp[:, :, 7:].abs().max()) == 0
    xp = F.pad(x, (1, 1, 1, 1))
    y = sum(torch.einsum("mk,bkhw->bmhw", wp[3 * ky + kx, :5, :7], xp[:, :, ky:ky + 6, kx:kx + 9]) for ky in range(3) for kx in range(3))
    torch.testing.assert_close(y, F.conv2d(x, w, padding=1), rtol=1e-5, atol=1e-5)


def test_conv3x3_store_mode_formulas_match_torch_shuffles():
    """include/vmambair_b200.h documents the vmb_conv3x3 store modes as index formulas; they must be nn.PixelUnshuffle(2) /
    nn.PixelShuffle(2) / F.interpolate(..., 'nearest') exactly (the kernels implement the formulas; this pins the formulas)"""
    import torch.nn.functional as F
    torch.manual_seed(1)
    B, M, H, W = 2, 8, 6, 10
    y = torch.randn(B, M, H, W)
    un = torch.empty(B, 4 * M, H // 2, W // 2)
    sh = torch.empty(B, M // 4, 2 * H, 2 * W)
    for m in range(M):
        for yy in range(H):
            for xx in range(W):
                un[:, 4 * m + 2 * (yy % 2) + xx % 2, yy // 2, xx // 2] = y[:, m, yy, xx]
                sh[:, m // 4, 2 * yy + (m // 2) % 2, 2 * xx + m % 2] = y[:, m, yy, xx]
    assert torch.equal(un, F.pixel_unshuffle(y, 2)) and torch.equal(sh, F.pixel_shuffle(y, 2))
    s = 2
    add = torch.randn(B, M, H // s, W // s)
    near = torch.empty(B, M, H, W)
    for yy in range(H):
        for xx in range(W):
            near[:, :, yy, xx] = add[:, :, yy // s, xx // s]
    assert torch.equal(near, F.interpolate(add, scale_factor=s, mode="nearest"))
    # cross-scan orders documented for vmb_cross_scan(_multi): pi_1(w*H + h) = h*W + w and the reversed orders
    Hh, Ww = 3, 5
    img = torch.arange(Hh * Ww).view(Hh, Ww)
    col_major = torch.tensor([img[h, w] for w in range(Ww) for h in range(Hh)])
    assert torch.equal(col_major, img.t().contiguous().view(-1))
