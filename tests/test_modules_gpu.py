"""GPU parity of the drop-in modules (through the C-ABI kernels) against golden outputs of the real
reference modules and against the CPU module oracle."""
import os

import numpy as np
import pytest
import torch

import vmambair_b200.archs as archs
from oracle import oss_ref

pytestmark = pytest.mark.gpu

# fp32 parity: cuDNN/cuBLAS must not silently use TF32 for the library convs/GEMMs outside the OSS kernels
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def _load_block(golden_dir, tag, variant, dim):
    z = np.load(os.path.join(golden_dir, f"block_{tag}.npz"))
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias",
                            variant=variant)
    blk.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}, strict=True)
    return blk.cuda(), z


CASES = [("sisr_c48", "sisr", 48), ("m32_c32", "mamber32", 32), ("m33_c32", "mamber33", 32), ("realsr_c32", "realsr", 32)]


@pytest.mark.parametrize("tag,variant,dim", CASES)
def test_block_forward_golden(golden_dir, tag, variant, dim):
    blk, z = _load_block(golden_dir, tag, variant, dim)
    x = torch.from_numpy(z["x"]).cuda()
    with torch.no_grad():
        y_inf = blk(x)                   # inference path (fused kernels)
    y_trn = blk.forward_compose(x)       # training path
    ref = torch.from_numpy(z["y"])
    torch.testing.assert_close(y_trn.detach().cpu(), ref, rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(y_inf.cpu(), ref, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("tag,variant,dim", [CASES[0], CASES[3]])
def test_block_backward_golden(golden_dir, tag, variant, dim):
    blk, z = _load_block(golden_dir, tag, variant, dim)
    x = torch.from_numpy(z["x"]).cuda().requires_grad_()
    y = blk.forward_compose(x)
    y.backward(torch.from_numpy(z["dout"]).cuda())
    ref = torch.from_numpy(z["dx"])
    assert (x.grad.cpu() - ref).abs().max() <= 2e-3 * ref.abs().max() + 1e-5
    for n, p in blk.named_parameters():
        r = torch.from_numpy(z[f"grad/{n}"])
        err = (p.grad.cpu() - r).abs().max()
        if n.endswith("conv_cout.bias"):  # a constant added before channel_norm: its true gradient is exactly 0, both sides are round-off
            assert err < 2e-2, (n, float(err))
            continue
        assert err <= 3e-3 * r.abs().max().clamp_min(1e-6) + 1e-5, (n, float(err), float(r.abs().max()))


def test_tiny_net_golden(net_sisr_tiny):
    z = net_sisr_tiny
    net = archs.MambaSISR6(dim=8, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).eval()
    net.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z if k.startswith("sd/")}, strict=True)
    net = net.cuda()
    with torch.no_grad():
        y = net(torch.from_numpy(z["x"]).cuda())
    torch.testing.assert_close(y.cpu(), torch.from_numpy(z["y"]), rtol=1e-3, atol=1e-4)


def test_config1_block_c48_64x64_vs_cpu_oracle():
    """BASELINE config 1: single OSS block forward, B=1 C=48 64x64, fp32 -- GPU vs the CPU oracle."""
    torch.manual_seed(0)
    blk = archs.MamberBlock(dim=48, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias")
    x = torch.randn(1, 48, 64, 64)
    sd = {k: v.detach().clone() for k, v in blk.state_dict().items()}
    ref = oss_ref.block(sd, "", x)
    blk = blk.cuda()
    with torch.no_grad():
        y = blk(x.cuda())
    torch.testing.assert_close(y.cpu(), ref, rtol=1e-3, atol=1e-4)


def test_bf16_inference_engine_close_to_fp32_oracle():
    from vmambair_b200.engine import InferenceEngine
    torch.manual_seed(0)
    net = archs.MambaSISR6(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1)
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    x = torch.rand(2, 3, 32, 32)
    ref = oss_ref.net_forward(sd, x, "sisr")
    eng = InferenceEngine(net, 2, 32, 32, dtype=torch.bfloat16)
    y = eng.run(x.to(torch.bfloat16)).float()
    assert (y - ref).abs().max() < 0.08 and (y - ref).abs().mean() < 0.01
    y2 = eng.run(x.to(torch.bfloat16)).float()  # graph replay; the pooled sums use fp32 atomics -> last-bit jitter only
    assert (y - y2).abs().max() < 0.02


def test_lowres_parallel_branches_do_not_change_the_result():
    """levels below full resolution on parallel sub-batch branches of the graph (images are independent units)"""
    import copy
    from vmambair_b200.engine import InferenceEngine
    torch.manual_seed(1)
    net = archs.MambaSISR6(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1)
    x = torch.rand(4, 3, 64, 64).to(torch.bfloat16)
    y1 = InferenceEngine(copy.deepcopy(net), 4, 64, 64, dtype=torch.bfloat16).run(x).float().clone()
    y2 = InferenceEngine(copy.deepcopy(net), 4, 64, 64, dtype=torch.bfloat16, lowres_chains=2).run(x).float().clone()
    y4 = InferenceEngine(copy.deepcopy(net), 4, 64, 64, dtype=torch.bfloat16, lowres_chains=4).run(x).float().clone()
    # the scan's lane mapping depends on the number of rows, so the split changes fp32 summation order, nothing else
    assert (y1 - y2).abs().max() < 0.03 and (y1 - y4).abs().max() < 0.03 and (y1 - y2).abs().mean() < 2e-3


@pytest.mark.parametrize("cls,size,batch", [("Mamber32", 256, 1), ("MambaRealSR11", 128, 2)])
def test_large_tiles_fused_path_matches_composed_path(cls, size, batch):
    """BASELINE configs 4 / 5 geometry (deraining 256x256: L = 65 536 at level 1; RealSR 128x128: L = 16 384) through the
    fused inference pipeline against the composed torch + scan-operator path of the same module, fp32"""
    torch.manual_seed(4)
    kw = dict(num_blocks=[1, 1, 1, 1], num_refinement_blocks=1)
    net = getattr(archs, cls)(**kw).cuda().eval()
    x = torch.rand(batch, 3, size, size, device="cuda")
    with torch.no_grad():
        y_fused = net(x)
    with torch.enable_grad():
        y_comp = net(x).detach()
    assert y_fused.shape == y_comp.shape
    torch.testing.assert_close(y_fused, y_comp, rtol=2e-3, atol=2e-4)


def test_unmodified_call_pattern_selective_scan_cuda_core():
    """The B0 boundary: fwd/bwd with the reference binding's signature and return order."""
    import vmambair_b200.selective_scan_cuda_core as core
    torch.manual_seed(0)
    u = torch.randn(1, 8, 70, device="cuda"); dl = torch.rand(1, 8, 70, device="cuda")
    A = -torch.rand(8, 16, device="cuda"); Bm = torch.randn(1, 2, 16, 70, device="cuda"); Cm = torch.randn(1, 2, 16, 70, device="cuda")
    D = torch.randn(8, device="cuda"); bias = torch.rand(8, device="cuda")
    out, x = core.fwd(u, dl, A, Bm, Cm, D, bias, True, 1)
    assert out.shape == u.shape and x.dtype == torch.float32
    g = core.bwd(u, dl, A, Bm, Cm, D, bias, torch.randn_like(out), x, True, 1)
    assert len(g) == 7 and g[0].shape == u.shape and g[2].shape == A.shape and g[3].shape == Bm.shape


def test_wide_net_dim64_falls_back_per_block_and_runs():
    """ADVICE r1: MambaSISR6(dim=64) has a C = 512 latent level, beyond the fused kernels' K <= 384 LayerNorm prologue: that level
    takes the composed path (with a warning), the others the fused kernels, and the result equals the all-composed forward."""
    import warnings
    torch.manual_seed(4)
    net = archs.MambaSISR6(dim=64, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to("cuda").eval()
    x = torch.rand(1, 3, 32, 32, device="cuda")
    with torch.no_grad(), warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        y = net(x)
        assert any("fused OSS block not available" in str(i.message) for i in w)
        from vmambair_b200 import unet
        unet.set_mode("torch")
        try:
            blocks = [m for m in net.modules() if isinstance(m, archs.MamberBlock)]
            fwd = archs.MamberBlock.forward
            archs.MamberBlock.forward = lambda self, t, out=None: self.forward_compose(t)
            ref = net(x)
        finally:
            archs.MamberBlock.forward = fwd
            unet.set_mode("native")
    assert len(blocks) == 8 and torch.isfinite(y).all()
    torch.testing.assert_close(y, ref, rtol=2e-3, atol=2e-4)

