"""GPU parity of the TRAINING path (vmambair_b200.fused_train: forward and backward of every fused stage on this library's
kernels) against the reference-autograd goldens (tests/golden/block_*.npz: dx and every parameter gradient of the real
reference MamberBlock) and against the composed torch path."""
import os

import numpy as np
import pytest
import torch

import vmambair_b200.archs as archs

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def _load_block(golden_dir, tag, variant, dim):
    z = np.load(os.path.join(golden_dir, f"block_{tag}.npz"))
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant=variant)
    blk.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}, strict=True)
    return blk.cuda(), z


@pytest.mark.parametrize("tag,variant,dim", [("sisr_c48", "sisr", 48), ("realsr_c32", "realsr", 32)])
def test_block_fused_training_path_matches_reference_autograd(golden_dir, tag, variant, dim):
    """forward value, dx and all parameter gradients of the fused training path vs the goldens of the real reference block"""
    archs.set_train_path("fused")
    blk, z = _load_block(golden_dir, tag, variant, dim)
    x = torch.from_numpy(z["x"]).cuda().requires_grad_()
    y = blk(x)  # grad enabled -> fused_train
    assert y.grad_fn is not None and "Tail" in type(y.grad_fn).__name__
    torch.testing.assert_close(y.detach().cpu(), torch.from_numpy(z["y"]), rtol=1e-3, atol=1e-4)
    y.backward(torch.from_numpy(z["dout"]).cuda())
    ref = torch.from_numpy(z["dx"])
    assert (x.grad.cpu() - ref).abs().max() <= 2e-3 * ref.abs().max() + 1e-5
    for n, p in blk.named_parameters():
        r = torch.from_numpy(z[f"grad/{n}"])
        assert p.grad is not None, n
        err = (p.grad.cpu() - r).abs().max()
        if n.endswith("conv_cout.bias"):  # true gradient exactly 0 (constant added before channel_norm): both sides round-off
            assert err < 2e-2, (n, float(err))
            continue
        assert err <= 3e-3 * r.abs().max().clamp_min(1e-6) + 1e-5, (n, float(err), float(r.abs().max()))


@pytest.mark.parametrize("variant,dim", [("mamber32", 32), ("mamber33", 32)])
def test_block_fused_training_path_matches_composed_autograd(variant, dim):
    """additive channel gate (Mamber32) and dc_inner = 2 (Mamber33): fused training path vs torch autograd over the composed path"""
    torch.manual_seed(3)
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant=variant).cuda()
    x = torch.randn(2, dim, 16, 24, device="cuda")
    dout = torch.randn(2, dim, 16, 24, device="cuda")
    grads = {}
    for path in ("fused", "compose"):
        archs.set_train_path(path)
        blk.zero_grad(set_to_none=True)
        xx = x.clone().requires_grad_()
        blk(xx).backward(dout)
        grads[path] = [xx.grad.clone()] + [p.grad.clone() for p in blk.parameters()]
    archs.set_train_path("fused")
    names = ["x"] + [n for n, _ in blk.named_parameters()]
    for n, a, b in zip(names, grads["fused"], grads["compose"]):
        tol = 2e-2 if n.endswith("conv_cout.bias") else 3e-3 * float(b.abs().max().clamp_min(1e-6)) + 1e-5
        assert float((a - b).abs().max()) <= tol, (n, float((a - b).abs().max()), float(b.abs().max()))


@pytest.mark.parametrize("variant,dim", [("sisr", 48), ("mamber32", 32)])
def test_direct_grad_accumulation_equals_autograd_accumulation(variant, dim):
    """fused_train.set_direct_grads(True) (what optim.FlatAdam switches on): the backward kernels add into existing fp32 .grad buffers
    and autograd receives None -- the resulting .grad must equal the AccumulateGrad route, including accumulation over two backwards"""
    from vmambair_b200 import fused_train
    torch.manual_seed(7)
    archs.set_train_path("fused")
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant=variant).cuda()
    x = torch.randn(2, dim, 16, 24, device="cuda")
    dout = torch.randn(2, dim, 16, 24, device="cuda")
    res = {}
    try:
        for direct in (False, True):
            fused_train.set_direct_grads(direct)
            for p in blk.parameters():
                p.grad = torch.zeros_like(p)
            ptrs = [p.grad.data_ptr() for p in blk.parameters()]
            for _ in range(2):  # two micro-steps accumulate
                xx = x.clone().requires_grad_()
                blk(xx).backward(dout)
            assert ptrs == [p.grad.data_ptr() for p in blk.parameters()]  # the buffers were written in place
            res[direct] = [xx.grad.clone()] + [p.grad.clone() for p in blk.parameters()]
    finally:
        fused_train.set_direct_grads(False)
    names = ["x"] + [n for n, _ in blk.named_parameters()]
    for n, a, b in zip(names, res[True], res[False]):
        tol = 2e-2 if n.endswith("conv_cout.bias") else 1e-4 * float(b.abs().max().clamp_min(1e-6)) + 1e-6
        assert float((a - b).abs().max()) <= tol, (n, float((a - b).abs().max()), float(b.abs().max()))
    assert all(float(g.abs().max()) > 0 for n, g in zip(names, res[True]) if not n.endswith("conv_cout.bias")), "a gradient stayed zero"


@pytest.mark.parametrize("amp", [False, True])
def test_side_stream_weight_gradients_equal_single_stream_on_a_net(amp):
    """the weight-gradient kernels on the second stream (fused_train._Side) vs everything on one stream: a 4-level net with FlatAdam's
    flat gradient buffer, eager and replayed from a CUDA graph.  fp32 activations: only the order of the fp32 atomic adds differs
    (1e-4); bf16 autocast: the forward itself is reproducible only up to bf16 rounding flips behind the out_norm statistics'
    atomics (0 ... 2e-3 on the output, 2e-3 ... 1e-2 on the gradients between identical single-stream runs),
    so that case only guards against gross errors (a missing or doubled weight gradient is O(1))."""
    import torch.nn.functional as F
    from vmambair_b200 import fused_train
    from vmambair_b200.optim import FlatAdam
    torch.manual_seed(11)
    archs.set_train_path("fused")
    net = archs.MambaSISR6(dim=16, num_blocks=[2, 1, 1, 1], num_refinement_blocks=2).cuda().train()
    opt = FlatAdam(net.parameters(), lr=1e-4)
    lq, gt = torch.rand(2, 3, 32, 32, device="cuda"), torch.rand(2, 3, 128, 128, device="cuda")
    tol = 5e-2 if amp else 1e-4

    def fwd_bwd():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            out = net(lq)
        loss = F.l1_loss(out.float(), gt)
        loss.backward()
        return loss

    dist = lambda a, b: float((a - b).norm() / b.norm())
    res = {}
    try:
        for side in (False, True):
            fused_train._Side.on = side
            opt.flat_grad.zero_()
            fwd_bwd()
            torch.cuda.synchronize()
            res[side] = opt.flat_grad.clone()
        assert float(res[False].abs().max()) > 0
        assert dist(res[True], res[False]) <= tol, dist(res[True], res[False])
        # CUDA-graph capture of the forked / joined backward
        fused_train._Side.on = True
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            opt.flat_grad.zero_()
            fwd_bwd()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        opt.check_views()
        opt.flat_grad.zero_()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fwd_bwd()
        for _ in range(2):
            opt.flat_grad.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert dist(opt.flat_grad, res[False]) <= tol, dist(opt.flat_grad, res[False])
    finally:
        fused_train._Side.on = True
        fused_train.set_direct_grads(False)


@pytest.mark.parametrize("B,M,K,L", [(4, 510, 96, 4096), (2, 96, 255, 1024), (1, 35, 48, 520), (3, 192, 96, 256)])
@pytest.mark.parametrize("per_batch", [False, True])
def test_pixlin_wgrad_matches_fp32_contraction(B, M, K, L, per_batch):
    """dW[m,k] = sum_{b,p} dy[b,m,p] x[b,k,p]: the split-pixel mma.sync kernel (bf16 in, fp32 accumulate) vs an fp32 einsum of the
    same bf16-rounded operands; also through channel-offset views (strided rows)."""
    from vmambair_b200 import ops
    torch.manual_seed(B * 7 + M)
    dy_full = torch.randn(B, M + 8, L, device="cuda").to(torch.bfloat16)
    dy = dy_full[:, 8:]  # a channel-offset view, like the d z_pre half of dxz
    x = torch.randn(B, K, L, device="cuda").to(torch.bfloat16)
    got = ops.pixlin_wgrad(dy, x, per_batch=per_batch)
    ref = torch.einsum("bmp,bkp->bmk", dy.float(), x.float())
    ref = ref if per_batch else ref.sum(0)
    assert got.dtype == torch.float32 and got.shape == ref.shape
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-2 * float(ref.abs().max()) * 1e-2 + 1e-3)


@pytest.mark.parametrize("variant,dim", [("sisr", 48), ("mamber32", 96), ("mamber33", 32), ("realsr", 64)])
def test_channel_branch_backward_matches_torch_autograd(variant, dim):
    """vmb_channel_branch_bwd (one CTA per image) vs torch autograd over SS2D_1.cforward_pooled: dpooled and every channel parameter"""
    from vmambair_b200 import fused_train
    torch.manual_seed(11)
    a = archs.SS2D_1(d_model=dim, ssm_ratio=1, variant=variant).cuda()
    L = 24 * 16
    pooled = (torch.randn(3, dim, device="cuda") * L * 0.3)
    dc = torch.randn(3, dim, device="cuda")
    names = [n for n, _ in a.named_parameters()]
    res = {}
    for path in ("kernel", "torch"):
        a.zero_grad(set_to_none=True)
        pp = pooled.clone().requires_grad_()
        c = fused_train.channel_gate(a, pp, L) if path == "kernel" else a.cforward_pooled(pp * (1.0 / L))
        if path == "kernel":
            assert "Channel" in type(c.grad_fn).__name__
        c.backward(dc)
        res[path] = (c.detach().clone(), pp.grad.clone(), {n: (p.grad.clone() if p.grad is not None else None) for n, p in a.named_parameters()})
    ck, dpk, gk = res["kernel"]
    ct, dpt, gt = res["torch"]
    torch.testing.assert_close(ck, ct, rtol=1e-3, atol=1e-4)
    assert (dpk - dpt).abs().max() <= 2e-3 * dpt.abs().max() + 1e-7
    for n in names:
        if gt[n] is None:
            continue
        assert gk[n] is not None, n
        tol = 2e-2 if n.endswith("conv_cout.bias") else 3e-3 * float(gt[n].abs().max().clamp_min(1e-6)) + 1e-6
        assert float((gk[n] - gt[n]).abs().max()) <= tol, (n, float((gk[n] - gt[n]).abs().max()), float(gt[n].abs().max()))
