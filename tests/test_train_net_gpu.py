"""Gradients of the training path (vmambair_b200.fused_train) against float64 autograd of the module oracle (oracle/oss_ref.py, its scan
the C oracle's analytic backward: cscan.Scan), block by block at the training net's level shapes and for the benchmarked training step
end to end (vmambair_b200.train_bench: MambaSISR6 [15,1,1,1]+15, 4 x 3x64x64 LQ, bf16 autocast, one CUDA graph, gradients straight into
FlatAdam's flat buffer, weight gradients on the side stream).  The oracle's torch ops run in float64 on the GPU, its scan on the CPU.

Bounds, per tensor (y, dx and every parameter gradient), printed beside each check:
  * fp32 (TF32 off): max|got - ref64| <= max(2e-4 max|ref64|, 2 max|ref32 - ref64|), ref32 = the oracle in float32 (fp32 scan, TF32 off)
    -- the convention of tests/test_gan_gpu.py and tests/test_perceptual_gpu.py;
  * bf16 autocast: against emu = the oracle with bf16 storage (oss_ref.STORE_DTYPE) in float64 arithmetic, the yardstick of
    tests/test_bench_parity_gpu.py extended to gradients: max err <= 3 x emu's + 1e-3 max|ref64|, mean |err| <= 1.5 x emu's + 1e-4 max|ref64|.
Two groups take a different bound, each for the reason given at CHANNEL and _check.
"""
import time
import warnings

import pytest
import torch

import vmambair_b200.archs as archs
from oracle import cscan, oss_ref
from vmambair_b200 import fused, fused_train

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

GATE = {"sisr": "mul", "realsr": "mul", "mamber32": "add", "mamber33": "mul"}


# The channel-direction parameters get their gradients from B x C numbers, the pooled sums and the gate gradient dc, each a sum over
# all L pixels; the kernels sum them in another order than the sequential oracle, and under bf16 from another rounding pattern.  One
# sample of the yardstick does not bound a second there: measured, fp32 realsr C = 384 attn.Dsc at 3.4 x ref32's error (a cancelling
# sum: ref32 itself is 3.3e-4 of max|ref64| off), bf16 sisr C = 192 16x16 attn.dtc_projs_* at 8.7 x emu's max error (3.5e-2 of
# max|ref64|), and the mean over their few elements is no second statistic.  So: fp32 4 x the ref32 multiple instead of 1 x (the kernels sum with
# fp32 atomics, their order varies from run to run), bf16 a floor of 5e-2 of
# max|ref64| on the max error and no mean criterion.  Their fp32 cases still hold them to 2e-4 of max|ref64| where ref32 is tight.
CHANNEL = ("attn.conv_cin.", "attn.xc_proj_weight", "attn.dtc_projs_", "attn.Ac_logs", "attn.Dsc", "attn.conv_cout.weight")


def _channel(name):  # a block's parameter ("attn.Dsc") or a net's ("refinement.14.attn.Dsc")
    return any(("." + name).find("." + p) >= 0 for p in CHANNEL)


def _check(tag, got, ref64, yard, bf16, k32=2):
    """-> list of failure strings for the tensors of `got` ({name: tensor}); yard: ref32 (fp32) or emu (bf16), same keys;
    k32: the multiple of ref32's error the fp32 bound allows"""
    bad = []
    for k in ref64:
        g, r, e = got[k], ref64[k], yard[k]
        assert g is not None and g.shape == r.shape, (tag, k)
        err = (g.double() - r).abs()
        dy = (e - r).abs()
        scale = float(r.abs().max())
        if k.endswith("conv_cout.bias"):
            # true gradient 0 (a constant added in front of channel_norm): the float64 references hold no round-off to measure ours
            # by, ours holds its fp32 sum's.  Absolute bound of tests/test_train_gpu.py (measured up to 1.8e-3)
            ok = float(err.max()) <= 2e-2
            line = f"{tag} {k}: max {float(err.max()):.3e} <= 2e-2 (true gradient 0)"
        elif bf16 and _channel(k):
            lim_max = max(3 * float(dy.max()) + 1e-3 * scale, 5e-2 * scale)
            ok = float(err.max()) <= lim_max
            line = (f"{tag} {k}: max {float(err.max()):.3e} <= {lim_max:.3e} (channel direction; emu max {float(dy.max()):.3e}, "
                    f"max|ref| {scale:.3e})")
        elif bf16:
            lim_max, lim_mean = 3 * float(dy.max()) + 1e-3 * scale, 1.5 * float(dy.mean()) + 1e-4 * scale
            ok = float(err.max()) <= lim_max and float(err.mean()) <= lim_mean
            line = (f"{tag} {k}: max {float(err.max()):.3e} <= {lim_max:.3e}, mean {float(err.mean()):.3e} <= {lim_mean:.3e} "
                    f"(emu max {float(dy.max()):.3e} mean {float(dy.mean()):.3e}, max|ref| {float(r.abs().max()):.3e})")
        else:
            lim = max(2e-4 * scale, (4 * k32 if _channel(k) else k32) * float(dy.max()))
            ok = float(err.max()) <= lim
            line = (f"{tag} {k}: max {float(err.max()):.3e} <= {lim:.3e} "
                    f"(ref32 max {float(dy.max()):.3e}, max|ref| {float(r.abs().max()):.3e})")
        print(("ok   " if ok else "FAIL ") + line)
        if not ok:
            bad.append(line)
    return bad


def _leaves(mod, dtype):
    return {k: v.detach().to(dtype).clone().requires_grad_() for k, v in mod.state_dict().items()}


def _with_store(store, fn):
    oss_ref.STORE_DTYPE = store
    try:
        with torch.autocast("cuda", enabled=False):
            return fn()
    finally:
        oss_ref.STORE_DTYPE = None


# ----------------------------------------------------------------------------- one block at each level shape of the training net
def _oracle_block(blk, x, dout, gate, dtype, store=None):
    sd = _leaves(blk, dtype)
    xx = x.detach().to(dtype).requires_grad_()

    def run():
        y = oss_ref.block(sd, "", xx, gate)
        y.backward(dout.to(dtype))
        return y.detach()

    y = _with_store(store, run)
    return {"y": y, "dx": xx.grad, **{k: p.grad for k, p in sd.items()}}


CASES = [("sisr", 48, 64), ("sisr", 96, 64), ("sisr", 96, 32), ("sisr", 192, 16), ("sisr", 384, 8),
         ("realsr", 48, 64), ("realsr", 384, 8), ("mamber32", 48, 64), ("mamber33", 48, 64)]


@pytest.mark.parametrize("amp", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("variant,C,H", CASES)
def test_block_gradients_match_float64_oracle(variant, C, H, amp, monkeypatch):
    """MamberBlock at B = 4 on the fused training path (fp32, or bf16 x under autocast as the net feeds its blocks) vs oss_ref.block in
    float64 autograd on the same rounded x, the same perturbed parameters and the same seeded dout"""
    cscan.use_host_threads()
    archs.set_train_path("fused")
    g = torch.Generator().manual_seed(C * 1000 + H + sum(map(ord, variant)))
    torch.manual_seed(C + H)
    blk = archs.MamberBlock(dim=C, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant=variant)
    with torch.no_grad():  # away from init, where the LayerNorm biases are 0 and the weights 1 and hide dropped terms
        for p in blk.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g))
    blk = blk.cuda()
    dt = torch.bfloat16 if amp else torch.float32
    x = torch.randn(4, C, H, H, generator=g).to(dt).cuda()
    dout = torch.randn(4, C, H, H, generator=g).to(dt).cuda()

    routes, real_gate = [], fused_train.channel_gate

    def spy(a, pooled, L):
        c = real_gate(a, pooled, L)
        routes.append(type(c.grad_fn).__name__)
        return c

    monkeypatch.setattr(fused_train, "channel_gate", spy)
    xx = x.clone().requires_grad_()
    assert fused.unsupported_reason(blk, xx) is None
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            y = blk(xx)
    assert not [w for w in caught if "not available" in str(w.message)]
    assert "Tail" in type(y.grad_fn).__name__, "the fused training path did not run"
    assert y.dtype == dt
    # the channel gate: the _Channel kernels below C = 384, torch autograd at 384, whose (2 dc, 16, C) state history exceeds one CTA's
    # shared memory (fused_train.channel_gate)
    assert len(routes) == 1 and ("Channel" in routes[0]) == (C < 384), routes
    y.backward(dout)
    torch.cuda.synchronize()
    got = {"y": y.detach(), "dx": xx.grad, **{n: p.grad for n, p in blk.named_parameters()}}

    gate = GATE[variant]
    ref64 = _oracle_block(blk, x, dout, gate, torch.float64)
    yard = _oracle_block(blk, x, dout, gate, torch.float64, torch.bfloat16) if amp else _oracle_block(blk, x, dout, gate, torch.float32)
    bad = _check(f"{variant} C={C} {H}x{H} {'bf16' if amp else 'fp32'}", got, ref64, yard, amp)
    assert not bad, "\n".join(bad)


# ----------------------------------------------------------------------------- the benchmarked training step, end to end
def _oracle_net(net, lq, dtype, store=None, gt=None, dout=None):
    """oss_ref.net_forward under autograd, image by image (the parameter gradients are linear in dout: they add up over the images),
    which keeps the float64 graph of the 50 blocks to one image's.  With gt: dout = the L1 gradient at this output, sign(out - gt) / numel.
    -> (out, dout, {name: grad})"""
    sd = _leaves(net, dtype)
    outs, douts = [], []

    def run():
        for i in range(lq.shape[0]):
            out = oss_ref.net_forward(sd, lq[i:i + 1].to(dtype), "sisr")
            d = torch.sign(out.detach().double() - gt[i:i + 1]) / gt.numel() if dout is None else dout[i:i + 1]
            out.backward(d.to(dtype))
            outs.append(out.detach())
            douts.append(d)

    _with_store(store, run)
    return torch.cat(outs), torch.cat(douts), {k: p.grad for k, p in sd.items()}


def test_training_step_gradients_match_float64_oracle():
    """The benchmarked step (train_bench.run_train): the bench net, FlatAdam's flat gradient buffer, bf16 autocast, forward + backward
    warmed up on a side stream, captured in one CUDA graph and replayed; and the same net in fp32, eager, through autograd's .grad.
    Output and every parameter gradient vs the float64 oracle, fed the same upstream gradient: the L1 gradient at the float64
    output, so that a sign flip where out ~ gt cannot decide the result."""
    import bench
    from vmambair_b200.optim import FlatAdam
    cscan.use_host_threads()
    archs.set_train_path("fused")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    net = bench.build_net("full").cuda().train()
    blocks = [m for m in net.modules() if isinstance(m, archs.MamberBlock)]
    assert len(blocks) == 50
    g = torch.Generator().manual_seed(100)
    # bf16-representable LQ: autocast's cast in front of patch_embed is exact, every run sees the same image
    lq = torch.rand(4, 3, 64, 64, generator=g).to(torch.bfloat16).float().cuda()
    gt = torch.rand(4, 3, 256, 256, generator=g).double().cuda()

    out64, dout, ref64 = _oracle_net(net, lq, torch.float64, gt=gt)
    ref64 = {"out": out64, **ref64}
    t_ref = time.time()
    names = [n for n, _ in net.named_parameters()]

    fused_blocks = []
    hooks = [b.register_forward_hook(lambda m, i, o: fused_blocks.append("Tail" in type(o.grad_fn).__name__)) for b in blocks]
    side_on = fused_train._Side.on
    res = {}
    try:
        # ours, as train_bench runs it
        fused_train._Side.on = True
        opt = FlatAdam(net.parameters(), lr=2e-4, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.0, ema_decay=0.999)
        d16 = dout.float()

        def fwd_bwd():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = net(lq)
            out.float().backward(d16)
            return out

        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                opt.flat_grad.zero_()
                fwd_bwd()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        assert fused_blocks == [True] * (2 * len(blocks)), "an OSS block left the fused training path"
        opt.check_views()
        opt.flat_grad.zero_()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out_s = fwd_bwd()
        opt.flat_grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
        o = 0
        got = {"out": out_s.detach().float().clone()}
        for n, p in net.named_parameters():
            got[n] = opt.flat_grad[o:o + p.numel()].view_as(p).clone()
            o += p.numel()
        res["bf16"] = got

        # ours in fp32, eager, through autograd's .grad
        fused_train.set_direct_grads(False)
        fused_blocks.clear()
        for p in net.parameters():
            p.grad = None
        out = net(lq)
        assert fused_blocks == [True] * len(blocks), "an OSS block left the fused training path"
        out.backward(dout.float())
        torch.cuda.synchronize()
        res["fp32"] = {"out": out.detach(), **{n: p.grad for n, p in net.named_parameters()}}
    finally:
        for h in hooks:
            h.remove()
        fused_train.set_direct_grads(False)
        fused_train._Side.on = side_on
    assert set(names) | {"out"} == set(ref64)

    out32, _, ref32 = _oracle_net(net, lq, torch.float32, dout=dout)
    ref32 = {"out": out32, **ref32}
    out_e, _, emu = _oracle_net(net, lq, torch.float64, store=torch.bfloat16, dout=dout)
    emu = {"out": out_e, **emu}
    # fp32 through 50 blocks: ours and ref32 each carry one sample of round-off compounded over every backward stage, ours from
    # fp32 atomics whose order changes run to run, over ~1 600 tensors.  Two runs of the same code put the gradient of
    # encoder_level1.5.attn.out_norm.body.weight at 0.9 x and 1.01 x of 2 x ref32's error, so the net takes 4 x (the blocks keep 2 x)
    bad = _check("net fp32", res["fp32"], ref64, ref32, False, k32=4) + _check("net bf16", res["bf16"], ref64, emu, True)
    print(f"training-step test: float64 oracle {t_ref - t0:.1f} s, all {time.time() - t0:.1f} s, "
          f"peak GPU memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
    assert not bad, "\n".join(bad)
