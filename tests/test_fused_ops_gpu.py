"""Unit parity of each fused OSS-block stage (through the C-ABI) against the same op in plain fp32 torch."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

TOL = {torch.float32: (1e-4, 1e-4), torch.bfloat16: (3e-2, 3e-2), torch.float16: (4e-3, 4e-3)}


def close(a, b, dtype, scale=1.0):
    rtol, atol = TOL[dtype]
    torch.testing.assert_close(a.float().cpu(), b.float().cpu(), rtol=rtol, atol=atol * scale)


def ln_ref(x, w, b):
    mu = x.mean(1, keepdim=True)
    var = x.var(1, keepdim=True, unbiased=False)
    y = (x - mu) / torch.sqrt(var + 1e-5) if b is not None else x / torch.sqrt(var + 1e-5)
    y = y * w.view(1, -1, 1)
    return y + b.view(1, -1, 1) if b is not None else y


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("K,M,P", [(48, 96, 256), (96, 140, 4096), (127, 48, 100), (384, 768, 64), (1021, 384, 64), (20, 17, 37)])
def test_pixlin_plain(dtype, K, M, P):
    from vmambair_b200 import ops
    torch.manual_seed(K + M)
    x = torch.randn(2, K, P, device="cuda").to(dtype)
    w = (torch.randn(M, K, device="cuda") / K ** 0.5).to(dtype)
    bias = torch.randn(M, device="cuda")
    out = ops.pixlin(x, w, bias)
    ref = torch.einsum("mk,bkp->bmp", w.float(), x.float()) + bias.view(1, -1, 1)
    close(out, ref, dtype)
    out32 = ops.pixlin(x, w, None, out_dtype=torch.float32)
    assert out32.dtype == torch.float32
    close(out32, ref - bias.view(1, -1, 1), dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("K,M,P,B", [(510, 96, 4096, 4), (512, 96, 1024, 2), (1021, 200, 64, 3), (400, 48, 520, 1), (510, 96, 72, 2)])
def test_pixlin_kstream_path(dtype, K, M, P, B, monkeypatch):
    """reduction-heavy plain GEMMs (K > 384: the EFFN / x_proj data gradients of the training path) run the K-streamed kernel:
    against the fp32 contraction and against the resident-K kernel (VMB_PL_KSTREAM=0), bias / SiLU range / residual, strided views"""
    from vmambair_b200 import ops
    torch.manual_seed(K + M)
    big = torch.randn(B, K + 8, P, device="cuda").to(dtype)
    x = big[:, 8:]                                         # channel-offset view
    w = ops.pad_weight((torch.randn(M, K, device="cuda") / K ** 0.5).to(dtype))
    bias = torch.randn(M, device="cuda")
    res = torch.randn(B, M, P, device="cuda").to(dtype)
    ref = torch.einsum("mk,bkp->bmp", w[:, :K].float(), x.float())
    monkeypatch.setenv("VMB_PIXLIN_TC", "0")
    outs = {}
    for ks in ("1", "0"):
        monkeypatch.setenv("VMB_PL_KSTREAM", ks)
        o_plain = ops.pixlin(x, w)
        o_full = ops.pixlin(x, w, bias, residual=res, act=(0, M // 2))
        outs[ks] = (o_plain, o_full)
    close(outs["1"][0], ref, dtype)
    r2 = ref + bias.view(1, -1, 1)
    r2 = torch.cat([F.silu(r2[:, :M // 2]), r2[:, M // 2:]], 1) + res.float()
    close(outs["1"][1], r2, dtype, scale=2.0)
    # same accumulation precision as the resident-K kernel: equal up to the summation order
    assert (outs["1"][0].float() - outs["0"][0].float()).abs().max() <= 2e-2 * ref.abs().max()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("ln_mode", [1, 2])
def test_pixlin_ln_act_residual_gate(dtype, ln_mode):
    from vmambair_b200 import ops
    torch.manual_seed(3)
    B, K, M, P = 2, 96, 192, 320
    x = (torch.randn(B, K, P, device="cuda") * 2 + 0.5).to(dtype)
    w = (torch.randn(M, K, device="cuda") / K ** 0.5).to(dtype)
    bias = torch.randn(M, device="cuda")
    lw, lb = torch.rand(K, device="cuda") + 0.5, torch.randn(K, device="cuda") * 0.1
    out = ops.pixlin(x, w, bias, ln=(ln_mode, lw, lb if ln_mode == 1 else None), act=(96, 192))
    xn = ln_ref(x.float(), lw, lb if ln_mode == 1 else None)
    if dtype != torch.float32:
        xn = xn.to(dtype).float()
    ref = torch.einsum("mk,bkp->bmp", w.float(), xn) + bias.view(1, -1, 1)
    ref = torch.cat([ref[:, :96], F.silu(ref[:, 96:])], 1)
    close(out, ref, dtype)
    # gate prologue + residual epilogue on a strided (channel-offset) input view
    big = torch.randn(B, 2 * K, P, device="cuda").to(dtype)
    xv = big[:, K:]
    res = torch.randn(B, M, P, device="cuda").to(dtype)
    g = torch.randn(B, K, device="cuda")
    for mode in (1, 2):
        out = ops.pixlin(xv, w, bias, residual=res, gate=g, gate_mode=mode)
        xg = xv.float() * (1 + g[:, :, None]) if mode == 1 else xv.float() + g[:, :, None]
        if dtype != torch.float32:
            xg = xg.to(dtype).float()
        ref = torch.einsum("mk,bkp->bmp", w.float(), xg) + bias.view(1, -1, 1) + res.float()
        close(out, ref, dtype, scale=4.0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H,W", [(64, 64), (12, 8), (7, 9)])
def test_dwconv_modes(dtype, H, W):
    from vmambair_b200 import ops
    torch.manual_seed(1)
    B, C = 2, 10
    x = torch.randn(B, 2 * C, H, W, device="cuda").to(dtype)
    w = torch.randn(2 * C, 1, 3, 3, device="cuda") * 0.3
    b = torch.randn(2 * C, device="cuda") * 0.1
    conv = F.conv2d(x.float(), w, b, padding=1, groups=2 * C)
    o0 = ops.dwconv3x3(x.view(B, 2 * C, H * W)[:, :C], w.view(-1, 9)[:C].contiguous(), b[:C].contiguous(), C, H, W, 0)
    close(o0, F.silu(conv[:, :C]).flatten(2), dtype)
    o1 = ops.dwconv3x3(x.view(B, 2 * C, H * W), w.view(-1, 9).contiguous(), b, C, H, W, 1)
    close(o1, (F.gelu(conv[:, :C]) * conv[:, C:]).flatten(2), dtype, scale=2.0)
    o2 = ops.dwconv3x3(x.view(B, 2 * C, H * W), w.view(-1, 9).contiguous(), None, C, H, W, 1)
    conv_nb = F.conv2d(x.float(), w, None, padding=1, groups=2 * C)
    close(o2, (F.gelu(conv_nb[:, :C]) * conv_nb[:, C:]).flatten(2), dtype, scale=2.0)


@pytest.mark.parametrize("H,W", [(64, 64), (16, 24), (5, 3), (72, 40), (128, 136)])
def test_cross_scan_bit_exact(H, W, golden_dir):
    """the six-direction gather must be bit-exact (BASELINE.json): compare with the reference's index maps."""
    from vmambair_b200 import ops
    torch.manual_seed(0)
    B, C = 2, 6
    x = torch.randn(B, C, H, W, device="cuda")
    xs = ops.cross_scan([x.view(B, C, H * W)] * 4, C, H, W)
    rows, cols = x.flatten(2), x.transpose(2, 3).flatten(2)
    ref = torch.stack([rows, cols, rows.flip(-1), cols.flip(-1)], 1)
    assert torch.equal(xs, ref)
    # distinct sources per direction (strided channel views of one tensor)
    big = torch.randn(B, 4, C + 3, H * W, device="cuda")
    out = ops.cross_scan([big[:, k, :C] for k in range(4)], C, H, W)
    v = [big[:, k, :C].reshape(B, C, H, W) for k in range(4)]
    ref = torch.stack([v[0].flatten(2), v[1].transpose(2, 3).flatten(2), v[2].flatten(2).flip(-1),
                       v[3].transpose(2, 3).flatten(2).flip(-1)], 1)
    assert torch.equal(out, ref)
    xb = x.to(torch.bfloat16)
    assert torch.equal(ops.cross_scan([xb.view(B, C, H * W)] * 4, C, H, W)[:, 1], xb.transpose(2, 3).flatten(2))
    # 16-bit, distinct sources, all four orders (the 16 B-vector kernel when H, W are multiples of 8)
    bb = big.to(torch.bfloat16)
    outb = ops.cross_scan([bb[:, k, :C] for k in range(4)], C, H, W)
    vb = [bb[:, k, :C].reshape(B, C, H, W) for k in range(4)]
    refb = torch.stack([vb[0].flatten(2), vb[1].transpose(2, 3).flatten(2), vb[2].flatten(2).flip(-1),
                        vb[3].transpose(2, 3).flatten(2).flip(-1)], 1)
    assert torch.equal(outb, refb)


def test_cross_scan_matches_reference_golden(golden_dir):
    import os
    import numpy as np
    from vmambair_b200 import ops
    z = np.load(os.path.join(golden_dir, "cross_scan.npz"))
    x = torch.from_numpy(z["x"]).cuda()
    B, C, H, W = x.shape
    xs = ops.cross_scan([x.view(B, C, H * W)] * 4, C, H, W)
    assert torch.equal(xs.cpu(), torch.from_numpy(z["xs"]))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C,H,W", [(48, 16, 24), (96, 64, 64), (32, 5, 7)])
def test_merge_norm_gate(dtype, C, H, W):
    from vmambair_b200 import ops
    torch.manual_seed(2)
    B, L = 2, H * W
    ys = torch.randn(B, 4, C, L, device="cuda").to(dtype)
    zbig = torch.randn(B, 2 * C, L, device="cuda").to(dtype)
    z = zbig[:, C:]
    lw, lb = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
    y2, pooled = ops.merge_norm_gate(ys, z, lw, lb, C, H, W)
    f = ys.float()
    y = f[:, 0] + f[:, 2].flip(-1) + f[:, 1].view(B, C, W, H).transpose(2, 3).reshape(B, C, L) \
        + f[:, 3].flip(-1).view(B, C, W, H).transpose(2, 3).reshape(B, C, L)
    yn = ln_ref(y, lw, lb)
    if dtype != torch.float32:
        yn = yn.to(dtype).float()
    ref = yn * z.float()
    close(y2, ref, dtype, scale=2.0)
    torch.testing.assert_close(pooled.cpu(), y2.float().sum(-1).cpu(), rtol=2e-3, atol=2e-2)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C,H,W,B", [(96, 64, 64, 3), (48, 32, 16, 2), (96, 16, 48, 1), (50, 16, 16, 2), (130, 32, 32, 1)])
@pytest.mark.parametrize("inplace", [False, True])
def test_merge_single_kernel_path(dtype, C, H, W, B, inplace, monkeypatch):
    """H, W multiples of 16 and C <= 146: ONE kernel (16 x 16 pixel tiles, all channels per CTA, cp.async ring over the channels).
    Against the fp32 composition, against the two-kernel path (VMB_MERGE_FUSED=0), both direction layouts, SiLU inside or outside,
    and the workspace handed to the backward (merged fp32 values + per-pixel sum / sum of squares)."""
    from vmambair_b200 import ops
    torch.manual_seed(C + H)
    L = H * W
    ys = torch.randn(B, 4, C, L, device="cuda").to(dtype)
    zbig = torch.randn(B, 2 * C, L, device="cuda").to(dtype)
    z = zbig[:, C:]
    lw, lb = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
    f = ys.float()
    T = lambda t: t.view(B, C, W, H).transpose(2, 3).reshape(B, C, L)
    if inplace:
        y = ((f[:, 0] + f[:, 2]) + T(f[:, 1])) + T(f[:, 3])
    else:
        y = ((f[:, 0] + f[:, 2].flip(-1)) + T(f[:, 1])) + T(f[:, 3].flip(-1))
    yn = ln_ref(y, lw, lb).to(dtype).float()
    out = {}
    for fused in ("1", "0"):
        monkeypatch.setenv("VMB_MERGE_FUSED", fused)
        y2a, pa = ops.merge_norm_gate(ys, z, lw, lb, C, H, W, in_place_order=inplace)
        y2b, pb, ws = ops.merge_norm_gate(ys, z, lw, lb, C, H, W, in_place_order=inplace, z_preact=True, return_ws=True)
        out[fused] = (y2a, pa, y2b, pb, ws.view(torch.float32)[:B * C * L + 2 * B * L].clone())
    y2a, pa, y2b, pb, ws = out["1"]
    close(y2a, yn * z.float(), dtype, scale=2.0)
    close(y2b, yn * F.silu(z.float()), dtype, scale=2.0)
    torch.testing.assert_close(pa, y2a.float().sum(-1), rtol=2e-3, atol=2e-2)
    torch.testing.assert_close(pb, y2b.float().sum(-1), rtol=2e-3, atol=2e-2)
    # the merged fp32 values are bit-identical to the two-kernel path (same summation order); the statistics differ by their own
    # summation order over the channels only
    assert torch.equal(ws[:B * C * L], out["0"][4][:B * C * L])
    torch.testing.assert_close(ws[:B * C * L].view(B, C, L), y, rtol=0, atol=0)
    torch.testing.assert_close(ws[B * C * L:], out["0"][4][B * C * L:], rtol=1e-5, atol=1e-4)
    # outputs of the two paths: equal except where the last bit of the statistics moved a rounding boundary
    assert (y2a.float() - out["0"][0].float()).abs().max() <= 2e-2 * y2a.float().abs().max()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("C,H,W", [(48, 16, 24), (96, 64, 64), (32, 8, 8), (16, 40, 24)])
def test_grouped_direction_aware_scan_equals_gathered_scan(dtype, C, H, W):
    """the in-kernel direction handling (transposed sources + reversed walk) reproduces cross_scan + flat scan:
    identical math, outputs returned in each source's own pixel order."""
    from vmambair_b200 import ops
    torch.manual_seed(5)
    B, N, L = 2, 16, H * W
    x = torch.randn(B, C, L, device="cuda").to(dtype)
    dbl = (torch.randn(B, 4, C + 2 * N, L, device="cuda") * 0.5).to(dtype)   # per-direction delta|B|C in NATURAL pixel order
    A = -torch.rand(4 * C, N, device="cuda") - 0.1
    D = torch.randn(4 * C, device="cuda")
    bias = torch.rand(4 * C, device="cuda") - 4.0
    # gathered reference path (already verified against the oracle)
    xs = ops.cross_scan([x] * 4, C, H, W)
    g = ops.cross_scan([dbl[:, k] for k in range(4)], C + 2 * N, H, W)
    ys_ref, _ = ops.selective_scan_fwd(xs.view(B, 4 * C, L), g[:, :, :C].reshape(B, 4 * C, L), A, g[:, :, C:C + N].contiguous(),
                                       g[:, :, C + N:].contiguous(), D, bias, True, need_ckpt=False)
    ys_ref = ys_ref.view(B, 4, C, L)
    # direction-aware path: directions 1,3 read plane-transposed copies
    xt = ops.transpose_hw(x, H, W)
    dt_ = [dbl[:, 0].contiguous(), ops.transpose_hw(dbl[:, 1].contiguous(), H, W), dbl[:, 2].contiguous(),
           ops.transpose_hw(dbl[:, 3].contiguous(), H, W)]
    us = [x, xt, x, xt]
    ys = ops.selective_scan_fwd_grouped(us, [t[:, :C] for t in dt_], [t[:, C:C + N] for t in dt_], [t[:, C + N:] for t in dt_],
                                        [0, 0, 1, 1], A, D, bias, True)
    # map back: k=0 as is; k=2 was written at memory-reversed positions -> flip to scan order; k=1/3 are in transposed order
    torch.testing.assert_close(ys[:, 0].float(), ys_ref[:, 0].float(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ys[:, 1].float(), ys_ref[:, 1].float(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ys[:, 2].flip(-1).float(), ys_ref[:, 2].float(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ys[:, 3].flip(-1).float(), ys_ref[:, 3].float(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("K,M,P,B", [(96, 192, 4096, 2), (48, 96, 256, 3), (96, 510, 1024, 2), (256, 96, 512, 1), (288, 768, 64, 4), (384, 96, 64, 2),
                                     (255, 96, 1024, 2), (127, 48, 512, 2), (48, 254, 1024, 1), (96, 510, 4096, 8)])
def test_pixlin_tcgen05_path(dtype, K, M, P, B, monkeypatch):
    """the persistent tensor-core kernel of pixlin_tc.cu (wgmma; the test keeps its original id), forced on for every legal
    shape, against fp32 torch: plain, LN+SiLU range, gate+residual."""
    from vmambair_b200 import ops
    monkeypatch.setenv("VMB_PIXLIN_TC", "2")
    torch.manual_seed(K + M + P)
    x = (torch.randn(B, K, P, device="cuda") * 1.5 + 0.3).to(dtype)
    w = ops.pad_weight((torch.randn(M, K, device="cuda") / K ** 0.5).to(dtype))
    wf = w[:, :K].float()
    bias = torch.randn(M, device="cuda")
    out = ops.pixlin(x, w, bias)
    close(out, torch.einsum("mk,bkp->bmp", wf, x.float()) + bias.view(1, -1, 1), dtype)
    lw, lb = torch.rand(K, device="cuda") + 0.5, torch.randn(K, device="cuda") * 0.1
    out = ops.pixlin(x, w, bias, ln=(1, lw, lb), act=(M // 2, M))
    xn = ln_ref(x.float(), lw, lb).to(dtype).float()
    ref = torch.einsum("mk,bkp->bmp", wf, xn) + bias.view(1, -1, 1)
    ref = torch.cat([ref[:, :M // 2], F.silu(ref[:, M // 2:])], 1)
    close(out, ref, dtype)
    res = torch.randn(B, M, P, device="cuda").to(dtype)
    g = torch.randn(B, K, device="cuda") * 0.5
    out = ops.pixlin(x, w, None, residual=res, gate=g, gate_mode=1)
    xg = (x.float() * (1 + g[:, :, None])).to(dtype).float()
    close(out, torch.einsum("mk,bkp->bmp", wf, xg) + res.float(), dtype, scale=4.0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("B,C,H,W", [(2, 96, 64, 64), (1, 8, 5, 7), (3, 48, 16, 24)])
def test_pixel_shuffle_nhwc_bit_exact(dtype, B, C, H, W):
    """the SR tail's PixelShuffle(2) on channels-last storage is the same permutation as F.pixel_shuffle"""
    from vmambair_b200 import ops
    torch.manual_seed(B + C + H)
    x = torch.randn(B, 4 * C, H, W, device="cuda").to(dtype)
    out = ops.pixel_shuffle2_nhwc(x.contiguous(memory_format=torch.channels_last))
    ref = F.pixel_shuffle(x, 2)
    assert out.shape == ref.shape and out.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(out.contiguous(), ref)
    # with the deferred conv bias: (x + bias) in fp32, rounded once to the storage dtype, then the same permutation
    bias = torch.randn(4 * C, device="cuda")
    outb = ops.pixel_shuffle2_nhwc(x.contiguous(memory_format=torch.channels_last), bias)
    refb = F.pixel_shuffle((x.float() + bias.view(1, -1, 1, 1)).to(dtype), 2)
    assert torch.equal(outb.contiguous(), refb)


def test_sr_tail_channels_last_matches_plain_tail():
    from vmambair_b200 import archs
    torch.manual_seed(3)
    net = archs.MambaSISR6(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).cuda().eval()
    feat = torch.randn(2, 32, 24, 40, device="cuda")
    with torch.no_grad():
        a = net._tail_channels_last(feat)
        b = net.tail(feat)
    assert a.shape == b.shape and a.is_contiguous()
    torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("variant,dim", [("sisr", 96), ("mamber33", 48), ("realsr", 64), ("mamber32", 40)])
def test_channel_branch_versions_agree(variant, dim, monkeypatch):
    """the channel-direction OSS: restructured kernel (v2, default) against the first version, all model variants"""
    from vmambair_b200 import archs, fused, ops
    torch.manual_seed(dim)
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant=variant).cuda()
    with torch.no_grad():
        for p_ in blk.parameters():
            p_.add_(0.05 * torch.randn_like(p_))
    c = fused._prepare(blk, torch.float32, torch.device("cuda"))
    pooled = torch.randn(5, dim, device="cuda") * 40.0
    monkeypatch.setenv("VMB_CH_V", "1")
    v1 = ops.channel_branch(pooled, 1.0 / 64, c["ch"], dim)
    monkeypatch.setenv("VMB_CH_V", "2")
    v2 = ops.channel_branch(pooled, 1.0 / 64, c["ch"], dim)
    torch.testing.assert_close(v2, v1, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("H,W", [(64, 64), (8, 8), (16, 32), (32, 16), (4, 256)])
def test_dwconv_row_block_kernel_bit_identical(dtype, H, W, monkeypatch):
    """the 4-row / shuffle-halo kernel (default for power-of-two planes) against the strip kernel: same fmaf order"""
    from vmambair_b200 import ops
    torch.manual_seed(H + W)
    B, C = 3, 7
    x = torch.randn(B, 2 * C + 3, H, W, device="cuda").to(dtype)  # channel-offset view: x_cs != H*W rows of a larger tensor
    xin = x.view(B, 2 * C + 3, H * W)[:, 1:2 * C + 1]
    w = (torch.randn(2 * C, 9, device="cuda") * 0.3).contiguous()
    b = torch.randn(2 * C, device="cuda") * 0.1
    outs = {}
    for v in ("1", "2", "3"):  # 3: the row-block kernel with all row loads issued before the arithmetic
        monkeypatch.setenv("VMB_DW_V", v)
        outs[v] = (ops.dwconv3x3(xin[:, :C], w[:C].contiguous(), b[:C].contiguous(), C, H, W, 0),
                   ops.dwconv3x3(xin, w, b, C, H, W, 1), ops.dwconv3x3(xin, w, None, C, H, W, 1),
                   ops.dwconv3x3(xin, w, None, 2 * C, H, W, 2)) + ops.dwconv3x3_t(xin[:, :C], w[:C].contiguous(), b[:C].contiguous(), C, H, W)
    for v in ("2", "3"):
        for a, r in zip(outs[v], outs["1"]):
            assert torch.equal(a, r)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("hw", [(64, 64), (32, 48), (10, 12)])
def test_cross_scan_multi_equals_separate_launches(hw, dtype):
    """vmb_cross_scan_multi (one launch for the x / delta / B|C gathers of a block, one for the du / ddelta / dB / dC scatters of its
    backward) against one vmb_cross_scan per segment: a permutation, so bit-exact; (10, 12) takes the per-segment fallback"""
    from vmambair_b200 import ops
    H, W = hw
    B, C, N, L = 2, 24, 16, H * W
    torch.manual_seed(0)
    xc = torch.randn(B, C, L, device="cuda").to(dtype)
    dbl4 = torch.randn(B, 4, C + 2 * N, L, device="cuda").to(dtype)
    segs = [([xc] * 4, C), ([dbl4[:, k, :C] for k in range(4)], C), ([dbl4[:, k, C:] for k in range(4)], 2 * N)]
    got = ops.cross_scan_multi([(s, r, None) for s, r in segs], H, W)
    for (s, r), g in zip(segs, got):
        assert torch.equal(g, ops.cross_scan(s, r, H, W))
    # scatter direction: four segments, three of them into slices of one tensor, H and W swapped
    du, dd = torch.randn(B, 4 * C, L, device="cuda").to(dtype), torch.randn(B, 4 * C, L, device="cuda").to(dtype)
    dB, dC = torch.randn(B, 4, N, L, device="cuda").to(dtype), torch.randn(B, 4, N, L, device="cuda").to(dtype)
    wide = torch.zeros(B, 4, C + 2 * N, L, device="cuda", dtype=dtype)
    ref = torch.zeros_like(wide)
    back = [([du.view(B, 4, C, L)[:, k] for k in range(4)], C, None), ([dd.view(B, 4, C, L)[:, k] for k in range(4)], C, wide[:, :, :C]),
            ([dB[:, k] for k in range(4)], N, wide[:, :, C:C + N]), ([dC[:, k] for k in range(4)], N, wide[:, :, C + N:])]
    g0 = ops.cross_scan_multi(back, W, H)[0]
    assert torch.equal(g0, ops.cross_scan(back[0][0], C, W, H))
    ops.cross_scan(back[1][0], C, W, H, out=ref[:, :, :C])
    ops.cross_scan(back[2][0], N, W, H, out=ref[:, :, C:C + N])
    ops.cross_scan(back[3][0], N, W, H, out=ref[:, :, C + N:])
    assert torch.equal(wide, ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32, torch.float16])
@pytest.mark.parametrize("geom", [(2, 24, 64, 64), (3, 10, 16, 8), (1, 7, 32, 48), (2, 5, 12, 20)])
def test_dwconv_with_transposed_second_output(geom, dtype):
    """vmb_dwconv3x3_t = vmb_dwconv3x3 (mode 0) + vmb_transpose_hw of its result, from one launch on the row-block path
    ((32, 48) and (12, 20) take the per-pass fallback): bit-identical to the two-pass result"""
    from vmambair_b200 import ops
    B, C, H, W = geom
    torch.manual_seed(7)
    xz = torch.randn(B, 2 * C, H * W, device="cuda").to(dtype)
    w9, b = torch.randn(C, 9, device="cuda"), torch.randn(C, device="cuda")
    ref = ops.dwconv3x3(xz[:, :C], w9, b, C, H, W, 0)
    out, out_t = ops.dwconv3x3_t(xz[:, :C], w9, b, C, H, W)
    assert torch.equal(out, ref)
    assert torch.equal(out_t, ops.transpose_hw(ref, H, W))
    assert torch.equal(out_t.view(B, C, W, H), ref.view(B, C, H, W).transpose(2, 3))
