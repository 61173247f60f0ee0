"""Direction-aware grouped scan with checkpoints and its backward (vmb_selective_scan_fwd_grouped / _bwd_grouped), and the differentiable
four-direction operator built on them (vmambair_b200.cross_scan: cross_selective_scan, CrossScan, CrossMerge), against the flat scan
on gathered operands, a torch composition of the reference's operator, and the reference's own outputs
(tests/golden/cross_selective_scan.npz, RealSR/VmambaIR/archs/MambaRealSR11_arch.py:325-434)."""
import os

import numpy as np
import pytest
import torch

import vmambair_b200.archs as archs
from vmambair_b200 import cross_scan as cs
from vmambair_b200 import ops
from vmambair_b200.selective_scan import selective_scan_fn

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

BWD_TOL = {torch.float32: 2e-3, torch.float16: 6e-3, torch.bfloat16: 4e-2}  # test_scan_gpu.py backward bounds


def _gen(seed):
    g = torch.Generator().manual_seed(seed)
    return lambda *s: torch.randn(*s, generator=g), lambda *s: torch.rand(*s, generator=g)


def _grouped_operands(b, C, L, N, dtype, seed, sliced=False):
    """the operator's layout: u of groups 0/2 = x, of 1/3 = x^T (own tensors); delta / B / C slices of two (B, 2, C+2N, L) tensors.
    sliced: every source is a channel-slice view of a wider tensor."""
    rn, r = _gen(seed)
    pad = 8 if sliced else 0
    xw = rn(b, C + 2 * pad, L)
    xtw = rn(b, C + 2 * pad, L)
    RN = C + 2 * N
    d02 = rn(b, 2, RN + pad, L)
    d13 = rn(b, 2, RN + pad, L)
    for d in (d02, d13):
        d[:, :, :C] = 0.5 * r(b, 2, C, L)
    cast = lambda t: t.to(dtype).cuda()
    xw, xtw, d02, d13 = map(cast, (xw, xtw, d02, d13))
    x, xt = xw[:, pad:pad + C], xtw[:, pad:pad + C]
    d02, d13 = d02[:, :, pad:], d13[:, :, pad:]
    src = [(x, d02[:, 0]), (xt, d13[:, 0]), (x, d02[:, 1]), (xt, d13[:, 1])]
    us = [s[0] for s in src]
    deltas = [s[1][:, :C] for s in src]
    Bs = [s[1][:, C:C + N] for s in src]
    Cs = [s[1][:, C + N:C + 2 * N] for s in src]
    A = (-0.5 * r(4 * C, N)).cuda()
    Dv = rn(4 * C).cuda()
    bias = (0.5 * r(4 * C)).cuda()
    return us, deltas, Bs, Cs, A, Dv, bias


def _seq(t, rev):
    """memory order of a group's tensor -> its sequence order"""
    return t.flip(-1) if rev else t


def _flat(us, deltas, Bs, Cs):
    revs = [0, 0, 1, 1]
    u = torch.cat([_seq(t, r) for t, r in zip(us, revs)], 1).contiguous()
    dl = torch.cat([_seq(t, r) for t, r in zip(deltas, revs)], 1).contiguous()
    Bm = torch.stack([_seq(t, r) for t, r in zip(Bs, revs)], 1).contiguous()
    Cm = torch.stack([_seq(t, r) for t, r in zip(Cs, revs)], 1).contiguous()
    return u, dl, Bm, Cm


# (C, H, W): non-square, L = 384 < one 512-position pair of chunks, the largest bench shape, L = 600 not a multiple of the 256-position
# chunk, L = 6144 far past the 64-position checkpoint interval
SHAPES = [(16, 40, 24), (48, 16, 24), (96, 64, 64), (16, 20, 30), (16, 64, 96)]
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def _check(got, ref, dtype, name):
    tol = BWD_TOL[dtype]
    g, r = got.double().cpu(), ref.double().cpu()
    scale = r.abs().max().clamp_min(1e-6)
    err = (g - r).abs().max()
    assert err <= tol * scale + 1e-5, f"{name}: max err {err:.3e} vs scale {scale:.3e} (tol {tol})"


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("batch", [1, 8])
@pytest.mark.parametrize("dtype", DTYPES)
def test_grouped_bwd_equals_flat_bwd_on_gathered_operands(shape, batch, dtype):
    C, H, W = shape
    L, N = H * W, 16
    if dtype != torch.float32 and L % 8:
        pytest.skip("16-bit grouped scan needs L % 8 == 0")
    us, deltas, Bs, Cs, A, Dv, bias = _grouped_operands(batch, C, L, N, dtype, seed=C + L + batch)
    rn, _ = _gen(L)
    douts = [rn(batch, C, L).to(dtype).cuda() for _ in range(4)]
    revs = [0, 0, 1, 1]
    _, ckpt = ops.selective_scan_fwd_grouped(us, deltas, Bs, Cs, revs, A, Dv, bias, True, need_ckpt=True)
    dus, dds, dA, dBs, dCs, dD, dbias = ops.selective_scan_bwd_grouped(us, deltas, Bs, Cs, douts, revs, A, Dv, bias, ckpt, True)
    u, dl, Bm, Cm = _flat(us, deltas, Bs, Cs)
    go = torch.cat([_seq(t, r) for t, r in zip(douts, revs)], 1).contiguous()
    _, fck = ops.selective_scan_fwd(u, dl, A, Bm, Cm, Dv, bias, True, need_ckpt=True)
    fdu, fdd, fdA, fdB, fdC, fdD, fdbias = ops.selective_scan_bwd(u, dl, A, Bm, Cm, Dv, bias, go, fck, True)
    for g in range(4):
        rv = revs[g]
        _check(dus[g], _seq(fdu[:, g * C:(g + 1) * C], rv), dtype, f"du{g}")
        _check(dds[g], _seq(fdd[:, g * C:(g + 1) * C], rv), dtype, f"ddelta{g}")
        _check(dBs[g], _seq(fdB[:, g], rv), dtype, f"dB{g}")
        _check(dCs[g], _seq(fdC[:, g], rv), dtype, f"dC{g}")
    for n, a, b in (("dA", dA, fdA), ("dD", dD, fdD), ("dbias", dbias, fdbias)):
        _check(a, b, dtype, n)


@pytest.mark.parametrize("dtype", DTYPES)
def test_grouped_bwd_channel_slice_sources(dtype):
    C, L, N, b = 32, 40 * 24, 16, 2
    us, deltas, Bs, Cs, A, Dv, bias = _grouped_operands(b, C, L, N, dtype, seed=5, sliced=True)
    rn, _ = _gen(9)
    dwide = rn(b, 4, C + 8, L).to(dtype).cuda()
    douts = [dwide[:, g, 4:4 + C] for g in range(4)]
    revs = [0, 0, 1, 1]
    _, ckpt = ops.selective_scan_fwd_grouped(us, deltas, Bs, Cs, revs, A, Dv, bias, True, need_ckpt=True)
    dus, dds, dA, dBs, dCs, dD, dbias = ops.selective_scan_bwd_grouped(us, deltas, Bs, Cs, douts, revs, A, Dv, bias, ckpt, True)
    u, dl, Bm, Cm = _flat(us, deltas, Bs, Cs)
    go = torch.cat([_seq(t, r) for t, r in zip(douts, revs)], 1).contiguous()
    _, fck = ops.selective_scan_fwd(u, dl, A, Bm, Cm, Dv, bias, True, need_ckpt=True)
    fdu, fdd, fdA, fdB, fdC, fdD, fdbias = ops.selective_scan_bwd(u, dl, A, Bm, Cm, Dv, bias, go, fck, True)
    for g in range(4):
        _check(dus[g], _seq(fdu[:, g * C:(g + 1) * C], revs[g]), dtype, f"du{g}")
        _check(dds[g], _seq(fdd[:, g * C:(g + 1) * C], revs[g]), dtype, f"ddelta{g}")
        _check(dBs[g], _seq(fdB[:, g], revs[g]), dtype, f"dB{g}")
        _check(dCs[g], _seq(fdC[:, g], revs[g]), dtype, f"dC{g}")
    _check(dA, fdA, dtype, "dA")


def test_grouped_bwd_rejects_unaligned_rows():
    us, deltas, Bs, Cs, A, Dv, bias = _grouped_operands(1, 16, 40 * 24, 16, torch.bfloat16, seed=1)
    _, ckpt = ops.selective_scan_fwd_grouped(us, deltas, Bs, Cs, [0, 0, 1, 1], A, Dv, bias, True, need_ckpt=True)
    bad = [t[..., 1:] for t in us]  # base pointers off the 16 B grid, L no longer a multiple of 8
    with pytest.raises(RuntimeError, match="16 B-aligned"):
        ops.selective_scan_bwd_grouped(bad, [t[..., 1:] for t in deltas], [t[..., 1:] for t in Bs], [t[..., 1:] for t in Cs],
                                       [t[..., 1:] for t in us], [0, 0, 1, 1], A, Dv, bias, ckpt, True)


@pytest.mark.parametrize("shape", [(16, 40, 24), (48, 16, 24), (16, 64, 96)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_grouped_fwd_checkpoints(shape, dtype):
    C, H, W = shape
    L, N, b = H * W, 16, 2
    us, deltas, Bs, Cs, A, Dv, bias = _grouped_operands(b, C, L, N, dtype, seed=L)
    revs = [0, 0, 1, 1]
    out0 = ops.selective_scan_fwd_grouped(us, deltas, Bs, Cs, revs, A, Dv, bias, True)
    out1, ckpt = ops.selective_scan_fwd_grouped(us, deltas, Bs, Cs, revs, A, Dv, bias, True, need_ckpt=True)
    assert torch.equal(out0, out1), "checkpoints changed the output"
    u, dl, Bm, Cm = _flat(us, deltas, Bs, Cs)
    _, fck = ops.selective_scan_fwd(u, dl, A, Bm, Cm, Dv, bias, True, need_ckpt=True)
    assert ckpt.shape == fck.shape
    torch.testing.assert_close(ckpt, fck, rtol=1e-3, atol=1e-4 * float(fck.abs().max()))


# ----------------------------------------------------------------------------- the operator
def _params(D, N, R, seed, with_bias=True, dtype=torch.float32):
    rn, r = _gen(seed)
    p = dict(x_proj_weight=0.3 * rn(4, R + 2 * N, D), x_proj_bias=0.1 * rn(4, R + 2 * N) if with_bias else None,
             dt_projs_weight=0.5 * rn(4, D, R), dt_projs_bias=-4.0 + 0.5 * r(4, D),
             A_logs=torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(4 * D, 1) + 0.1 * rn(4 * D, N),
             Ds=1.0 + 0.2 * rn(4 * D))
    return {k: (v.cuda().requires_grad_() if v is not None else None) for k, v in p.items()}


def _norm(D, seed):
    n = archs.LayerNorm(D, "WithBias").cuda()
    rn, _ = _gen(seed)
    with torch.no_grad():
        n.body.weight.copy_(1.0 + 0.2 * rn(D))
        n.body.bias.copy_(0.1 * rn(D))
    return n


def _composed(x, p, norm):
    """the reference operator restated in torch (CrossScan, einsums, CrossMerge) around this library's selective_scan_fn"""
    B, D, H, W = x.shape
    L = H * W
    N, R = p["A_logs"].shape[1], p["dt_projs_weight"].shape[2]
    x_hwwh = torch.stack([x.flatten(2), x.transpose(2, 3).flatten(2)], 1)
    xs = torch.cat([x_hwwh, x_hwwh.flip(-1)], 1)
    x_dbl = torch.einsum("b k d l, k c d -> b k c l", xs, p["x_proj_weight"].to(x.dtype))
    if p["x_proj_bias"] is not None:
        x_dbl = x_dbl + p["x_proj_bias"].to(x.dtype).view(1, 4, -1, 1)
    dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
    dts = torch.einsum("b k r l, k d r -> b k d l", dts, p["dt_projs_weight"].to(x.dtype))
    ys = selective_scan_fn(xs.reshape(B, -1, L), dts.reshape(B, -1, L), -torch.exp(p["A_logs"].float()), Bs.contiguous(),
                           Cs.contiguous(), p["Ds"].float(), p["dt_projs_bias"].reshape(-1).float(), True).view(B, 4, D, L)
    ys = ys.float()
    y2 = ys[:, 0:2] + ys[:, 2:4].flip(-1)
    y = y2[:, 0] + y2[:, 1].view(B, D, W, H).transpose(2, 3).reshape(B, D, L)
    return norm(y.view(B, D, H, W)).to(x.dtype)


def _ours(x, p, norm):
    return cs.cross_selective_scan(x, p["x_proj_weight"], p["x_proj_bias"], p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"],
                                   p["Ds"], norm)


def _run_both(B, D, H, W, N, R, dtype, with_bias, seed=0, ref_dtype=None):
    """-> [(y, grads) of the operator in `dtype`, (y, grads) of the composition in ref_dtype (default: dtype)] on the same inputs"""
    rn, _ = _gen(seed + 1)
    x0 = rn(B, D, H, W).to(dtype).cuda()
    g = rn(B, D, H, W).cuda()
    res = []
    for fn, dt in ((_ours, dtype), (_composed, ref_dtype or dtype)):
        p = _params(D, N, R, seed, with_bias)
        norm = _norm(D, seed + 2)
        x = x0.to(dt).clone().requires_grad_()
        y = fn(x, p, norm)
        y.float().backward(g)
        grads = {"x": x.grad, **{k: v.grad for k, v in p.items() if v is not None},
                 "norm_w": norm.body.weight.grad, "norm_b": norm.body.bias.grad}
        res.append((y.detach(), grads))
    return res


@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("shape", [(2, 16, 8, 12, 16, 4), (1, 48, 16, 24, 16, 3), (2, 16, 7, 9, 16, 4), (1, 24, 8, 8, 24, 2)])
def test_operator_fp32_equals_composition(shape, with_bias):
    """(7, 9): H*W % 4 != 0 and (d_state 24) take the gathered path inside the same Function"""
    B, D, H, W, N, R = shape
    (y, g), (yr, gr) = _run_both(B, D, H, W, N, R, torch.float32, with_bias)
    torch.testing.assert_close(y, yr, rtol=1e-3, atol=1e-4)
    for k in gr:
        torch.testing.assert_close(g[k], gr[k], rtol=1e-3, atol=1e-4 * max(1.0, float(gr[k].abs().max())), msg=lambda m: f"{k}: {m}")


@pytest.mark.parametrize("shape", [(2, 32, 16, 24, 16, 4), (1, 16, 10, 13, 16, 4)])
def test_operator_bf16_close_to_composition(shape):
    """bf16 operator and bf16 composition (gathered copies, einsums, the flat scan) against the fp32 composition on the same
    (bf16-valued) inputs: the operator's error stays within the module tests' bf16 bounds (max 0.08, mean 0.01 of the scale) or, where
    bf16 rounding of 16-bit scan operands alone exceeds the max bound, within 1.5x the composition's own bf16 error.
    (10, 13): H*W % 8 != 0 -> the gathered path"""
    B, D, H, W, N, R = shape
    (y, g), (y32, g32) = _run_both(B, D, H, W, N, R, torch.bfloat16, True, ref_dtype=torch.float32)
    _, (yc, gc) = _run_both(B, D, H, W, N, R, torch.bfloat16, True)
    for k, a, c, r in [("y", y, yc, y32)] + [(k, g[k], gc[k], g32[k]) for k in g32]:
        s = float(r.abs().max().clamp_min(1e-6)) if k != "y" else 1.0
        e, ec = (a.float() - r.float()).abs(), (c.float() - r.float()).abs()
        assert float(e.max()) < max(0.08 * s, 1.5 * float(ec.max())) and float(e.mean()) < 0.01 * s, \
            (k, float(e.max()), float(ec.max()), float(e.mean()), s)


def test_operator_pinned_to_reference_golden(golden_dir):
    """fp32 operator against the reference's own cross_selective_scan (tests/golden/make_golden_cross_scan.py)"""
    z = np.load(os.path.join(golden_dir, "cross_selective_scan.npz"))
    t = lambda k: torch.from_numpy(z[k]).cuda()
    p = {k: t(k).requires_grad_() for k in ("x_proj_weight", "x_proj_bias", "dt_projs_weight", "dt_projs_bias", "A_logs", "Ds")}
    D = p["Ds"].numel() // 4
    norm = archs.LayerNorm(D, "WithBias").cuda()
    with torch.no_grad():
        norm.body.weight.copy_(t("norm_w"))
        norm.body.bias.copy_(t("norm_b"))
    x = t("x").requires_grad_()
    y = _ours(x, p, norm)
    y.backward(t("dout"))
    torch.testing.assert_close(y.detach().cpu(), torch.from_numpy(z["y"]), rtol=1e-3, atol=1e-4)
    got = {"x": x.grad, **{k: v.grad for k, v in p.items()}, "norm_w": norm.body.weight.grad, "norm_b": norm.body.bias.grad}
    for k, v in got.items():
        r = torch.from_numpy(z[f"grad/{k}"])
        assert v.shape == r.shape, k
        torch.testing.assert_close(v.cpu(), r, rtol=1e-3, atol=1e-4 * max(1.0, float(r.abs().max())), msg=lambda m: f"{k}: {m}")


def test_cross_scan_and_merge_match_reference(golden_dir):
    z = np.load(os.path.join(golden_dir, "cross_scan.npz"))
    x = torch.from_numpy(z["x"]).cuda().requires_grad_()
    xs = cs.CrossScan.apply(x)
    assert torch.equal(xs.detach().cpu(), torch.from_numpy(z["xs"]))  # the gather is bit-exact
    ys = torch.from_numpy(z["ys"]).cuda().requires_grad_()
    y = cs.CrossMerge.apply(ys)
    torch.testing.assert_close(y.detach().cpu(), torch.from_numpy(z["y"]), rtol=1e-6, atol=1e-6)
    # backward: CrossScan's adjoint is CrossMerge's forward and vice versa (reference :337-343, :358-368)
    gx = torch.randn_like(xs)
    xs.backward(gx)
    B, _, C, L = gx.shape
    H, W = x.shape[2:]
    g2 = gx[:, 0:2] + gx[:, 2:4].flip(-1)
    ref_dx = (g2[:, 0] + g2[:, 1].view(B, C, W, H).transpose(2, 3).reshape(B, C, L)).view_as(x)
    torch.testing.assert_close(x.grad, ref_dx, rtol=1e-6, atol=1e-6)
    gy = torch.randn_like(y)
    y.backward(gy)
    ref_dys = torch.stack([gy, gy.view(B, C, H, W).transpose(2, 3).reshape(B, C, L)], 1)
    ref_dys = torch.cat([ref_dys, ref_dys.flip(-1)], 1).view_as(ys)
    assert torch.equal(ys.grad, ref_dys)


def test_forward_corev2_matches_operator():
    torch.manual_seed(0)
    m = archs.SS2D_1(d_model=16, ssm_ratio=1, variant="realsr").cuda()
    x = torch.randn(2, 12, 16, 16, device="cuda")  # (B, H, W, D) channels-last
    y = m.forward_corev2(x)
    ref = cs.cross_selective_scan(x.permute(0, 3, 1, 2).contiguous(), m.x_proj_weight, None, m.dt_projs_weight, m.dt_projs_bias,
                                  m.A_logs, m.Ds, m.out_norm)
    assert torch.equal(y, ref) and y.shape == (2, 16, 12, 16)
    assert torch.equal(m.forward_corev2(x.permute(0, 3, 1, 2), channel_first=True), ref)


def test_operator_argument_errors():
    p = _params(16, 16, 4, 0)
    norm = _norm(16, 0)
    x = torch.randn(1, 16, 8, 8, device="cuda")
    with pytest.raises(NotImplementedError):
        cs.cross_selective_scan(x, p["x_proj_weight"], None, p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"], p["Ds"], norm,
                                softmax_version=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        cs.cross_selective_scan(x.cpu(), p["x_proj_weight"], None, p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"], p["Ds"], norm)
    y1 = cs.cross_selective_scan(x, p["x_proj_weight"], None, p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"], p["Ds"], norm, nrows=3)
    y2 = cs.cross_selective_scan(x, p["x_proj_weight"], None, p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"], p["Ds"], norm)
    assert torch.equal(y1, y2)  # nrows is accepted and ignored


def test_operator_forward_backward_in_one_cuda_graph():
    B, D, H, W, N, R = 2, 32, 16, 24, 16, 4
    p = _params(D, N, R, 3)
    norm = _norm(D, 4)
    x = torch.randn(B, D, H, W, device="cuda", requires_grad=True)
    g = torch.randn(B, D, H, W, device="cuda")
    params = [x] + [v for v in p.values() if v is not None] + list(norm.parameters())

    def step():
        for t in params:
            t.grad = None
        y = _ours(x, p, norm)
        y.backward(g)
        return y.detach()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            y_eager = step()
    torch.cuda.current_stream().wait_stream(s)
    eager = [y_eager.clone()] + [t.grad.clone() for t in params]
    for t in params:
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_static = _ours(x, p, norm)
        y_static.backward(g)
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    got = [y_static.detach()] + [t.grad for t in params]
    for a, b in zip(got, eager):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5 * max(1.0, float(b.abs().max())))
