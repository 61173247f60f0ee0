"""The differentiable two-direction channel scan (vmambair_b200.cross_scan: cross_selective_scanC, CrossScanC, CrossMergeC; kernels
vmb_cross_selective_scan_c_fwd / _bwd) against a torch composition of the reference's operator on the library's flat scan, and against
the reference's own outputs (tests/golden/cross_selective_scan_c.npz, RealSR/VmambaIR/archs/MambaRealSR11_arch.py:438-534)."""
import math
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

REALSR = [(48, 3), (96, 6), (192, 12), (384, 24)]  # (L = C, R = ceil(C/16)) of the RealSR channel calls, D = 1, N = 16
PARAMS = ("x_proj_weight", "x_proj_bias", "dt_projs_weight", "dt_projs_bias", "A_logs", "Ds")


def _gen(seed):
    g = torch.Generator().manual_seed(seed)
    return lambda *s: torch.randn(*s, generator=g), lambda *s: torch.rand(*s, generator=g)


def _params(D, N, R, seed, with_bias=True):
    rn, r = _gen(seed)
    p = dict(x_proj_weight=0.3 * rn(2, R + 2 * N, D), x_proj_bias=0.1 * rn(2, R + 2 * N) if with_bias else None,
             dt_projs_weight=0.5 * rn(2, D, R), dt_projs_bias=-4.0 + 0.5 * r(2, D),
             A_logs=torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(2 * D, 1) + 0.1 * rn(2 * D, N),
             Ds=1.0 + 0.2 * rn(2 * D))
    return {k: (v.cuda().requires_grad_() if v is not None else None) for k, v in p.items()}


def _norm(L, seed):
    n = archs.LayerNorm(L, "WithBias").cuda()
    rn, _ = _gen(seed)
    with torch.no_grad():
        n.body.weight.copy_(1.0 + 0.2 * rn(L))
        n.body.bias.copy_(0.1 * rn(L))
    return n


def _composed(x, p, norm):
    """the reference operator restated in torch (CrossScanC, einsums, CrossMergeC) around this library's selective_scan_fn, fp32"""
    B, D, L = x.shape
    N, R = p["A_logs"].shape[1], p["dt_projs_weight"].shape[2]
    xs = torch.stack([x, x.flip(-1)], 1)
    x_dbl = torch.einsum("b k d l, k c d -> b k c l", xs, p["x_proj_weight"])
    if p["x_proj_bias"] is not None:
        x_dbl = x_dbl + p["x_proj_bias"].view(1, 2, -1, 1)
    dts, Bs, Cs = torch.split(x_dbl, [R, N, N], dim=2)
    dts = torch.einsum("b k r l, k d r -> b k d l", dts, p["dt_projs_weight"])
    ys = selective_scan_fn(xs.reshape(B, -1, L), dts.reshape(B, -1, L).contiguous(), -torch.exp(p["A_logs"].float()), Bs.contiguous(),
                           Cs.contiguous(), p["Ds"].float(), p["dt_projs_bias"].reshape(-1).float(), True).view(B, 2, D, L)
    y = ys[:, 0] + ys[:, 1].flip(-1)
    return norm(y.transpose(1, 2).unsqueeze(2).contiguous())


def _ours(x, p, norm, **kw):
    return cs.cross_selective_scanC(x, p["x_proj_weight"], p["x_proj_bias"], p["dt_projs_weight"], p["dt_projs_bias"], p["A_logs"],
                                    p["Ds"], norm, **kw)


def _run(fn, x0, g, D, L, N, R, with_bias, seed):
    p = _params(D, N, R, seed, with_bias)
    norm = _norm(L, seed + 2)
    x = x0.clone().requires_grad_()
    y = fn(x, p, norm)
    y.float().backward(g)
    grads = {"x": x.grad, **{k: v.grad for k, v in p.items() if v is not None}, "norm_w": norm.body.weight.grad,
             "norm_b": norm.body.bias.grad}
    return y.detach(), grads


def _close(got, ref, name, rtol=1e-3):
    torch.testing.assert_close(got.float(), ref.float(), rtol=rtol, atol=1e-4 * max(1.0, float(ref.abs().max())),
                               msg=lambda m: f"{name}: {m}")


def _check_fp32(B, D, L, R, N, with_bias, seed=0):
    rn, _ = _gen(seed + 1)
    x0 = rn(B, D, L).cuda()
    g = rn(B, L, 1, D).cuda()
    y, gr = _run(_ours, x0, g, D, L, N, R, with_bias, seed)
    yr, grr = _run(_composed, x0, g, D, L, N, R, with_bias, seed)
    assert y.shape == yr.shape == (B, L, 1, D)
    _close(y, yr, "y")
    assert set(gr) == set(grr)
    for k in grr:
        assert gr[k].shape == grr[k].shape and gr[k].dtype == grr[k].dtype, k
        _close(gr[k], grr[k], k)


@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("LR", REALSR)
def test_realsr_shapes_fp32_equal_composition(LR, B, with_bias):
    L, R = LR
    assert ops.cross_scan_c_supported(1, L, R, 16)
    _check_fp32(B, 1, L, R, 16, with_bias, seed=L + B)


@pytest.mark.parametrize("shape", [(2, 2, 96, 6, 16), (3, 4, 48, 3, 16)])
def test_fused_wider_D_fp32_equal_composition(shape):
    B, D, L, R, N = shape
    assert ops.cross_scan_c_supported(D, L, R, N)
    _check_fp32(B, D, L, R, N, True, seed=D)


# composed path: the state history alone (2 x 16 x 4096 fp32) is 512 KB; d_state 24 > 16; D = 17 > 16
@pytest.mark.parametrize("shape", [(2, 1, 4096, 4, 16), (2, 1, 48, 3, 24), (2, 17, 32, 2, 8)])
def test_composed_path_fp32_equal_composition(shape):
    B, D, L, R, N = shape
    assert not ops.cross_scan_c_supported(D, L, R, N)
    _check_fp32(B, D, L, R, N, True, seed=L)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("LR", [(48, 3), (384, 24)])
def test_16bit_x_equals_fp32_composition_up_to_output_rounding(LR, dtype):
    """internals are fp32, so against the fp32 composition on the same 16-bit-valued x (and the incoming gradient rounded the way the
    output cast's backward rounds it) y and dx differ by their rounding to x's dtype, the fp32 parameter gradients by fp32 noise"""
    L, R = LR
    B, D, N = 3, 1, 16
    rn, _ = _gen(L + 7)
    x16 = rn(B, D, L).to(dtype).cuda()
    g = rn(B, L, 1, D).cuda()
    y, gr = _run(_ours, x16, g, D, L, N, R, True, 5)
    yr, grr = _run(_composed, x16.float(), g.to(dtype).float(), D, L, N, R, True, 5)
    assert y.dtype == dtype and gr["x"].dtype == dtype
    u16 = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11  # one unit in the last place, relative
    _close(y, yr, "y", rtol=u16 + 1e-3)
    _close(gr["x"], grr["x"], "x", rtol=u16 + 1e-3)
    for k in grr:
        if k != "x":
            assert gr[k].dtype == torch.float32
            _close(gr[k], grr[k], k)


@pytest.mark.parametrize("case", ["realsr", "general"])
def test_operator_pinned_to_reference_golden(golden_dir, case):
    """fp32 operator against the reference's own cross_selective_scanC (tests/golden/make_golden_cross_scan_c.py)"""
    z = np.load(os.path.join(golden_dir, "cross_selective_scan_c.npz"))
    t = lambda k: torch.from_numpy(z[f"{case}/{k}"]).cuda()
    p = {k: (t(k).requires_grad_() if f"{case}/{k}" in z else None) for k in PARAMS}
    x = t("x").requires_grad_()
    B, D, L = x.shape
    N, R = p["A_logs"].shape[1], p["dt_projs_weight"].shape[2]
    assert ops.cross_scan_c_supported(D, L, R, N)
    norm = archs.LayerNorm(L, "WithBias").cuda()
    with torch.no_grad():
        norm.body.weight.copy_(t("norm_w"))
        norm.body.bias.copy_(t("norm_b"))
    y = _ours(x, p, norm)
    y.backward(t("dout"))
    torch.testing.assert_close(y.detach().cpu(), torch.from_numpy(z[f"{case}/y"]), rtol=1e-3, atol=1e-4)
    got = {"x": x.grad, **{k: v.grad for k, v in p.items() if v is not None}, "norm_w": norm.body.weight.grad,
           "norm_b": norm.body.bias.grad}
    for k, v in got.items():
        r = torch.from_numpy(z[f"{case}/grad/{k}"])
        assert v.shape == r.shape, k
        torch.testing.assert_close(v.cpu(), r, rtol=1e-3, atol=1e-4 * max(1.0, float(r.abs().max())), msg=lambda m: f"{k}: {m}")


def _ref_cross_scan_c(x):  # the reference's CrossScanC.forward / CrossMergeC.backward (:441-448, :469-475), restated
    B, D, L = x.shape
    xs = x.new_empty((B, 2, D, L))
    xs[:, 0] = x
    xs[:, 1] = torch.flip(x, dims=[-1])
    return xs


def test_cross_scan_c_and_merge_c_match_reference():
    x = torch.randn(3, 2, 37, device="cuda", requires_grad=True)
    xs = cs.CrossScanC.apply(x)
    assert torch.equal(xs, _ref_cross_scan_c(x.detach()))  # the gather is bit-exact
    ys = torch.randn(3, 2, 2, 37, device="cuda", requires_grad=True)
    y = cs.CrossMergeC.apply(ys)
    assert torch.equal(y, ys[:, 0].detach() + ys[:, 1].detach().flip(dims=[-1]))
    # each backward is the other's forward
    gx = torch.randn_like(xs)
    xs.backward(gx)
    assert torch.equal(x.grad, cs.CrossMergeC.apply(gx))
    gy = torch.randn_like(y)
    y.backward(gy)
    assert torch.equal(ys.grad, cs.CrossScanC.apply(gy))


@pytest.mark.parametrize("d_model", [48, 96])
def test_cforward_corev2_matches_operator_and_composed_core(d_model):
    torch.manual_seed(0)
    m = archs.SS2D_1(d_model=d_model, ssm_ratio=1, variant="realsr").cuda()
    y2 = torch.randn(2, d_model, 12, 16, device="cuda")
    c = m.cforward_corev2(y2, channel_first=True)
    ref = cs.cross_selective_scanC(m.pooling(y2).view(2, 1, d_model), m.xc_proj_weight, None, m.dtc_projs_weight, m.dtc_projs_bias,
                                   m.Ac_logs, m.Dsc, m.channel_norm)
    assert c.shape == (2, d_model, 1, 1) and torch.equal(c, ref)
    assert torch.equal(m.cforward_corev2(y2.permute(0, 2, 3, 1)), ref)  # channels-last input
    torch.testing.assert_close(c, m.cforward_core(y2), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("variant", ["sisr", "mamber32", "mamber33"])
def test_cforward_corev2_rejects_other_variants(variant):
    m = archs.SS2D_1(d_model=16, ssm_ratio=1, variant=variant).cuda()
    with pytest.raises(NotImplementedError, match="realsr"):
        m.cforward_corev2(torch.randn(1, 16, 4, 4, device="cuda"), channel_first=True)


def _grads_once(x, p, norm, g):
    for t in [x, *[v for v in p.values() if v is not None], *norm.parameters()]:
        t.grad = None
    _ours(x, p, norm).backward(g)
    return [x.grad.clone()] + [v.grad.clone() for v in p.values() if v is not None]


@pytest.mark.parametrize("LR", [(96, 6), (384, 24)])
def test_backward_is_bitwise_reproducible(LR):
    L, R = LR
    B = 8
    p = _params(1, 16, R, 11)
    norm = _norm(L, 12)
    x = torch.randn(B, 1, L, device="cuda", requires_grad=True)
    g = torch.randn(B, L, 1, 1, device="cuda")
    a, b = _grads_once(x, p, norm, g), _grads_once(x, p, norm, g)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_launch_census():
    B, L, R = 4, 192, 12
    p = _params(1, 16, R, 1)
    norm = _norm(L, 2)
    x = torch.randn(B, 1, L, device="cuda", requires_grad=True)
    n0 = ops.launch_count()
    y = _ours(x, p, norm)
    assert ops.launch_count() - n0 == 1, "the forward is one library launch"
    n1 = ops.launch_count()
    y.backward(torch.randn_like(y))
    assert ops.launch_count() - n1 <= 2, "the backward is at most two library launches"


def test_forward_backward_in_one_cuda_graph():
    B, D, L, R, N = 4, 1, 96, 6, 16
    p = _params(D, N, R, 3)
    norm = _norm(L, 4)
    x = torch.randn(B, D, L, device="cuda", requires_grad=True)
    g = torch.randn(B, L, 1, D, device="cuda")
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


def test_argument_errors():
    L, R, N = 48, 3, 16
    p = _params(1, N, R, 0, with_bias=False)
    norm = _norm(L, 0)
    x = torch.randn(2, 1, L, device="cuda")
    with pytest.raises(NotImplementedError):
        _ours(x, p, norm, softmax_version=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        _ours(x.cpu(), p, norm)
    with pytest.raises(RuntimeError, match="expected"):
        _ours(torch.randn(2, 2, L, device="cuda"), p, norm)  # D does not match the parameters
    bad = dict(p, x_proj_weight=torch.randn(2, R + 2 * N + 1, 1, device="cuda"))
    with pytest.raises(RuntimeError, match="expected"):
        _ours(x, bad, norm)
    assert torch.equal(_ours(x, p, norm, nrows=3), _ours(x, p, norm))  # nrows is accepted and ignored
    assert math.isfinite(float(_ours(x, p, norm, to_dtype=False).detach().sum()))
