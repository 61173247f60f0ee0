"""fp32 output from 16-bit inputs (`selective_scan_cuda_oflex`) and the state-dimension-1 layout (`selective_scan_cuda_ndstate`).

Every case is checked against the float64 oracle (oracle.cscan) on the same dtype-rounded inputs, on both forward paths (TMA
kernel, generic kernel) and both backward paths (TMA kernel; generic kernel).  Each case asserts the launcher's path condition,
so a layout cannot drift onto the other path unnoticed.

fp32 accuracy is shown, not assumed: the forward bound is test_scan_gpu.py's fp32 bound (its relative term capped at a quarter of
the 16-bit unit roundoff, which only tightens it for fp16), and the test asserts that one 16-bit rounding of `out` breaks it.  The backward's fp32-level bound is set by the fp32 operator on the same values (16-bit inputs
are exact in fp32); the test asserts that rounding dout to 16 bits first breaks it for dA, dD and ddelta_bias."""
import ctypes as C

import pytest
import torch

from oracle import cscan

pytestmark = pytest.mark.gpu

DT16 = [torch.bfloat16, torch.float16]
U16 = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}  # unit roundoff
GRAD_NAMES = ("du", "ddelta", "dA", "dB", "dC", "dD", "dbias")


def make_inputs(b, D, L, N, G, dtype, seed=0, has_D=True, has_bias=True):
    """the reference test's distributions (test_selective_scan.py:406-441), rounded to `dtype` once"""
    g = torch.Generator().manual_seed(seed)
    A = -0.5 * torch.rand(D, N, generator=g)
    delta = 0.5 * torch.rand(b, D, L, generator=g)
    Bm, Cm, u = torch.randn(b, G, N, L, generator=g), torch.randn(b, G, N, L, generator=g), torch.randn(b, D, L, generator=g)
    Dv = torch.randn(D, generator=g) if has_D else None
    bias = 0.5 * torch.rand(D, generator=g) if has_bias else None
    return u.to(dtype), delta.to(dtype), A, Bm.to(dtype), Cm.to(dtype), Dv, bias


def cuda(ts):
    return [None if t is None else t.cuda() for t in ts]


# ----------------------------------------------------------------------------- path conditions (scan_fwd_tma_pick, scan_bwd_tma_pick)
def _aligned(*ts):
    return all(t.data_ptr() % 16 == 0 for t in ts)


def _mult(v, *strides):
    return all(s % v == 0 for s in strides)


def fwd_takes_tma(u, delta, Bm, Cm, out, N, G):
    """scan_fwd_tma_pick (csrc/scan_fwd_tma.cu) on the vec_ok of vmb_selective_scan_fwd (csrc/api.cu)"""
    v, vo = 16 // u.element_size(), 16 // out.element_size()
    vec_ok = _aligned(u, delta, Bm, Cm, out) and _mult(v, u.stride(0), u.stride(1), delta.stride(0), delta.stride(1),
                                                      *Bm.stride()[:3], *Cm.stride()[:3]) and _mult(vo, out.stride(0), out.stride(1))
    b, D, L = u.shape
    npad = (N + 15) // 16 * 16
    if not vec_ok or npad != 16 or L < 512:
        return False
    want = 8 * torch.cuda.get_device_properties(u.device).multi_processor_count
    rb, ss = 2, 1
    while ss < 4 and (b * D) // rb * ss < want:
        ss <<= 1
    return (D // G) % (rb * 4 // ss) == 0


def bwd_takes_tma(u, N, G):
    """scan_bwd_tma_pick for the dense tensors these tests pass (vec_ok holds: contiguous, L % 8 == 0)"""
    b, D, L = u.shape
    if L % 8 or (N + 15) // 16 * 16 != 16 or L < 512:
        return False
    sms = torch.cuda.get_device_properties(u.device).multi_processor_count
    rb, ss = 2, 1
    while ss < 4 and (b * D) // (rb * 4 // ss) * 2 <= 2 * sms:
        ss <<= 1
    return (D // G) % (rb * 4 // ss) == 0


# ----------------------------------------------------------------------------- direct C-ABI forward (caller-chosen `out`)
def fwd_into(out, u, delta, A, Bm, Cm, Dv, bias, softplus, out_f32):
    from vmambair_b200 import _lib, ops
    b, d, l = u.shape
    n, g = A.shape[1], Bm.shape[1]
    P = ops._ptr
    a = _lib.ScanFwdArgs(
        u=P(u), delta=P(delta), A=P(A), Bm=P(Bm), Cm=P(Cm), D=P(Dv), delta_bias=P(bias), out=P(out), ckpt=None,
        batch=b, dim=d, seqlen=l, dstate=n, ngroups=g, u_bs=u.stride(0), u_ds=u.stride(1), delta_bs=delta.stride(0),
        delta_ds=delta.stride(1), out_bs=out.stride(0), out_ds=out.stride(1), B_bs=Bm.stride(0), B_gs=Bm.stride(1), B_ns=Bm.stride(2),
        C_bs=Cm.stride(0), C_gs=Cm.stride(1), C_ns=Cm.stride(2), delta_softplus=int(softplus), dtype=ops._DT[u.dtype], out_f32=out_f32)
    return _lib.lib().vmb_selective_scan_fwd(C.byref(a), ops._stream(u))


def fp32_fwd_bound(ins, softplus, ref64, rtol=1e-3):
    """test_scan_gpu.py's fp32 bound: 1e-3 rel / 1e-5 abs plus 8x the fp32 oracle's own distance from float64"""
    ref32 = cscan.scan_fwd(*ins, softplus)
    return 1e-5 + rtol * ref64.abs() + 8.0 * (ref32.double() - ref64).abs().max()


def check_fp32_out(out, ins, softplus, dtype):
    assert out.dtype == torch.float32
    ref64 = cscan.scan_fwd(*ins, softplus, fp64=True)
    # the relative term is at most a quarter of the 16-bit unit roundoff: 1e-3 for bf16 (2^-8 / 4 = 9.8e-4), 1.2e-4 for fp16, whose
    # rounding error (<= 2^-11 relative) 1e-3 would not resolve
    bound = fp32_fwd_bound(ins, softplus, ref64, rtol=min(1e-3, U16[dtype] / 4))
    err = (out.double().cpu() - ref64).abs()
    assert bool((err <= bound).all()), f"{int((err > bound).sum())} / {err.numel()} beyond the fp32 bound; max err {err.max():.3e}"
    # the bound is tighter than one 16-bit rounding of out: an implementation that rounds, then widens, fails it
    rounded = (ref64.to(dtype).double() - ref64).abs()
    assert bool((rounded > bound).any()), "the fp32 bound does not resolve a 16-bit rounding of out"


FWD_FLAGS = [(True, True, True), (False, False, True), (True, False, False), (False, True, False)]  # has_D, has_bias, softplus


@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("flags", FWD_FLAGS)
@pytest.mark.parametrize("dtype", DT16)
def test_fwd_fp32_out_tma_path(dtype, flags, groups):
    has_D, has_bias, softplus = flags
    from vmambair_b200 import ops
    b, D, L, N = 2, 64, 1024, 16
    ins = make_inputs(b, D, L, N, groups, dtype, seed=31 + groups, has_D=has_D, has_bias=has_bias)
    g = cuda(ins)
    out, _ = ops.selective_scan_fwd(*g, softplus, need_ckpt=False, out_float=True)
    assert fwd_takes_tma(g[0], g[1], g[3], g[4], out, N, groups)
    check_fp32_out(out, ins, softplus, dtype)
    # with checkpoints (MODE 1): same output
    out_ck, ck = ops.selective_scan_fwd(*g, softplus, need_ckpt=True, out_float=True)
    assert ck is not None and torch.equal(out_ck, out)


@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("flags", FWD_FLAGS)
@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("case", ["short", "dstate20", "out_offset"])
def test_fwd_fp32_out_generic_path(case, dtype, flags, groups):
    has_D, has_bias, softplus = flags
    from vmambair_b200 import ops
    b, D, L, N = {"short": (2, 32, 300, 16), "dstate20": (1, 32, 640, 20), "out_offset": (2, 32, 1024, 16)}[case]
    ins = make_inputs(b, D, L, N, groups, dtype, seed=7 * L + groups, has_D=has_D, has_bias=has_bias)
    g = cuda(ins)
    if case == "out_offset":  # out one element into its storage: aligned inputs, unaligned out
        out = torch.empty(b * D * L + 1, dtype=torch.float32, device="cuda")[1:].view(b, D, L)
        assert fwd_into(out, *g, softplus, 1) == 0
        ck = None
    else:
        out, ck = ops.selective_scan_fwd(*g, softplus, need_ckpt=True, out_float=True)
    assert not fwd_takes_tma(g[0], g[1], g[3], g[4], out, N, groups)
    torch.cuda.synchronize()
    check_fp32_out(out, ins, softplus, dtype)


@pytest.mark.parametrize("dtype", DT16)
def test_fwd_fp32_out_row_stride_of_four(dtype):
    """out rows 16 B aligned in fp32 elements only (row stride L + 4): still the TMA path, values exact"""
    b, D, L, N, G = 2, 64, 1024, 16, 2
    ins = make_inputs(b, D, L, N, G, dtype, seed=5)
    g = cuda(ins)
    buf = torch.full((b, D, L + 4), float("nan"), dtype=torch.float32, device="cuda")
    out = buf[:, :, :L]
    assert fwd_takes_tma(g[0], g[1], g[3], g[4], out, N, G)
    assert fwd_into(out, *g, True, 1) == 0
    torch.cuda.synchronize()
    check_fp32_out(out, ins, True, dtype)
    assert bool(buf[:, :, L:].isnan().all()), "wrote beyond the rows"


@pytest.mark.parametrize("dtype", DT16)
def test_fwd_out_float_false_unchanged(dtype):
    """out_float=False is the plain operator, bit for bit; the fp32 out rounds to it"""
    from vmambair_b200 import ops
    g = cuda(make_inputs(2, 64, 1024, 16, 2, dtype, seed=2))
    o16, _ = ops.selective_scan_fwd(*g, True, need_ckpt=False)
    o16b, _ = ops.selective_scan_fwd(*g, True, need_ckpt=False, out_float=False)
    o32, _ = ops.selective_scan_fwd(*g, True, need_ckpt=False, out_float=True)
    assert o16.dtype == dtype and torch.equal(o16, o16b)
    assert torch.equal(o32.to(dtype), o16)


# ----------------------------------------------------------------------------- backward with fp32 dout
def run_bwd(g, dout, softplus):
    from vmambair_b200 import ops
    _, ck = ops.selective_scan_fwd(*g, softplus, need_ckpt=True)
    grads = ops.selective_scan_bwd(*g, dout, ck, softplus, dout_float=True)
    torch.cuda.synchronize()
    return grads


def _misaligned(t):
    """a copy of t one element into its storage"""
    return torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)[1:].view(t.shape).copy_(t)


def max_err(got, ref):
    return (got.double().cpu() - ref).abs().max().item()


@pytest.mark.parametrize("path", ["tma", "generic"])
@pytest.mark.parametrize("flags", [(True, True, True), (False, False, False), (True, True, False)])
@pytest.mark.parametrize("dtype", DT16)
def test_bwd_fp32_dout(path, dtype, flags):
    has_D, has_bias, softplus = flags
    b, D, L, N, G = 2, 64, 1024, 16, 2
    ins = make_inputs(b, D, L, N, G, dtype, seed=101, has_D=has_D, has_bias=has_bias)
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(102))  # fp32
    # generic: every dout one element into its storage, so its rows are not 16 B aligned (vec_ok false), on a layout that otherwise
    # takes the TMA kernel
    place = _misaligned if path == "generic" else (lambda t: t)
    g = cuda(ins)
    assert bwd_takes_tma(g[0], N, G)
    d = place(dout.cuda())
    assert (d.data_ptr() % 16 != 0) == (path == "generic")
    ours = run_bwd(g, d, softplus)
    ref = cscan.scan_bwd(*ins, dout, softplus)
    # the fp32 operator on the same values (16-bit inputs are exact in fp32): the fp32-level error of these gradients
    g32 = cuda([None if t is None else t.float() for t in ins])
    f32 = run_bwd(g32, place(dout.cuda()), softplus)
    # the same 16-bit operator with dout rounded to 16 bits first
    pre = run_bwd(g, place(dout.to(dtype).cuda()), softplus)
    for i, n in enumerate(GRAD_NAMES):
        if ref[i] is None:
            assert ours[i] is None and pre[i] is None, n
            continue
        assert ours[i].dtype == (dtype if n in ("du", "ddelta", "dB", "dC") else torch.float32), n
        assert ours[i].shape == ref[i].shape, n
        scale = ref[i].abs().max().item()
        e32 = max_err(f32[i], ref[i])
        fp32_bound = 4.0 * e32 + 1e-6 * scale
        err = (ours[i].double().cpu() - ref[i]).abs()
        if n in ("dA", "dD", "dbias"):
            assert err.max().item() <= fp32_bound, f"{n}: max err {err.max():.3e} vs fp32 bound {fp32_bound:.3e}"
            e_pre = max_err(pre[i], ref[i])
            assert e_pre > fp32_bound, f"{n}: rounding dout first stays within the bound ({e_pre:.3e} <= {fp32_bound:.3e})"
        else:  # 16-bit outputs: one rounding of a value within the fp32-level error
            bound = U16[dtype] * ref[i].abs() + 2.0 * fp32_bound
            bad = err > bound
            assert not bad.any(), f"{n}: {int(bad.sum())} elements beyond one 16-bit rounding; max err {err.max():.3e}"


@pytest.mark.parametrize("dtype", DT16)
def test_bwd_fp32_dout_generic_shapes(dtype):
    """the generic kernel by input alone: short sequence, dstate 20 (two state tiles), two rows per group"""
    for (b, D, L, N, G) in [(2, 32, 300, 16, 2), (1, 16, 640, 20, 1), (1, 6, 200, 16, 3)]:
        ins = make_inputs(b, D, L, N, G, dtype, seed=L)
        dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(L + 1))
        g = cuda(ins)
        assert not bwd_takes_tma(g[0], N, G)
        ours = run_bwd(g, dout.cuda(), True)
        f32 = run_bwd(cuda([None if t is None else t.float() for t in ins]), dout.cuda(), True)
        ref = cscan.scan_bwd(*ins, dout, True)
        for i, n in enumerate(GRAD_NAMES):
            scale = ref[i].abs().max().item()
            fp32_bound = 4.0 * max_err(f32[i], ref[i]) + 1e-6 * scale
            err = (ours[i].double().cpu() - ref[i]).abs()
            bound = fp32_bound if n in ("dA", "dD", "dbias") else U16[dtype] * ref[i].abs() + 2.0 * fp32_bound
            assert bool((err <= bound).all()), f"{(b, D, L, N, G)} {n}: max err {err.max():.3e}"


# ----------------------------------------------------------------------------- the two modules
def test_oflex_module_signature():
    from vmambair_b200 import selective_scan_cuda_oflex as m
    b, D, L, N, G = 2, 64, 512, 16, 2
    u, delta, A, Bm, Cm, Dv, bias = cuda(make_inputs(b, D, L, N, G, torch.bfloat16, seed=3))
    res = m.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1, True)
    assert isinstance(res, list) and len(res) == 2
    out, x = res
    assert out.dtype == torch.float32 and out.shape == (b, D, L) and x.dtype == torch.float32
    out16, x16 = m.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1, False)
    assert out16.dtype == torch.bfloat16
    out_f, _ = m.fwd(*[t.float() for t in (u, delta)], A, Bm.float(), Cm.float(), Dv, bias, True, 1, True)
    assert out_f.dtype == torch.float32
    dout = torch.randn_like(out)
    gr = m.bwd(u, delta, A, Bm, Cm, Dv, bias, dout, x, True, 1)
    assert isinstance(gr, list) and len(gr) == 7
    want = [(torch.bfloat16, (b, D, L)), (torch.bfloat16, (b, D, L)), (torch.float32, (D, N)), (torch.bfloat16, (b, G, N, L)),
            (torch.bfloat16, (b, G, N, L)), (torch.float32, (D,)), (torch.float32, (D,))]
    for t, (dt, sh) in zip(gr, want):
        assert t.dtype == dt and tuple(t.shape) == sh
    gr_none = m.bwd(u, delta, A, Bm, Cm, None, None, dout, x, True, 1)
    assert gr_none[5] is None and gr_none[6] is None


def test_ndstate_module_signature_and_values():
    from vmambair_b200 import selective_scan_cuda_ndstate as m
    b, D, L, G = 2, 32, 777, 2
    u, delta, A, Bm, Cm, Dv, bias = make_inputs(b, D, L, 1, G, torch.float32, seed=8)
    A1, B1, C1 = A.view(D), Bm.squeeze(2), Cm.squeeze(2)  # the ndstate layout
    gu, gd, gA, gB, gC, gD, gb = cuda((u, delta, A1, B1, C1, Dv, bias))
    out, x = m.fwd(gu, gd, gA, gB, gC, gD, gb, True, 1)
    assert out.dtype == torch.float32 and out.shape == (b, D, L)
    ref64 = cscan.scan_fwd(u, delta, A, Bm, Cm, Dv, bias, True, fp64=True)
    ins = (u, delta, A, Bm, Cm, Dv, bias)
    err = (out.double().cpu() - ref64).abs()
    assert bool((err <= fp32_fwd_bound(ins, True, ref64)).all()), f"max err {err.max():.3e}"
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(9))
    gr = m.bwd(gu, gd, gA, gB, gC, gD, gb, dout.cuda(), x, True, 1)
    assert len(gr) == 7
    assert gr[2].shape == (D,) and gr[3].shape == (b, G, L) and gr[4].shape == (b, G, L)
    ref = cscan.scan_bwd(*ins, dout, True)
    ref = [ref[0], ref[1], ref[2].view(D), ref[3].squeeze(2), ref[4].squeeze(2), ref[5], ref[6]]
    for n, got, r in zip(GRAD_NAMES, gr, ref):
        e = max_err(got, r)
        assert e <= 2e-3 * r.abs().max().item() + 1e-5, f"{n}: max err {e:.3e}"
    out16, _ = m.fwd(*[t.half() for t in (gu, gd)], gA, gB.half(), gC.half(), gD, gb, True, 1)
    assert out16.dtype == torch.float16  # the ndstate module keeps the input dtype (cpp:207)


def _fn_like_reference(module, mode):
    """The call pattern of the reference's build_selective_scan_fn (test_selective_scan.py:18-160) for its "ssoflex" and
    "sscorendstate" modes, written out here: autograd over module.fwd / module.bwd."""

    class Fn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, u, delta, A, B, C, D, delta_bias, delta_softplus):
            if mode == "ssoflex":
                out, x, *_ = module.fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, 1, True)
            else:
                A, B, C = A.view(-1), B.squeeze(2), C.squeeze(2)
                out, x, *_ = module.fwd(u, delta, A, B, C, D, delta_bias, delta_softplus, 1)
            ctx.softplus = delta_softplus
            ctx.save_for_backward(u, delta, A, B, C, D, delta_bias, x)
            return out

        @staticmethod
        def backward(ctx, dout):
            u, delta, A, B, C, D, delta_bias, x = ctx.saved_tensors
            du, ddelta, dA, dB, dC, dD, ddb, *_ = module.bwd(u, delta, A, B, C, D, delta_bias, dout.contiguous(), x, ctx.softplus, 1)
            if mode == "sscorendstate":
                dA, dB, dC = dA.unsqueeze(1), dB.unsqueeze(2), dC.unsqueeze(2)
            return du, ddelta, dA, dB, dC, dD, ddb, None

    def fn(u, delta, A, B, C, D, delta_bias, delta_softplus):
        out = Fn.apply(u, delta, A, B, C, D, delta_bias, delta_softplus)
        return out.to(u.dtype) if mode == "ssoflex" else out

    return fn


@pytest.mark.parametrize("mode", ["ssoflex", "sscorendstate"])
def test_reference_harness_pattern_autograd(mode):
    from vmambair_b200 import selective_scan_cuda_ndstate, selective_scan_cuda_oflex
    module = selective_scan_cuda_oflex if mode == "ssoflex" else selective_scan_cuda_ndstate
    dtype = torch.bfloat16 if mode == "ssoflex" else torch.float32
    N = 16 if mode == "ssoflex" else 1
    b, D, L, G = 2, 64, 1024, 2
    ins = make_inputs(b, D, L, N, G, dtype, seed=12)
    leaves = [None if t is None else t.cuda().requires_grad_() for t in ins]
    out = _fn_like_reference(module, mode)(*leaves, True)
    assert out.dtype == dtype
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(13))
    out.backward(dout.to(dtype).cuda())
    # the autograd graph hands the fp32 Function output a gradient of the cast back to out's dtype
    ref = cscan.scan_bwd(*ins, dout.to(dtype), True)
    tol = 4e-2 if dtype == torch.bfloat16 else 2e-3
    for n, leaf, r in zip(GRAD_NAMES, leaves, ref):
        assert leaf.grad is not None and leaf.grad.shape == leaf.shape, n
        e = max_err(leaf.grad, r)
        assert e <= tol * r.abs().max().item() + 1e-5, f"{n}: max err {e:.3e}"


# ----------------------------------------------------------------------------- against the reference's own kernels
@pytest.mark.parametrize("case", [("oflex", torch.bfloat16), ("oflex", torch.float16), ("ndstate", torch.float32),
                                  ("ndstate", torch.bfloat16)])
def test_vs_reference_cuda_kernels(case):
    """The two modules against the reference's selective_scan_cuda_oflex / selective_scan_cuda_ndstate on the same tensors (stored
    outputs, oracle/ref_kernel_golden_oflex.py: large outputs at 4096 seeded points, dA / dD / ddelta_bias whole), at the tolerances
    of the core module's reference-kernel test (test_bench_parity_gpu.py).  The fp32 `out` of oflex is held to the fp32 tolerance."""
    from oracle import ref_kernel_golden_oflex as rk
    from tests.test_bench_parity_gpu import _ref_tol
    from vmambair_b200 import selective_scan_cuda_ndstate, selective_scan_cuda_oflex
    kind, itype = case
    golden = rk.load()
    args, dout = rk.inputs(kind, itype)
    args = [t.cuda() for t in args]
    if kind == "oflex":
        m = selective_scan_cuda_oflex
        out_o, x_o = m.fwd(*args, True, 1, True)
    else:
        m = selective_scan_cuda_ndstate
        out_o, x_o = m.fwd(*args, True, 1)
    go = m.bwd(*args, dout.cuda(), x_o, True, 1)
    assert len(go) == 7
    rtol, atol, rtolw, atolw = _ref_tol(itype)
    r32, a32, _, _ = _ref_tol(torch.float32)
    out_tol = (r32, a32) if out_o.dtype == torch.float32 else (rtol, atol)
    tols = [out_tol, (rtol * 2, atol * 2), (rtol * 5, atol * 10), (rtolw, atolw * 5), (rtol, atol), (rtol, atol), (rtolw, atolw),
            (rtolw, atolw)]
    tg = rk.tag(kind, itype)
    for n, t, (rt, at) in zip(rk.NAMES, (out_o,) + tuple(go), tols):
        assert str(t.dtype) == str(golden[f"{tg}/{n}_dtype"]), (n, t.dtype, golden[f"{tg}/{n}_dtype"])
        assert tuple(t.shape) == tuple(golden[f"{tg}/{n}_shape"].tolist()), (n, tuple(t.shape))
        a, r = rk.sample(n, t), golden[f"{tg}/{n}"].float()
        if n in rk.WHOLE:
            at = at + 1e-3 * float(r.abs().max())
        bad = (a - r).abs() > at + rt * r.abs()
        assert not bad.any(), f"{n}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float((a - r).abs().max()):.3e}, max |ref| {float(r.abs().max()):.3e}"


# ----------------------------------------------------------------------------- argument errors
def test_errors_raise():
    from vmambair_b200 import _lib, ops, selective_scan_cuda_ndstate
    g = cuda(make_inputs(1, 16, 512, 16, 2, torch.bfloat16, seed=1))
    g32 = cuda(make_inputs(1, 16, 512, 16, 2, torch.float32, seed=1))
    out32 = torch.empty(1, 16, 512, device="cuda")
    out16 = torch.empty(1, 16, 512, device="cuda", dtype=torch.bfloat16)
    # C ABI: out_f32 only with 16-bit inputs, and only 0 / 1
    assert fwd_into(out32, *g32, True, 1) != 0
    assert "out_f32" in _lib.lib().vmb_last_error().decode()
    assert fwd_into(out16, *g, True, 2) != 0
    assert fwd_into(out16, *g, True, 0) == 0
    _, ck = ops.selective_scan_fwd(*g, True, need_ckpt=True)
    with pytest.raises(RuntimeError):  # fp16 dout against bf16 inputs
        ops.selective_scan_bwd(*g, torch.randn(1, 16, 512, device="cuda").half(), ck, True, dout_float=True)
    # an fp32 dout against bf16 inputs only where asked for: the core module rejects it, as the reference's (cus/selective_scan.cpp:259)
    from vmambair_b200 import selective_scan_cuda_core
    with pytest.raises(RuntimeError):
        ops.selective_scan_bwd(*g, torch.randn(1, 16, 512, device="cuda"), ck, True)
    with pytest.raises(RuntimeError):
        selective_scan_cuda_core.bwd(*g, torch.randn(1, 16, 512, device="cuda"), ck, True, 1)
    with pytest.raises(RuntimeError):  # fp64 dout
        ops.selective_scan_bwd(*g, torch.randn(1, 16, 512, device="cuda").double(), ck, True)
    with pytest.raises(RuntimeError):  # bf16 dout against fp32 inputs
        _, ck32 = ops.selective_scan_fwd(*g32, True, need_ckpt=True)
        ops.selective_scan_bwd(*g32, torch.randn(1, 16, 512, device="cuda").bfloat16(), ck32, True)
    # C ABI: dout_f32 with fp32 inputs
    u, delta, A, Bm, Cm, Dv, bias = g32
    du, dd, dB, dC = (torch.empty_like(t) for t in (u, delta, Bm, Cm))
    dA, dD, db = torch.zeros_like(A), torch.zeros_like(Dv), torch.zeros_like(bias)
    L = _lib.lib()
    ws = torch.empty(L.vmb_scan_bwd_workspace_bytes(1, 2, 16, 512), dtype=torch.uint8, device="cuda")
    P = ops._ptr
    a = _lib.ScanBwdArgs(u=P(u), delta=P(delta), A=P(A), Bm=P(Bm), Cm=P(Cm), D=P(Dv), delta_bias=P(bias), dout=P(u), ckpt=P(ck32),
                         du=P(du), ddelta=P(dd), dA=P(dA), dB=P(dB), dC=P(dC), dD=P(dD), ddelta_bias=P(db), workspace=P(ws),
                         batch=1, dim=16, seqlen=512, dstate=16, ngroups=2, u_bs=u.stride(0), u_ds=u.stride(1),
                         delta_bs=delta.stride(0), delta_ds=delta.stride(1), dout_bs=u.stride(0), dout_ds=u.stride(1),
                         du_bs=du.stride(0), du_ds=du.stride(1), ddelta_bs=dd.stride(0), ddelta_ds=dd.stride(1),
                         B_bs=Bm.stride(0), B_gs=Bm.stride(1), B_ns=Bm.stride(2), C_bs=Cm.stride(0), C_gs=Cm.stride(1),
                         C_ns=Cm.stride(2), delta_softplus=1, dtype=_lib.DT_F32, dout_f32=1)
    assert L.vmb_selective_scan_bwd(C.byref(a), ops._stream(u)) != 0
    assert "dout_f32" in L.vmb_last_error().decode()
    # ndstate: the (D,) / (B, G, L) layout only
    with pytest.raises(RuntimeError):
        selective_scan_cuda_ndstate.fwd(g[0], g[1], g[2], g[3], g[4], g[5], g[6], True, 1)


# ----------------------------------------------------------------------------- CUDA graphs
def test_cuda_graph_replay():
    from vmambair_b200 import ops
    b, D, L, N, G = 2, 64, 1024, 16, 2
    g = cuda(make_inputs(b, D, L, N, G, torch.bfloat16, seed=21))
    dout = torch.randn(b, D, L, device="cuda")

    def step():
        out, ck = ops.selective_scan_fwd(*g, True, need_ckpt=True, out_float=True)
        return (out,) + tuple(ops.selective_scan_bwd(*g, dout, ck, True, dout_float=True))

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()  # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured[0], eager[0])  # the forward is deterministic
    for n, c, e in zip(GRAD_NAMES, captured[1:], eager[1:]):
        # dB, dC, dA, dD, ddelta_bias are reduced with fp32 atomics: equal up to summation order
        tol = 2.0 ** -7 if c.dtype == torch.bfloat16 else 1e-5
        torch.testing.assert_close(c, e, rtol=tol, atol=1e-5 * e.abs().max().item(), msg=n)
