"""Deterministic mode of the operator layer: the scan backward (flat and grouped, TMA and generic kernels) and the weight-gradient GEMM
behind cross_selective_scan, selected by torch.use_deterministic_algorithms(True) or deterministic=True.  Each case asserts which kernel
its layout takes (the launchers' conditions), that repeated runs are bit-equal, that the workspace contents never matter, that the
accumulate-into contract holds, and that the values match the float64 oracle, the reference-kernel goldens and the atomic path."""
import os
import subprocess
import sys
import warnings

import pytest
import torch

from tests import test_bench_parity_gpu as tbp
from tests import test_cross_selective_scan_gpu as tcs
from tests import test_scan_gpu as tsg
from tests import test_scan_oflex_gpu as tso
from tests.test_scan_oflex_gpu import GRAD_NAMES, U16, bwd_takes_tma, cuda, make_inputs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def det_flag():
    """torch.use_deterministic_algorithms(True) for the test, the previous setting restored afterwards"""
    prev, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn_only)


def tags_of(fn):
    """-> (fn's result, the set of library timing tags it ran)"""
    from vmambair_b200 import ops
    rec = []
    ops.set_timing(rec)
    try:
        res = fn()
        torch.cuda.synchronize()
    finally:
        ops.set_timing(None)
    return res, {r[0] for r in rec}


def tma_ss(b, D):
    """the state split scan_bwd_tma_pick chooses (bwd_tma_ss, csrc/scan_bwd_tma.cu)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ss = 1
    while ss < 4 and (b * D) // (2 * 4 // ss) * 2 <= 2 * sms:
        ss <<= 1
    return ss


def assert_all_equal(a, b, what):
    for n, x, y in zip(GRAD_NAMES, a, b):
        if x is None:
            assert y is None, (what, n)
            continue
        assert torch.equal(x, y), f"{what}: {n} differs (max {float((x.double() - y.double()).abs().max()):.3e})"


# ----------------------------------------------------------------------------- flat operator
# (name, b, D, L, N, G, dtype, dout fp32, has_D, has_bias, softplus, layout) -> TMA (with its state split) or generic
SS_OF = {"tma_ss1_bf16": 1, "tma_ss2_fp16": 2, "tma_ss4_fp32": 4}  # the state split each of these batch sizes selects
FLAT = [
    ("tma_ss1_bf16", 4, 384, 1024, 16, 4, torch.bfloat16, False, True, True, True, "dense"),
    ("tma_ss2_fp16", 2, 384, 1024, 16, 2, torch.float16, False, True, True, True, "dense"),
    ("tma_ss4_fp32", 1, 384, 1024, 16, 1, torch.float32, False, True, True, True, "dense"),
    ("tma_fp32_noD_nobias", 2, 64, 1024, 16, 2, torch.float32, False, False, False, False, "dense"),
    ("tma_bf16_dout32", 2, 64, 1024, 16, 2, torch.bfloat16, True, True, True, True, "dense"),
    ("tma_fp16_dout32_nosoftplus", 2, 64, 1024, 16, 4, torch.float16, True, True, False, False, "dense"),
    ("tma_bf16_dstate12", 2, 64, 1024, 12, 1, torch.bfloat16, False, True, True, True, "dense"),
    ("generic_short_fp32", 2, 32, 300, 16, 2, torch.float32, False, True, True, True, "dense"),
    ("generic_short_bf16_noD", 2, 32, 300, 16, 4, torch.bfloat16, False, False, True, False, "dense"),
    ("generic_dstate20_fp16", 1, 32, 640, 20, 1, torch.float16, False, True, True, True, "dense"),
    ("generic_dstate64_fp32", 1, 16, 700, 64, 2, torch.float32, False, True, False, True, "dense"),
    ("generic_offset_bf16", 2, 32, 1024, 16, 2, torch.bfloat16, False, True, True, True, "offset"),
    ("generic_short_fp16_dout32", 2, 32, 300, 16, 2, torch.float16, True, True, True, True, "dense"),
    ("generic_offset_bf16_dout32", 2, 32, 1024, 16, 4, torch.bfloat16, True, False, False, True, "offset"),
    ("tma_ndstate_fp32", 2, 48, 1024, 1, 2, torch.float32, False, True, True, True, "dense"),
    ("generic_ndstate_bf16", 2, 48, 300, 1, 1, torch.bfloat16, False, True, True, True, "dense"),
    ("large_8x384x4096_bf16", 8, 384, 4096, 16, 4, torch.bfloat16, False, True, True, True, "dense"),
]


def _offset(t):
    """the same values one element into their storage: off the 16 B grid, so the launcher leaves the TMA kernel"""
    if t is None:
        return None
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def flat_case(case):
    name, b, D, L, N, G, dtype, d32, has_D, has_bias, softplus, layout = case
    from vmambair_b200 import ops
    ins = make_inputs(b, D, L, N, G, dtype, seed=L + N + G, has_D=has_D, has_bias=has_bias)
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(L + 7))
    dout = dout if d32 else dout.to(dtype)
    g, gd = cuda(ins), dout.cuda()
    if layout == "offset":
        g = [g[0], _offset(g[1])] + g[2:]  # delta off the grid
        gd = _offset(gd)
    _, ck = ops.selective_scan_fwd(*g, softplus, need_ckpt=True)
    if layout == "dense":  # TMA or generic by sizes alone; an operand off the 16 B grid always leaves the TMA kernel
        assert bwd_takes_tma(g[0], N, G) == (not name.startswith("generic")), name
    if name in SS_OF:
        assert tma_ss(b, D) == SS_OF[name], (name, tma_ss(b, D))
    return ins, dout, g, gd, ck, softplus, d32


def run_flat(g, gd, ck, softplus, d32, **kw):
    from vmambair_b200 import ops
    return ops.selective_scan_bwd(*g, gd, ck, softplus, dout_float=d32, **kw)


@pytest.mark.parametrize("case", FLAT, ids=[c[0] for c in FLAT])
def test_flat_repeatable_and_workspace_independent(case):
    _, _, g, gd, ck, softplus, d32 = flat_case(case)
    first, tags = tags_of(lambda: run_flat(g, gd, ck, softplus, d32, deterministic=True))
    assert tags == {"scan_bwd_det"}
    for _ in range(5):
        assert_all_equal(first, run_flat(g, gd, ck, softplus, d32, deterministic=True), "repeat")
    # every slot the finalize reads is written: NaN-filled and zero-filled workspaces give the same finite bits
    nws = _flat_ws_bytes(g, gd, ck, softplus, d32)
    assert nws > 0
    for fill in (float("nan"), 0.0):
        ws = torch.full(((nws + 3) // 4,), fill, dtype=torch.float32, device="cuda")
        got = run_flat(g, gd, ck, softplus, d32, deterministic=True, workspace=ws)
        assert_all_equal(first, got, f"workspace filled with {fill}")
    for t in first:
        assert t is None or bool(torch.isfinite(t).all())
    # accumulate-into: prefilled dA / dD / dbias receive the prefill plus one fixed-order sum
    pre = [torch.randn_like(first[2])] + [None if first[i] is None else torch.randn_like(first[i]) for i in (5, 6)]
    acc = [None if t is None else t.clone() for t in pre]
    got = run_flat(g, gd, ck, softplus, d32, deterministic=True, zeroed=tuple(acc))
    for i, p in zip((2, 5, 6), pre):
        if p is not None:
            assert torch.equal(got[i], p + first[i]), GRAD_NAMES[i]
    assert_all_equal(first[:2] + (None,) + first[3:5], got[:2] + (None,) + got[3:5], "accumulate-into: other outputs")
    # the atomic path: du / ddelta bit-equal (no sum across CTAs), the rest within fp32 reassociation
    atomic, tags = tags_of(lambda: run_flat(g, gd, ck, softplus, d32, deterministic=False))
    assert tags == {"scan_bwd"}
    for i, n_ in enumerate(GRAD_NAMES):
        if first[i] is None:
            continue
        if n_ in ("du", "ddelta"):
            assert torch.equal(first[i], atomic[i]), n_
            continue
        x, y = first[i].double(), atomic[i].double()
        scale = y.abs().max().item()
        bound = 2 * U16.get(first[i].dtype, 0.0) * y.abs() + 1e-4 * scale  # a 16-bit result may round the reassociated sum either way
        assert bool(((x - y).abs() <= bound).all()), f"{n_}: det vs atomic max {float((x - y).abs().max()):.3e} (scale {scale:.3e})"


def _flat_ws_bytes(g, gd, ck, softplus, d32):
    """vmb_scan_bwd_det_workspace_bytes on the arguments the wrapper builds (captured by running it with a recording workspace)"""
    from vmambair_b200 import ops
    seen = []
    orig = ops._workspace

    def spy(nbytes, given, dev, who):
        seen.append(nbytes)
        return orig(nbytes, given, dev, who)
    ops._workspace = spy
    try:
        run_flat(g, gd, ck, softplus, d32, deterministic=True)
    finally:
        ops._workspace = orig
    return seen[0]


def test_flat_workspace_formula():
    """the query returns 16 nc b G ceil16(N)/2 L + 4 b D (N + 2) bytes, nc = the CTAs (TMA) / warps (generic) sharing a group"""
    cases = [((4, 384, 1024, 16, 4, torch.bfloat16), 96 // 8), ((2, 384, 1024, 16, 2, torch.bfloat16), 192 // 4),
             ((1, 384, 1024, 16, 1, torch.bfloat16), 384 // 2), ((2, 32, 300, 16, 2, torch.float32), 16 // 2)]
    for (b, D, L, N, G, dt), nc in cases:
        g = cuda(make_inputs(b, D, L, N, G, dt, seed=1))
        from vmambair_b200 import ops
        _, ck = ops.selective_scan_fwd(*g, True, need_ckpt=True)
        gd = torch.randn(b, D, L, device="cuda").to(dt)
        if L >= 512:
            assert bwd_takes_tma(g[0], N, G) and (D // G) // nc == 2 * 4 // tma_ss(b, D)
        nbytes = _flat_ws_bytes(g, gd, ck, True, False)
        assert nbytes == 16 * nc * b * G * 8 * L + 4 * b * D * (N + 2), ((b, D, L, N, G), nbytes)


def test_flat_values_vs_oracle_and_reference_kernels(det_flag, monkeypatch):
    """under the flag, the flat operator's own value tests hold with the deterministic kernels: the float64-oracle bounds of
    test_scan_gpu.py / test_scan_oflex_gpu.py and the reference-kernel goldens at test_bench_parity_gpu.py's tolerances"""
    def run():
        for shape in tsg.BWD_SHAPES:
            tsg.test_bwd_vs_oracle(shape, torch.bfloat16, True)
            tsg.test_bwd_vs_oracle(shape, torch.float32, False)
        tsg.test_bwd_optional_args_none()
        tsg.test_bwd_model_like_full_row()
        for name in ["a", "b", "c", "d", "e"]:
            tsg.test_bwd_golden_vectors(os.path.join(ROOT, "tests", "golden"), name)
        for dt in tso.DT16:
            tso.test_bwd_fp32_dout("tma", dt, (True, True, True))
            tso.test_bwd_fp32_dout_generic_shapes(dt)
        for b in (8, 4, 1):
            for it in (torch.float32, torch.bfloat16):
                tbp.test_scan_fwd_bwd_vs_reference_cuda_kernel(b, it)
        for case in [("oflex", torch.bfloat16), ("oflex", torch.float16), ("ndstate", torch.float32), ("ndstate", torch.bfloat16)]:
            tso.test_vs_reference_cuda_kernels(case)
    _, tags = tags_of(run)
    assert "scan_bwd_det" in tags and "scan_bwd" not in tags, tags


# ----------------------------------------------------------------------------- grouped operator
GROUPED = [((16, 40, 24), 2, torch.float32, False), ((96, 64, 64), 8, torch.bfloat16, False), ((96, 64, 64), 1, torch.float16, False),
           ((48, 16, 24), 4, torch.bfloat16, True), ((16, 20, 30), 1, torch.float32, False)]


def _grouped_run(shape, batch, dtype, sliced, G=4, **kw):
    from vmambair_b200 import ops
    C, H, W = shape
    L, N = H * W, 16
    us, deltas, Bs, Cs, A, Dv, bias = tcs._grouped_operands(batch, C, L, N, dtype, seed=C + L + batch, sliced=sliced)
    revs = [0, 0, 1, 1][:G]
    us, deltas, Bs, Cs = us[:G], deltas[:G], Bs[:G], Cs[:G]
    A, Dv, bias = A[:G * C], Dv[:G * C], bias[:G * C]
    rn, _ = tcs._gen(L)
    douts = [rn(batch, C, L).to(dtype).cuda() for _ in range(G)]
    _, ckpt = ops.selective_scan_fwd_grouped(us, deltas, Bs, Cs, revs, A, Dv, bias, True, need_ckpt=True)
    return lambda **k2: ops.selective_scan_bwd_grouped(us, deltas, Bs, Cs, douts, revs, A, Dv, bias, ckpt, True, **{**kw, **k2})


def _flatten_grouped(r):
    dus, dds, dA, dBs, dCs, dD, dbias = r
    return (torch.stack(dus), torch.stack(dds), dA, torch.stack(dBs), torch.stack(dCs), dD, dbias)


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("shape,batch,dtype,sliced", GROUPED)
def test_grouped_repeatable_and_workspace_independent(shape, batch, dtype, sliced, G):
    run = _grouped_run(shape, batch, dtype, sliced, G)
    first, tags = tags_of(lambda: _flatten_grouped(run(deterministic=True)))
    assert tags == {"scan_bwd_det"}
    for _ in range(5):
        assert_all_equal(first, _flatten_grouped(run(deterministic=True)), "repeat")
    for t in first:
        assert bool(torch.isfinite(t).all())
    for fill in (float("nan"), 0.0):
        ws = torch.full((64 << 20,), fill, dtype=torch.float32, device="cuda")
        assert_all_equal(first, _flatten_grouped(run(deterministic=True, workspace=ws)), f"workspace filled with {fill}")
    pre = [torch.randn_like(first[i]) for i in (2, 5, 6)]
    got = _flatten_grouped(run(deterministic=True, zeroed=tuple(p.clone() for p in pre)))
    for i, p in zip((2, 5, 6), pre):
        assert torch.equal(got[i], p + first[i]), GRAD_NAMES[i]
    atomic, tags = tags_of(lambda: _flatten_grouped(run(deterministic=False)))
    assert tags == {"scan_bwd"}
    for i, n in enumerate(GRAD_NAMES):
        if n in ("du", "ddelta"):
            assert torch.equal(first[i], atomic[i]), n
        else:
            x, y = first[i].double(), atomic[i].double()
            scale = y.abs().max().item()
            tol = 2 * U16.get(first[i].dtype, 0.0) * y.abs() + 1e-4 * scale  # one 16-bit ulp: rounding either way
            assert bool(((x - y).abs() <= tol).all()), f"{n}: det vs atomic max {float((x - y).abs().max()):.3e}"


def test_grouped_values_under_flag(det_flag):
    """the grouped operator's value tests (against the flat operator on gathered / flipped copies) with both sides deterministic"""
    def run():
        for shape in tcs.SHAPES:
            for batch in (1, 8):
                for dt in tcs.DTYPES:
                    if dt != torch.float32 and shape[1] * shape[2] % 8:
                        continue
                    tcs.test_grouped_bwd_equals_flat_bwd_on_gathered_operands(shape, batch, dt)
        for dt in tcs.DTYPES:
            tcs.test_grouped_bwd_channel_slice_sources(dt)
    _, tags = tags_of(run)
    assert "scan_bwd_det" in tags and "scan_bwd" not in tags, tags


# ----------------------------------------------------------------------------- pixlin_wgrad
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(4, 136, 48, 4096), (1, 320, 96, 4096), (2, 64, 70, 520), (8, 40, 24, 1024)])
@pytest.mark.parametrize("mode", ["plain", "dbias", "per_batch", "per_batch_dbias"])
def test_wgrad_repeatable_and_exact_contract(mode, shape, dtype):
    from vmambair_b200 import ops
    B, M, K, L = shape
    gen = torch.Generator().manual_seed(M + K)
    dy = torch.randn(B, M, L, generator=gen).to(dtype).cuda()
    x = torch.randn(B, K, L, generator=gen).to(dtype).cuda()
    per_batch = mode.startswith("per_batch")
    with_bias = mode.endswith("dbias")
    oshape = (B, M, K) if per_batch else (M, K)

    def run(det, out=None, dbias=None, workspace=None):
        out = torch.zeros(oshape, device="cuda") if out is None else out
        dbias = (torch.zeros(M, device="cuda") if with_bias else None) if dbias is None else dbias
        ops.pixlin_wgrad(dy, x, per_batch=per_batch, out=out, dbias=dbias, deterministic=det, workspace=workspace)
        return out, dbias

    (w0, b0), tags = tags_of(lambda: run(True))
    assert tags == {"wgrad_det"}
    for _ in range(5):
        w1, b1 = run(True)
        assert torch.equal(w0, w1) and (b0 is None or torch.equal(b0, b1))
    for fill in (float("nan"), 0.0):
        ws = torch.full((B * 64 * M * (K + 1),), fill, device="cuda")
        w1, b1 = run(True, workspace=ws)
        assert torch.equal(w0, w1) and (b0 is None or torch.equal(b0, b1)) and bool(torch.isfinite(w1).all())
    pw = torch.randn(oshape, device="cuda")
    pb = torch.randn(M, device="cuda") if with_bias else None
    w1, b1 = run(True, out=pw.clone(), dbias=None if pb is None else pb.clone())
    assert torch.equal(w1, pw + w0) and (pb is None or torch.equal(b1, pb + b0))
    # values: float64 product of the 16-bit operands, and the atomic kernel within fp32 reassociation
    ref = torch.einsum("bml,bkl->bmk", dy.double(), x.double())
    ref = ref if per_batch else ref.sum(0)
    terms = torch.einsum("bml,bkl->bmk", dy.double().abs(), x.double().abs())
    terms = terms if per_batch else terms.sum(0)
    assert bool(((w0.double() - ref).abs() <= 1e-4 * terms + 1e-6).all())
    (wa, ba), tags = tags_of(lambda: run(False))
    assert tags == {"wgrad"}
    assert bool(((w0.double() - wa.double()).abs() <= 1e-4 * terms + 1e-6).all())
    if with_bias:
        rb = dy.double().sum((0, 2))
        assert bool(((b0.double() - rb).abs() <= 1e-4 * dy.double().abs().sum((0, 2)) + 1e-6).all())


# ----------------------------------------------------------------------------- public operators under the flag
def _scan_fn_grads(dtype, seed=3):
    from vmambair_b200.selective_scan import selective_scan_fn
    ins = make_inputs(2, 64, 1024, 16, 2, dtype, seed=seed)
    leaves = [None if t is None else t.cuda().requires_grad_() for t in ins]
    out = selective_scan_fn(*leaves, delta_softplus=True)
    out.float().square().sum().backward()
    return tuple(t.grad for t in leaves)


def test_selective_scan_fn_under_flag(det_flag):
    a, tags = tags_of(lambda: _scan_fn_grads(torch.bfloat16))
    assert "scan_bwd_det" in tags and "scan_bwd" not in tags
    b, _ = tags_of(lambda: _scan_fn_grads(torch.bfloat16))
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_selective_scan_fn_flag_off_keeps_atomic_path():
    assert not torch.are_deterministic_algorithms_enabled()
    _, tags = tags_of(lambda: _scan_fn_grads(torch.float32))
    assert "scan_bwd" in tags and "scan_bwd_det" not in tags


@pytest.mark.parametrize("module", ["core", "oflex", "ndstate"])
def test_reference_modules_under_flag(module, det_flag):
    from vmambair_b200 import selective_scan_cuda_core, selective_scan_cuda_ndstate, selective_scan_cuda_oflex
    dt = torch.float32 if module == "core" else torch.bfloat16
    b, D, L, G = 2, 96, 1024, 4
    u, delta, A, Bm, Cm, Dv, bias = cuda(make_inputs(b, D, L, 16, G, dt, seed=4))
    if module == "ndstate":
        A, Bm, Cm = A[:, 0].contiguous(), Bm[:, :, 0].contiguous(), Cm[:, :, 0].contiguous()
        m = selective_scan_cuda_ndstate
        out, x = m.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1)
    elif module == "oflex":
        m = selective_scan_cuda_oflex
        out, x = m.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1, True)
    else:
        m = selective_scan_cuda_core
        out, x = m.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1)
    dout = torch.randn_like(out)
    r1, tags = tags_of(lambda: m.bwd(u, delta, A, Bm, Cm, Dv, bias, dout, x, True, 1))
    assert tags == {"scan_bwd_det"}
    r2 = m.bwd(u, delta, A, Bm, Cm, Dv, bias, dout, x, True, 1)
    assert all(torch.equal(p, q) for p, q in zip(r1, r2))


_CHILD = r"""
import sys, torch
sys.path.insert(0, {root!r})
torch.use_deterministic_algorithms(True)
from tests.test_deterministic_gpu import {fn}
{fn}()
print("CHILD OK")
"""


def _in_child(fn):
    """runs fn of this module in a fresh interpreter with CUBLAS_WORKSPACE_CONFIG set (torch's cuBLAS needs it under the flag)"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(root=ROOT, fn=fn)], env=env, cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and "CHILD OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def child_cross_selective_scan():
    from vmambair_b200 import cross_scan as cs
    from vmambair_b200 import ops
    paths = set()
    for (H, W, dt) in [(16, 24, torch.bfloat16), (7, 9, torch.bfloat16), (16, 24, torch.float32)]:
        for with_bias in (True, False):
            B, D, N, R = 2, 48, 16, 3
            grouped = cs.grouped_supported(D, H * W, N, dt)
            paths.add(grouped)
            gen = torch.Generator().manual_seed(H * W)
            x = torch.randn(B, D, H, W, generator=gen).to(dt).cuda()
            prm = [torch.randn(4, R + 2 * N, D, generator=gen) * 0.2, torch.randn(4, R + 2 * N, generator=gen) * 0.1,
                   torch.randn(4, D, R, generator=gen) * 0.3, torch.rand(4, D, generator=gen) * 0.1 - 4,
                   torch.log(torch.arange(1, N + 1, dtype=torch.float32)).repeat(4 * D, 1), torch.ones(4 * D)]
            if not with_bias:
                prm[1] = None

            def step():
                xs = x.clone().requires_grad_()
                ps = [None if p is None else p.cuda().requires_grad_() for p in prm]
                y = cs.cross_selective_scan(xs, ps[0], ps[1], ps[2], ps[3], ps[4], ps[5], out_norm=torch.nn.Identity())
                y.float().square().sum().backward()
                return [xs.grad] + [p.grad for p in ps if p is not None]
            rec = []
            ops.set_timing(rec)
            g1 = step()
            ops.set_timing(None)
            tags = {r[0] for r in rec}
            assert "scan_bwd_det" in tags and "scan_bwd" not in tags and "wgrad" not in tags, tags
            if dt != torch.float32 and grouped:
                assert "wgrad_det" in tags, tags
            g2 = step()
            assert all(torch.equal(a, b) for a, b in zip(g1, g2)), (H, W, dt, with_bias)
    assert paths == {True, False}, "both the grouped and the gathered path"


def child_compose_blocks():
    from vmambair_b200 import archs, ops
    archs.set_train_path("compose")
    for variant in ("sisr", "realsr"):
        torch.manual_seed(0)
        blk = archs.MamberBlock(dim=32, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias",
                                variant=variant).cuda()
        x = torch.randn(2, 32, 16, 24, device="cuda")

        def step():
            blk.zero_grad(set_to_none=True)
            xs = x.clone().requires_grad_()
            blk(xs).square().mean().backward()
            return [xs.grad] + [p.grad for p in blk.parameters() if p.grad is not None]
        rec = []
        ops.set_timing(rec)
        g1 = step()
        ops.set_timing(None)
        assert "scan_bwd_det" in {r[0] for r in rec}
        g2 = step()
        assert len(g1) == len(g2) and all(torch.equal(a, b) for a, b in zip(g1, g2)), variant


def test_cross_selective_scan_under_flag_in_child():
    _in_child("child_cross_selective_scan")


def test_compose_block_under_flag_in_child_via_set_train_path():
    _in_child("child_compose_blocks")


# ----------------------------------------------------------------------------- graph capture, warning
def test_deterministic_backward_in_cuda_graph():
    from vmambair_b200 import ops
    g = cuda(make_inputs(2, 64, 1024, 16, 2, torch.bfloat16, seed=8))
    _, ck = ops.selective_scan_fwd(*g, True, need_ckpt=True)
    dout = torch.randn(2, 64, 1024, device="cuda").to(torch.bfloat16)
    eager = ops.selective_scan_bwd(*g, dout, ck, True, deterministic=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.selective_scan_bwd(*g, dout, ck, True, deterministic=True)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = ops.selective_scan_bwd(*g, dout, ck, True, deterministic=True)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert_all_equal(eager, captured, "graph replay")


def test_fused_block_warns_once_under_flag_naming_set_train_path():
    from vmambair_b200 import archs
    blk = archs.MamberBlock(dim=32, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias").cuda()
    x = torch.randn(1, 32, 16, 24, device="cuda")
    archs._FUSED_DET_WARNED = False
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        with torch.no_grad():
            blk(x)
    assert not [w for w in rec if "use_deterministic_algorithms" in str(w.message)], "warned without the flag"
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            with torch.no_grad():
                blk(x)
                blk(x)
        hits = [w for w in rec if "use_deterministic_algorithms" in str(w.message)]
        assert len(hits) == 1 and issubclass(hits[0].category, UserWarning)
        msg = str(hits[0].message)
        assert "set_train_path('compose')" in msg and "train_ops.cu" in msg and "channel_bwd.cu" in msg and "merge" in msg
    finally:
        torch.use_deterministic_algorithms(prev)
        archs._FUSED_DET_WARNED = False
