"""The `selective_scan_cuda` stand-in (z-gated forward, pair-layout checkpoints with the last state, gate backward) and the
autograd entry `mamba_selective_scan_fn`, against the float64 oracle composed with the gate (test_scan_z_cpu.py), on both forward
paths (TMA kernel; generic kernel for an L < 512 or a u that is not 16 B aligned)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import cscan
from tests.test_scan_z_cpu import CASES, GRADS, case_inputs

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def make_inputs(b, D, L, N, G, dtype, seed=0, has_D=True, has_bias=True, has_z=True):
    """the reference test's distributions (test_selective_scan.py:411-441), rounded to `dtype` once"""
    g = torch.Generator().manual_seed(seed)
    A = -0.5 * torch.rand(D, N, generator=g)
    Bm, Cm = torch.randn(b, G, N, L, generator=g).to(dtype), torch.randn(b, G, N, L, generator=g).to(dtype)
    Dv = torch.randn(D, generator=g) if has_D else None
    z = torch.randn(b, D, L, generator=g).to(dtype) if has_z else None
    bias = 0.5 * torch.rand(D, generator=g) if has_bias else None
    u = torch.randn(b, D, L, generator=g).to(dtype)
    delta = (0.5 * torch.rand(b, D, L, generator=g)).to(dtype)
    return u, delta, A, Bm, Cm, Dv, z, bias


def cuda(ts):
    return [None if t is None else t.cuda() for t in ts]


def oracle(ins, dout, softplus):
    """float64 (out or out_z, grads in GRADS order) and the fp32 oracle's last state, on the dtype-rounded inputs"""
    u, delta, A, Bm, Cm, Dv, z, bias = ins
    ref = cscan.scan_fwd(u, delta, A, Bm, Cm, Dv, bias, softplus, fp64=True)
    _, last = cscan.scan_fwd(u, delta, A, Bm, Cm, Dv, bias, softplus, return_last_state=True)
    if z is None:
        du, dd, dA, dB, dC, dD, db = cscan.scan_bwd(u, delta, A, Bm, Cm, Dv, bias, dout, softplus)
        return ref, (du, dd, dA, dB, dC, None, dD, db), last
    z64, g64 = z.double(), dout.double()
    s = torch.sigmoid(z64)
    dz = g64 * ref * s * (1 + z64 * (1 - s))
    du, dd, dA, dB, dC, dD, db = cscan.scan_bwd(u, delta, A, Bm, Cm, Dv, bias, g64 * z64 * s, softplus)
    return ref * z64 * s, (du, dd, dA, dB, dC, dz, dD, db), last


def tolerances(dtype, has_z):
    """test_selective_scan.py:398-404"""
    rtol, atol = (6e-4, 2e-3) if dtype == torch.float32 else (3e-3, 5e-3)
    if dtype == torch.bfloat16:
        rtol, atol = 3e-2, 5e-2
    rtolw, atolw = 1e-3, 1e-3
    if has_z:
        rtolw, atolw = max(rtolw, rtol), max(atolw, atol)
    return rtol, atol, rtolw, atolw


SUMS = ("dA", "dB", "dC", "dD", "dbias")  # sums over the batch and / or the sequence


def close(x, ref, rtol, atol, what, floor=0.0):
    """|x - ref| <= atol + rtol |ref| + floor * max |ref| element-wise"""
    x = x.detach().double().cpu()
    ok = (x - ref).abs() <= atol + rtol * ref.abs() + floor * ref.abs().max()
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} / {ok.numel()} beyond rtol {rtol} atol {atol}; max err {(x - ref).abs().max():.3e}"


def run_fn(g, softplus, dout, misalign=False):
    """mamba_selective_scan_fn forward (return_last_state=True) + backward -> (out, state, grads in GRADS order).
    misalign: u one element into its storage, so that its rows are not 16 B aligned"""
    from vmambair_b200.selective_scan import mamba_selective_scan_fn
    ts = [None if t is None else t.detach().clone() for t in g]
    if misalign:  # vmb_selective_scan_fwd / _bwd: no 16 B rows (vec_ok false), so neither TMA kernel takes the call
        ts[0] = torch.empty(ts[0].numel() + 1, dtype=ts[0].dtype, device=ts[0].device)[1:].view(ts[0].shape).copy_(ts[0])
        assert ts[0].data_ptr() % 16 != 0
    u, delta, A, Bm, Cm, Dv, z, bias = [None if t is None else t.requires_grad_() for t in ts]
    out, state = mamba_selective_scan_fn(u, delta, A, Bm, Cm, Dv, z=z, delta_bias=bias, delta_softplus=softplus, return_last_state=True)
    out.backward(dout.cuda())
    grads = [t.grad if t is not None else None for t in (u, delta, A, Bm, Cm, z, Dv, bias)]
    return out, state, grads


# ----------------------------------------------------------------------------- the reference test's parametrization (:372-502)
@pytest.mark.parametrize("path", ["tma", "generic"])
@pytest.mark.parametrize("L", [64, 777, 4096])
@pytest.mark.parametrize("groups", [1, 2])
@pytest.mark.parametrize("softplus", [False, True])
@pytest.mark.parametrize("has_bias", [False, True])
@pytest.mark.parametrize("has_D", [False, True])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("has_z", [False, True])
def test_reference_parametrization(has_z, dtype, has_D, has_bias, softplus, groups, L, path):
    if path == "tma" and L < 512:
        pytest.skip("L < 512 runs the generic forward only")
    b, D, N = 2, 64, 16
    ins = make_inputs(b, D, L, N, groups, dtype, seed=L + 7 * groups, has_D=has_D, has_bias=has_bias, has_z=has_z)
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(5)).to(dtype)
    out, state, grads = run_fn(cuda(ins), softplus, dout, misalign=path == "generic")
    ref, rgrads, last = oracle(ins, dout, softplus)
    rtol, atol, rtolw, atolw = tolerances(dtype, has_z)
    assert out.dtype == dtype and state.dtype == torch.float32 and tuple(state.shape) == (b, D, N)
    close(out, ref, rtol, atol, "out")
    close(state, last.double(), rtol, atol, "last state")
    tol = {"du": (2 * rtol, 2 * atol), "ddelta": (5 * rtol, 10 * atol), "dA": (rtolw, 5 * atolw), "dB": (rtol, atol),
           "dC": (rtol, atol), "dz": (rtolw, atolw), "dD": (rtolw, atolw), "dbias": (rtolw, atolw)}
    for name, gx, gr in zip(GRADS, grads, rgrads):
        if gr is None:
            assert gx is None, name
        else:  # an element of a sum that cancels to near zero keeps the fp32 rounding of its large terms (dA reaches 1e6 at L = 4096)
            close(gx, gr, *tol[name], name, floor=1e-5 if name in SUMS else 0.0)


# ----------------------------------------------------------------------------- golden vectors of the reference function
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden(name):
    c = CASES[name]
    sp = bool(int(c["softplus"]))
    out, state, grads = run_fn(cuda(case_inputs(c)), sp, c["dout"])
    rtol, atol, rtolw, atolw = tolerances(torch.float32, True)
    close(out, c["out"].double(), rtol, atol, "out")
    close(state, c["last_state"].double(), rtol, atol, "last state")
    for gname, g in zip(GRADS, grads):
        if gname in c:
            close(g, c[gname].double(), rtolw, 5 * atolw, gname)


# ----------------------------------------------------------------------------- the last state at every seqlen
@pytest.mark.parametrize("has_z", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("L", [65, 100, 112, 113, 128, 129, 777])
def test_ragged_last_state(L, dtype, has_z):
    from vmambair_b200 import selective_scan_cuda, selective_scan_cuda_core
    ins = make_inputs(2, 32, L, 16, 2, dtype, seed=L, has_z=has_z)
    u, delta, A, Bm, Cm, Dv, z, bias = cuda(ins)
    out, x, *rest = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, True)
    assert len(rest) == int(has_z) and tuple(x.shape) == (2, 32, (L + 63) // 64, 32)
    _, last = cscan.scan_fwd(*[t for i, t in enumerate(ins) if i != 6], True, return_last_state=True)
    close(x[:, :, -1, 1::2], last.double(), 1e-4, 1e-4, "last state")
    assert bool((x[..., 0::2] == 0).all())
    # every interval the core layout writes holds the same state, bit for bit
    _, ck = selective_scan_cuda_core.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1)
    full = L // 64
    assert torch.equal(x[:, :, :full, 1::2], ck[:, :, :full])


# ----------------------------------------------------------------------------- z = None is the core operator
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("L", [300, 1024])
def test_no_z_equals_core(L, dtype):
    from vmambair_b200 import selective_scan_cuda, selective_scan_cuda_core
    ins = cuda(make_inputs(2, 64, L, 16, 2, dtype, seed=3, has_z=False))
    u, delta, A, Bm, Cm, Dv, _, bias = ins
    out, x = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, None, bias, True)
    out_c, ck = selective_scan_cuda_core.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1)
    assert torch.equal(out, out_c)
    dout = torch.randn_like(out)
    torch.use_deterministic_algorithms(True)
    try:
        g = selective_scan_cuda.bwd(u, delta, A, Bm, Cm, Dv, None, bias, dout, x, None, None, True, False)
        gc = selective_scan_cuda_core.bwd(u, delta, A, Bm, Cm, Dv, bias, dout, ck, True, 1)
    finally:
        torch.use_deterministic_algorithms(False)
    assert len(g) == 7
    for a, c in zip(g, gc):
        assert torch.equal(a, c)


# ----------------------------------------------------------------------------- the reference's call patterns
def test_realsr_mamba_ssm_calls():
    """MambaRealSR11_arch.py:294-295,309-313 (SSMODE = "mamba_ssm"): 4-D B/C, z = None, out = dz = None, recompute_out_z = False"""
    from vmambair_b200 import selective_scan_cuda
    u, delta, A, Bm, Cm, Dv, _, bias = cuda(make_inputs(1, 32, 640, 16, 4, torch.float32, seed=9, has_z=False))
    out, x, *rest = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, None, bias, True)
    assert rest == []
    dout = torch.randn_like(out)
    du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = selective_scan_cuda.bwd(
        u, delta, A, Bm, Cm, Dv, None, bias, dout, x, None, None, True, False)
    assert rest == [] and dB.shape == Bm.shape and dC.shape == Cm.shape and dA.dtype == torch.float32


def test_reference_wrapper_rest():
    """test_selective_scan.py:60,86,105-108,128: out_z is rest[0] of fwd, dz is rest[0] of bwd; 3-D B/C come back 3-D"""
    from vmambair_b200 import selective_scan_cuda
    u, delta, A, Bm, Cm, Dv, z, bias = cuda(make_inputs(2, 16, 200, 8, 1, torch.float16, seed=4))
    Bm, Cm = Bm[:, 0], Cm[:, 0]
    out, x, *rest = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, False)
    out_z = rest[0]
    close(out_z, (out.double() * F.silu(z.double())).cpu(), 2 ** -9, 1e-4, "out_z")
    dout = torch.randn_like(out)
    du, ddelta, dA, dB, dC, dD, ddelta_bias, *rest = selective_scan_cuda.bwd(
        u, delta, A, Bm, Cm, Dv, z, bias, dout, x, out, None, False, False)
    assert len(rest) == 1 and rest[0].shape == z.shape and rest[0].dtype == z.dtype
    assert dB.shape == Bm.shape and dC.shape == Cm.shape


@pytest.mark.parametrize("dtype", DTYPES)
def test_bwd_buffers(dtype):
    """a preallocated dz is written in place; recompute_out_z returns the forward's out_z (bit for bit in fp32; 16-bit: the
    forward rounds the fp32 accumulator times the gate once, the recompute starts from the rounded `out`)"""
    from vmambair_b200 import selective_scan_cuda
    u, delta, A, Bm, Cm, Dv, z, bias = cuda(make_inputs(2, 64, 1024, 16, 2, dtype, seed=8))
    out, x, out_z = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, True)
    dout = torch.randn_like(out)
    dz_ = torch.full_like(z, float("nan"))
    res = selective_scan_cuda.bwd(u, delta, A, Bm, Cm, Dv, z, bias, dout, x, out, dz_, True, True)
    assert len(res) == 9 and res[7] is dz_ and bool(torch.isfinite(dz_).all())
    ref_dz = selective_scan_cuda.bwd(u, delta, A, Bm, Cm, Dv, z, bias, dout, x, out, None, True, False)[7]
    assert torch.equal(dz_, ref_dz)
    if dtype == torch.float32:
        assert torch.equal(res[8], out_z)
    else:
        torch.testing.assert_close(res[8], out_z, rtol=2 * (2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11), atol=1e-6)


# ----------------------------------------------------------------------------- reproducibility, graphs, launches
def test_deterministic_repeats_and_graph_replay():
    from vmambair_b200 import selective_scan_cuda
    u, delta, A, Bm, Cm, Dv, z, bias = cuda(make_inputs(2, 64, 2048, 16, 2, torch.bfloat16, seed=12))
    out, x, out_z = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, True)
    dout = torch.randn_like(out)
    torch.use_deterministic_algorithms(True)
    try:
        g1 = selective_scan_cuda.bwd(u, delta, A, Bm, Cm, Dv, z, bias, dout, x, out, None, True, False)
        g2 = selective_scan_cuda.bwd(u, delta, A, Bm, Cm, Dv, z, bias, dout, x, out, None, True, False)
    finally:
        torch.use_deterministic_algorithms(False)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside the capture
        selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gout, gx, gz = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, True)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gout, out) and torch.equal(gx, x) and torch.equal(gz, out_z)


def test_launch_census():
    from vmambair_b200 import ops, selective_scan_cuda
    u, delta, A, Bm, Cm, Dv, z, bias = cuda(make_inputs(2, 64, 1024, 16, 2, torch.bfloat16, seed=13))
    n0 = ops.launch_count()
    out, x, out_z = selective_scan_cuda.fwd(u, delta, A, Bm, Cm, Dv, z, bias, True)
    n1 = ops.launch_count()
    selective_scan_cuda.bwd(u, delta, A, Bm, Cm, Dv, z, bias, torch.randn_like(out), x, out, None, True, False)
    n2 = ops.launch_count()
    assert (n1 - n0, n2 - n1) == (1, 3)  # gated forward; gate backward + scan backward + its finalize


# ----------------------------------------------------------------------------- invalid input
def test_invalid_input():
    from vmambair_b200 import _lib, ops, selective_scan_cuda
    u, delta, A, Bm, Cm, Dv, z, bias = cuda(make_inputs(1, 16, 256, 8, 1, torch.bfloat16, seed=1))
    with pytest.raises(RuntimeError, match="complex"):
        selective_scan_cuda.fwd(u, delta, torch.complex(A, A), Bm, Cm, Dv, z, bias, True)
    with pytest.raises(RuntimeError, match="variable"):
        selective_scan_cuda.fwd(u, delta, A, Bm[0, 0], Cm[0, 0], Dv, z, bias, True)
    P = ops._ptr
    out, out_z = torch.empty(u.shape, dtype=torch.float32, device="cuda"), torch.empty_like(u)
    b, d, l = u.shape

    def call(out, ckpt, out_f32, ckpt_pairs):
        a = _lib.ScanFwdArgs(
            u=P(u), delta=P(delta), A=P(A), Bm=P(Bm), Cm=P(Cm), D=P(Dv), delta_bias=P(bias), out=P(out), ckpt=P(ckpt),
            batch=b, dim=d, seqlen=l, dstate=8, ngroups=1, u_bs=u.stride(0), u_ds=u.stride(1), delta_bs=delta.stride(0),
            delta_ds=delta.stride(1), out_bs=out.stride(0), out_ds=out.stride(1), B_bs=Bm.stride(0), B_gs=Bm.stride(1),
            B_ns=Bm.stride(2), C_bs=Cm.stride(0), C_gs=Cm.stride(1), C_ns=Cm.stride(2), delta_softplus=1, dtype=ops._DT[u.dtype],
            out_f32=out_f32, z=P(z), out_z=P(out_z), z_bs=z.stride(0), z_ds=z.stride(1), out_z_bs=out_z.stride(0),
            out_z_ds=out_z.stride(1), ckpt_pairs=ckpt_pairs)
        return _lib.lib().vmb_selective_scan_fwd(C.byref(a), ops._stream(u))

    assert call(out, None, 1, 0) == 1 and "out_f32" in _lib.lib().vmb_last_error().decode()
    ck = torch.empty((b, d, (l + 63) // 64, 8), dtype=torch.float32, device="cuda")
    assert call(torch.empty_like(u), ck, 0, 0) == 1 and "pair" in _lib.lib().vmb_last_error().decode()
    assert call(torch.empty_like(u), None, 0, 0) == 0
    torch.cuda.synchronize()
