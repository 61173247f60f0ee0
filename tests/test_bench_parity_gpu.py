"""GPU parity on the BENCHMARKED configurations (BASELINE.json configs[1], [3], [4]) against the CPU module oracle,
and of the scan operator against the reference's own CUDA kernel on identical inputs (its outputs at seeded sample
points, stored in tests/golden/scan_ref_kernel.npz by oracle/ref_kernel_golden.py).

Tolerances
  * fp32 whole-network vs oracle/oss_ref.net_forward: rtol 1e-3 / atol 1e-4 (the module bar of the block goldens);
  * bf16 whole-network (bf16 weights + activations, fp32 scan state) vs the fp32 oracle: the yardstick is the oracle itself
    evaluated with bf16 STORAGE (oss_ref.STORE_DTYPE: every tensor the pipeline keeps between kernels rounded to bf16, fp32
    arithmetic) -- on the random-init 27-block bench net that emulation is already 0.028 mean / 0.18 max |err| off the fp32
    oracle (outputs in [-0.5, 3]).  Bound: mean |err| <= 1.5 x and max |err| <= 3 x the emulation's, and absolutely
    mean <= 0.05, max <= 0.5;
  * scan vs the reference CUDA kernel: the reference test's own tolerances (test_selective_scan.py:398-400, 490-502).
"""
import pytest
import torch

import vmambair_b200.archs as archs
from oracle import cscan, oss_ref, ref_kernel_golden

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def _oracle(net, x, kind):
    cscan.use_host_threads()
    sd = {k: v.detach().float().cpu().clone() for k, v in net.state_dict().items()}
    with torch.no_grad():
        return oss_ref.net_forward(sd, x.float().cpu(), kind)


def _oracle_bf16_storage(net, x, kind):
    """the fp32 oracle with bf16 storage emulation (see module docstring)"""
    oss_ref.STORE_DTYPE = torch.bfloat16
    try:
        return _oracle(net, x, kind)
    finally:
        oss_ref.STORE_DTYPE = None


def _bf16_bound(y, ref, emu):
    assert torch.isfinite(y).all()
    err = (y.float().cpu() - ref).abs()
    e_emu = (emu - ref).abs()
    msg = f"ours max {float(err.max()):.4f} mean {float(err.mean()):.5f}; bf16-storage oracle max {float(e_emu.max()):.4f} mean {float(e_emu.mean()):.5f}"
    assert err.mean() <= 1.5 * e_emu.mean() + 1e-3 and err.max() <= 3.0 * e_emu.max() + 1e-2, msg
    assert err.mean() <= 0.05 and err.max() <= 0.5, msg


# ----------------------------------------------------------------------------- BASELINE configs[1]: the bench net
def _bench_net_and_input():
    torch.manual_seed(0)
    net = archs.MambaSISR6().eval()  # "VmambaIR-light": class default [6,2,2,1]+6 (bench.py build_net("light"))
    x = torch.rand(8, 3, 64, 64, generator=torch.Generator().manual_seed(1234))
    return net, x


def test_bench_net_fp32_fused_vs_oracle():
    net, x = _bench_net_and_input()
    ref = _oracle(net, x, "sisr")
    net = net.cuda()
    with torch.no_grad():
        y = net(x.cuda())
    torch.testing.assert_close(y.cpu(), ref, rtol=1e-3, atol=1e-4)


def test_bench_net_bf16_engine_vs_oracle():
    from vmambair_b200.engine import InferenceEngine
    net, x = _bench_net_and_input()
    ref = _oracle(net, x.to(torch.bfloat16), "sisr")  # same bf16-rounded input, fp32 arithmetic
    emu = _oracle_bf16_storage(net, x.to(torch.bfloat16), "sisr")
    eng = InferenceEngine(net, 8, 64, 64, dtype=torch.bfloat16)
    y = eng.run(x.to(torch.bfloat16)).clone()
    _bf16_bound(y, ref, emu)


# ----------------------------------------------------------------------------- configs[3] / [4] geometry vs the oracle
@pytest.mark.parametrize("cls,kind,size,batch", [("Mamber32", "mamber32", 256, 1), ("MambaRealSR11", "realsr", 128, 2)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_config45_geometry_vs_oracle(cls, kind, size, batch, dtype):
    """deraining 256x256 (L = 65 536 at level 1) and RealSR 128x128 (L = 16 384), one block per stage, fused path vs the
    CPU oracle (not vs forward_compose)."""
    torch.manual_seed(4)
    net = getattr(archs, cls)(num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).eval()
    x = torch.rand(batch, 3, size, size, generator=torch.Generator().manual_seed(7))
    if dtype == torch.float32:
        ref = _oracle(net, x, kind)
        with torch.no_grad():
            y = net.cuda()(x.cuda())
        torch.testing.assert_close(y.cpu(), ref, rtol=1e-3, atol=1e-4)
    else:
        from vmambair_b200.engine import InferenceEngine
        ref = _oracle(net, x.to(dtype), kind)
        emu = _oracle_bf16_storage(net, x.to(dtype), kind)
        eng = InferenceEngine(net, batch, size, size, dtype=dtype, use_graph=False)
        _bf16_bound(eng.run(x.to(dtype)).clone(), ref, emu)


# ----------------------------------------------------------------------------- scan vs the reference CUDA kernel
def _ref_inputs(b, dim, L, itype, G=4, N=16):
    """distributions and seed of the reference test (test_selective_scan.py:406-441)"""
    torch.random.manual_seed(0)
    dev = "cuda"
    A = -0.5 * torch.rand(dim, N, device=dev)
    Bm = torch.randn(b, G, N, L, device=dev, dtype=itype)
    Cm = torch.randn(b, G, N, L, device=dev, dtype=itype)
    D = torch.randn(dim, device=dev)
    bias = 0.5 * torch.rand(dim, device=dev)
    u = torch.randn(b, dim, L, device=dev, dtype=itype)
    delta = 0.5 * torch.rand(b, dim, L, device=dev, dtype=itype)
    return u, delta, A, Bm, Cm, D, bias


def _ref_tol(itype):
    rtol, atol = (6e-4, 2e-3) if itype == torch.float32 else (3e-3, 5e-3)
    if itype == torch.bfloat16:
        rtol, atol = 3e-2, 5e-2
    return rtol, atol, 1e-3, 1e-3


@pytest.mark.parametrize("b", [8, 4, 1])
@pytest.mark.parametrize("itype", [torch.float32, torch.bfloat16])
def test_scan_fwd_bwd_vs_reference_cuda_kernel(b, itype):
    """u (b, 4*96, 4096): the north-star shape at the bench (8), training (4) and single-image (1) batch, against
    selective_scan_cuda_core.fwd / .bwd of the reference itself on the same tensors (stored outputs, see
    oracle/ref_kernel_golden.py: the large outputs at 4096 seeded points, dA / dD / ddelta_bias whole)."""
    import vmambair_b200.selective_scan_cuda_core as ours
    rk = ref_kernel_golden
    golden = rk.load()
    args, dout = rk.inputs(b, itype)
    args = [t.cuda() for t in args]
    rtol, atol, rtolw, atolw = _ref_tol(itype)
    out_o, x_o = ours.fwd(*args, True, 1)
    go = ours.bwd(*args, dout.cuda(), x_o, True, 1)
    # (rtol, atol) per output as in the reference test :490-502; the fp32 accumulators dA/dD/dbias sum b*L = 4k..32k terms in a
    # different order in the two kernels (both use float atomics), so their bound scales with the magnitude of the result
    tols = [(rtol, atol), (rtol * 2, atol * 2), (rtol * 5, atol * 10), (rtolw, atolw * 5), (rtol, atol), (rtol, atol), (rtolw, atolw),
            (rtolw, atolw)]
    u, delta, A, Bm, Cm, D, bias = args
    layout = (u, u, delta, A, Bm, Cm, D, bias)  # out, du, ddelta, dA, dB, dC, dD, ddelta_bias: the reference's output shapes
    assert len(go) == 7
    for n, t, like, (rt, at) in zip(rk.NAMES, (out_o,) + tuple(go), layout, tols):
        assert t.shape == like.shape, (n, tuple(t.shape), tuple(like.shape))
        a, r = rk.sample(n, t), golden[f"{rk.tag(b, itype)}/{n}"].float()
        if n in rk.WHOLE:
            at = at + 1e-3 * float(r.abs().max())
        bad = (a - r).abs() > at + rt * r.abs()
        assert not bad.any(), f"{n}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float((a - r).abs().max()):.3e}, max |ref| {float(r.abs().max()):.3e}"


def test_b0_boundary_values_match_oracle():
    """selective_scan_cuda_core.fwd/.bwd shim: values, not only shapes, against the sequential oracle."""
    import vmambair_b200.selective_scan_cuda_core as core
    torch.manual_seed(0)
    u = torch.randn(2, 8, 70); dl = torch.rand(2, 8, 70)
    A = -torch.rand(8, 16); Bm = torch.randn(2, 2, 16, 70); Cm = torch.randn(2, 2, 16, 70)
    D = torch.randn(8); bias = torch.rand(8); dout = torch.randn(2, 8, 70)
    cu = [t.cuda() for t in (u, dl, A, Bm, Cm, D, bias)]
    out, x = core.fwd(*cu, True, 1)
    ref = cscan.scan_fwd(u, dl, A, Bm, Cm, D, bias, True, fp64=True)
    torch.testing.assert_close(out.double().cpu(), ref, rtol=1e-3, atol=1e-5)
    grads = core.bwd(*cu, dout.cuda(), x, True, 1)
    refg = cscan.scan_bwd(u, dl, A, Bm, Cm, D, bias, dout, True)
    assert len(grads) == 7
    for n, a, r in zip(("du", "ddelta", "dA", "dB", "dC", "dD", "dbias"), grads, refg):
        torch.testing.assert_close(a.double().cpu(), r, rtol=2e-3, atol=2e-4, msg=lambda m, n=n: f"{n}: {m}")


@pytest.mark.parametrize("itype", [torch.float32, torch.bfloat16])
def test_bwd_north_star_shape_vs_oracle(itype):
    """backward at (1, 384, 4096) -- reference-test distribution, element-wise bound (reference test :490-502 pattern:
    rtol/atol scaled per output) against the analytic fp64 oracle."""
    from vmambair_b200 import ops
    args = [t.cpu() for t in _ref_inputs(1, 384, 4096, itype)]
    dout = torch.randn(1, 384, 4096, generator=torch.Generator().manual_seed(3)).to(itype)
    cu = [t.cuda() for t in args]
    out, ck = ops.selective_scan_fwd(*cu, True, True)
    grads = ops.selective_scan_bwd(*cu, dout.cuda(), ck, True)
    refg = cscan.scan_bwd(*args, dout, True)
    rtol, atol, rtolw, atolw = _ref_tol(itype)
    tols = [(rtol * 2, atol * 2), (rtol * 5, atol * 10), (rtolw, atolw * 5), (rtol, atol), (rtol, atol), (rtolw, atolw), (rtolw, atolw)]
    for n, a, r, (rt, at) in zip(("du", "ddelta", "dA", "dB", "dC", "dD", "dbias"), grads, refg, tols):
        a, r = a.double().cpu(), r.double()
        if n in ("dA", "dD", "dbias"):
            at = at + 1e-3 * float(r.abs().max())
        bad = (a - r).abs() > at + rt * r.abs()
        assert not bad.any(), f"{n}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float((a - r).abs().max()):.3e}"
