"""The selective-scan oracle's magnitudes (oracle/cscan.py scan_fwd_mag / scan_bwd_mag) and the element-wise bound built on them
(oracle/scan_bound.py), checked on the CPU:
  * the values the magnitude functions return are the float64 oracle's, bit for bit;
  * the sequential fp32 evaluations of the forward and of the analytic backward lie inside the bound at every element (sound);
  * each planted fault -- the kind of mistake a chunked, direction-aware scan kernel makes -- applied to the float64 result falls
    outside it (sharp)."""
import pytest
import torch

from oracle import cscan
from oracle import scan_bound as SB
from tests.test_scan_gpu import make_inputs

F32 = torch.float32
GRADS = ("du", "ddelta", "dA", "dB", "dC", "dD", "dbias")


def worst(got, ref, S, dtype=F32):
    """largest err / bound over the elements"""
    return float(((got.double() - ref).abs() / SB.bound(ref, S, dtype).clamp_min(1e-300)).max())


def outside(got, ref, S, dtype=F32):
    return int((~((got.double() - ref).abs() <= SB.bound(ref, S, dtype))).sum())


CASES = [  # b, D, L, N, G, model_like
    (2, 8, 4096, 16, 1, False),
    (2, 8, 4096, 16, 4, True),
    (1, 6, 4096, 40, 3, True),
    (2, 6, 1000, 40, 2, False),
    (2, 4, 777, 1, 2, False),
    (1, 4, 4096, 1, 1, True),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "b{}-D{}-L{}-N{}-G{}-{}".format(*c[:5], "model" if c[5] else "ref"))
def test_fp32_evaluation_inside_bound(case):
    b, D, L, N, G, model_like = case
    sp = True if model_like else bool(L % 2)  # the model-like dt needs the softplus; the reference distribution runs both ways
    ins = make_inputs(b, D, L, N, G, F32, seed=3, model_like=model_like)
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(4))
    ref, S = cscan.scan_fwd_mag(*ins, sp)
    assert worst(cscan.scan_fwd(*ins, sp), ref, S) < 0.25
    g, s = cscan.scan_bwd_mag(*ins, dout, sp)
    g32 = cscan.scan_bwd_f32(*ins, dout, sp)
    for name, x, y, z in zip(GRADS, g32, g, s):
        assert worst(x, y, z) < 0.25, name


@pytest.mark.parametrize("sp", [False, True])
def test_magnitude_values_are_the_float64_oracle(sp):
    """one OpenMP thread: the dA / dD / dbias partials of several threads are summed in arrival order"""
    ins = make_inputs(2, 6, 1000, 16, 3, F32, seed=5)
    dout = torch.randn(2, 6, 1000, generator=torch.Generator().manual_seed(6))
    cscan.set_threads(1)
    try:
        ref, _ = cscan.scan_fwd_mag(*ins, sp)
        assert torch.equal(ref, cscan.scan_fwd(*ins, sp, fp64=True))
        g, _ = cscan.scan_bwd_mag(*ins, dout, sp)
        for name, x, y in zip(GRADS, g, cscan.scan_bwd(*ins, dout, sp)):
            assert torch.equal(x, y), name
    finally:
        cscan.use_host_threads()


# ----------------------------------------------------------------------------- planted faults (sharpness)
FAULT_CASES = [(2, 8, 4096, 16, 4, False), (2, 8, 4096, 16, 4, True)]


def _shift(t, k=1):
    """t with positions l -> l - k along the last axis (the first k repeat position 0): a walk off by one position"""
    return torch.cat([t[..., :1].expand(*t.shape[:-1], k), t[..., :-k]], -1)


@pytest.fixture(scope="module", params=FAULT_CASES, ids=["ref", "model"])
def fault_case(request):
    b, D, L, N, G, model_like = request.param
    ins = make_inputs(b, D, L, N, G, F32, seed=7, model_like=model_like)
    dout = torch.randn(b, D, L, generator=torch.Generator().manual_seed(8))
    sp = True
    return ins, dout, sp, cscan.scan_fwd_mag(*ins, sp), cscan.scan_bwd_mag(*ins, dout, sp)


def test_fault_reversed_walk_off_by_one(fault_case):
    ins, dout, sp, (ref, S), (g, s) = fault_case
    u, delta, A, B, C, Dv, bias = ins
    assert outside(cscan.scan_fwd(_shift(u), _shift(delta), A, _shift(B), _shift(C), Dv, bias, sp, fp64=True), ref, S) > 0
    bad = cscan.scan_bwd(_shift(u), _shift(delta), A, _shift(B), _shift(C), Dv, bias, _shift(dout), sp)
    assert outside(bad[0], g[0], s[0]) > 0 and outside(bad[3], g[3], s[3]) > 0


@pytest.mark.parametrize("cut", [64, 256, 512 + 64])
def test_fault_dropped_carry(fault_case, cut):
    """the state is not carried across one checkpoint / chunk boundary: the positions after it restart from zero"""
    ins, dout, sp, (ref, S), (g, s) = fault_case
    u, delta, A, B, C, Dv, bias = ins
    tail = cscan.scan_fwd(u[..., cut:], delta[..., cut:], A, B[..., cut:], C[..., cut:], Dv, bias, sp, fp64=True)
    assert outside(tail, ref[..., cut:], S[..., cut:]) > 0
    # backward: the adjoint is not carried back across the boundary
    head = cscan.scan_bwd(u[..., :cut], delta[..., :cut], A, B[..., :cut], C[..., :cut], Dv, bias, dout[..., :cut], sp)
    assert outside(head[0], g[0][..., :cut], s[0][..., :cut]) > 0


def test_fault_neighbouring_dt(fault_case):
    ins, dout, sp, (ref, S), (g, s) = fault_case
    u, delta, A, B, C, Dv, bias = ins
    l = 1000
    d2 = delta.clone()
    d2[..., l] = delta[..., l + 1]
    assert outside(cscan.scan_fwd(u, d2, A, B, C, Dv, bias, sp, fp64=True), ref, S) > 0
    bad = cscan.scan_bwd(u, d2, A, B, C, Dv, bias, dout, sp)
    assert outside(bad[1][..., l], g[1][..., l], s[1][..., l]) > 0  # ddelta at that position


def test_fault_wrong_group_bc(fault_case):
    ins, dout, sp, (ref, S), (g, s) = fault_case
    u, delta, A, B, C, Dv, bias = ins
    perm = [1, 0] + list(range(2, B.shape[1]))  # groups 0 and 1 read each other's B / C
    assert outside(cscan.scan_fwd(u, delta, A, B[:, perm], C[:, perm], Dv, bias, sp, fp64=True), ref, S) > 0
    assert outside(cscan.scan_fwd(u, delta, A, B[:, perm], C, Dv, bias, sp, fp64=True), ref, S) > 0
    assert outside(cscan.scan_fwd(u, delta, A, B, C[:, perm], Dv, bias, sp, fp64=True), ref, S) > 0


def test_fault_last_ragged_dB_term_missing(fault_case):
    """one row's dh dt u missing from dB at the last position: u of that row zeroed there changes nothing else of dB[..., -1]"""
    ins, dout, sp, (ref, S), (g, s) = fault_case
    u, delta, A, B, C, Dv, bias = ins
    u2 = u.clone()
    u2[:, 0, -1] = 0
    bad = cscan.scan_bwd(u2, delta, A, B, C, Dv, bias, dout, sp)
    assert outside(bad[3][..., -1], g[3][..., -1], s[3][..., -1]) > 0


def test_fault_one_dD_halved(fault_case):
    ins, dout, sp, (ref, S), (g, s) = fault_case
    for d in range(g[5].shape[0]):
        bad = g[5].clone()
        bad[d] *= 0.5
        assert outside(bad, g[5], SB.atomic(s[5], 64)) == 1, d


def test_atomic_term():
    S = torch.tensor([1.0])
    assert float(SB.atomic(S, 0)) == 1.0 and float(SB.atomic(S, 2 * SB.K_EPS)) == 2.0
