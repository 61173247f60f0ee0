"""The float64 references of vmb_pixlin / vmb_conv3x3 (oracle/gemm_ref.py) and their element-wise bound, checked on the CPU against an
fp32 emulation of each kernel: the bound must hold for the emulation (sound) and break for each deliberately wrong emulation (sharp),
and the prologue's rounding-straddle term must switch on exactly at a rounding midpoint."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_ref as G

DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def violations(got, ref, S, dtype, T=None):
    """number of elements of got outside the bound of ref"""
    return int((~((got.double() - ref).abs() <= G.bound(ref, S, dtype, T))).sum())


# ----------------------------------------------------------------------------- pixlin
def emulate_pixlin(x, w, bias, residual, ln, gate, gate_mode, act, dtype, fault=None):
    """fp32 emulation of pixlin_mma_kernel / pixlin_f32_kernel: dtype operands, the fp32 LayerNorm / gate prologue rounded to dtype,
    fp32 accumulation in blocks of 16 along K, the fp32 epilogue and one rounding to dtype.  fault: one deliberate mistake."""
    xf, K = x.float(), x.shape[1]
    if ln is not None:
        mode, lw, lb = ln
        mu = xf.mean(1, keepdim=True)
        var = (xf - mu).square().sum(1, keepdim=True) / (K - 1 if fault == "var_k_minus_1" else K)
        rstd = torch.rsqrt(var + 1e-5)
        lw = lw.float().view(1, -1, 1)
        xf = (xf - mu) * rstd * lw + lb.float().view(1, -1, 1) if mode == 1 else xf * rstd * lw
    if gate is not None:
        g = gate.float().unsqueeze(-1)
        xf = xf * g + xf if gate_mode == 1 else xf + g
    if (ln is not None or gate is not None) and dtype != torch.float32:
        xf = xf.to(dtype).float()
    wf = w.float()
    kend = K - 1 if fault == "drop_last_k" else K
    acc = torch.zeros(x.shape[0], w.shape[0], x.shape[2])
    for k0 in range(0, kend, 16):
        k1 = min(k0 + 16, kend)
        acc += torch.einsum("mk,bkp->bmp", wf[:, k0:k1], xf[:, k0:k1])
    if bias is not None:
        b = bias.float().clone()
        if fault == "bias_missing":
            b[w.shape[0] // 2] = 0
        acc += b.view(1, -1, 1)
    a0, a1 = act
    if a0 < a1:
        acc[:, a0:a1] = F.silu(acc[:, a0:a1])
    if residual is not None:
        if fault == "residual_after_rounding":
            return (acc.to(dtype).float() + residual.float()).to(dtype)
        acc += residual.float()
    return acc.to(dtype)


def pixlin_case(dtype, B, K, M, P, pro, seed, act=True):
    """random operands of one pixlin call (dtype) and their float64 copies; pro: None / ("ln", mode) / ("gate", mode)"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale)
    x = (r(B, K, P) + (r(B, 1, P) if pro and pro[0] == "ln" else 0)).to(dtype)
    w = r(M, K, scale=K ** -0.5).to(dtype)
    bias, residual = r(M, scale=0.5), r(B, M, P).to(dtype)
    ln = gate = None
    gate_mode = 0
    if pro and pro[0] == "ln":
        ln = (pro[1], 1 + 0.5 * r(K), 0.5 * r(K) if pro[1] == 1 else None)
    elif pro and pro[0] == "gate":
        gate, gate_mode = r(B, K), pro[1]
    acts = (M // 3, M - M // 3) if act else (0, 0)
    args = dict(x=x, w=w, bias=bias, residual=residual, ln=ln, gate=gate, gate_mode=gate_mode, act=acts)
    d = lambda t: None if t is None else t.double()
    ref = G.pixlin_ref(d(x), d(w), d(bias), d(residual), None if ln is None else (ln[0], d(ln[1]), d(ln[2])), d(gate), gate_mode,
                       acts, dtype)
    return args, ref


PIX_SHAPES = [(2, 20, 24, 40), (1, 48, 96, 64), (2, 144, 40, 32), (1, 384, 70, 24), (1, 5, 16, 8)]  # (B, K, M, P)
PROLOGUES = [None, ("ln", 1), ("ln", 2), ("gate", 1), ("gate", 2)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pro", PROLOGUES)
@pytest.mark.parametrize("B,K,M,P", PIX_SHAPES)
def test_pixlin_bound_holds_for_the_kernel_emulation(dtype, pro, B, K, M, P):
    args, (ref, S, T) = pixlin_case(dtype, B, K, M, P, pro, seed=B * 1000 + K + M + P)
    got = emulate_pixlin(**args, dtype=dtype)
    assert violations(got, ref, S, dtype, T) == 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fault,pro", [("drop_last_k", None), ("drop_last_k", ("gate", 1)), ("var_k_minus_1", ("ln", 1)),
                                       ("var_k_minus_1", ("ln", 2)), ("bias_missing", None), ("residual_after_rounding", None)])
def test_pixlin_bound_catches_a_wrong_emulation(dtype, fault, pro):
    B, K, M, P = 2, 48, 40, 64
    args, (ref, S, T) = pixlin_case(dtype, B, K, M, P, pro, seed=7, act=fault != "residual_after_rounding")
    assert violations(emulate_pixlin(**args, dtype=dtype), ref, S, dtype, T) == 0
    if fault == "residual_after_rounding" and dtype == torch.float32:
        pytest.skip("fp32 output: rounding before the residual is the fp32 rounding the bound allows")
    assert violations(emulate_pixlin(**args, dtype=dtype, fault=fault), ref, S, dtype, T) > 0


def test_straddle_term_is_nonzero_only_near_a_midpoint():
    """x' = x + g (gate mode 2) computed exactly: at a bf16 rounding midpoint T = |w| ulp; on a bf16 value (half an ulp from either
    midpoint) and at a few straddle widths from the midpoint T = 0; just inside the straddle width T = |w| ulp again"""
    ulp = 2.0 ** -7  # bf16 spacing in [1, 2)
    x = torch.ones(1, 1, 5, dtype=torch.float64)
    e = G.K_EPS * G.EPS32 * 1.5  # the straddle width at |x| + |g| ~ 1.5: the prologue's fp32 error
    g = torch.tensor([[ulp / 2]], dtype=torch.float64)
    offs = torch.tensor([0.0, ulp / 2, 4 * e, -4 * e, e / 2], dtype=torch.float64)
    w = torch.tensor([[0.75]], dtype=torch.float64)
    T = torch.stack([G.pixlin_ref(x[..., i:i + 1] + o, w, gate=g, gate_mode=2, in_dtype=torch.bfloat16)[2].flatten()
                     for i, o in enumerate(offs)]).flatten()
    assert T.tolist() == [0.75 * ulp, 0.0, 0.0, 0.0, 0.75 * ulp]
    # the 16-bit rounding of the reference itself: the midpoint 1 + ulp / 2 rounds to even (1.0)
    ref = G.pixlin_ref(x[..., :1], w, gate=g, gate_mode=2, in_dtype=torch.bfloat16)[0]
    assert float(ref) == 0.75


def test_straddle_midpoints_on_both_signs_and_across_a_binade():
    """the neighbour of a rounded value is taken on x's side, with the spacing of that side (halved below a power of two)"""
    xs = torch.tensor([1 + 2.0 ** -8, -(1 + 2.0 ** -8), 1 - 2.0 ** -9, 1 - 2.0 ** -10, -(1 + 2.0 ** -7)], dtype=torch.float64)
    ulp, near = G.straddle(xs, torch.full_like(xs, 1e-12), torch.bfloat16)
    assert ulp.tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -8, 2.0 ** -7]
    assert near.tolist() == [True, True, True, False, False]


# ----------------------------------------------------------------------------- conv3x3
def emulate_conv3x3(x, w, bias, mode, add, add_scale, dtype, fault=None):
    """fp32 emulation of the conv3x3 kernels: dtype operands, fp32 accumulation, bias, the store of `mode`, one rounding"""
    xf, wf = x.float(), w.float()
    y = F.conv2d(xf, wf, bias.float(), padding=1)
    if fault == "tap_shifted":  # the top-left tap reads the pixel one to the right of its own
        w0 = torch.zeros_like(wf)
        w0[..., 0, 0] = wf[..., 0, 0]
        y = y - F.conv2d(xf, w0, padding=1) + F.conv2d(torch.roll(xf, -1, 3), w0, padding=1)
    if fault == "shuffle_bits_swapped":  # channel m = 4c + 2i + j stored as if it were 4c + 2j + i
        C = y.shape[1]
        m = torch.arange(C)
        y = y[:, (m & ~3) | ((m & 1) << 1) | ((m >> 1) & 1)]
    out = G.conv_store(y, mode, None if add is None else add.float(), add_scale)
    return out.to(dtype)


def conv_case(dtype, B, Cin, Cout, H, W, mode, seed, add_scale=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, W, generator=g).to(dtype)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (9 * Cin) ** -0.5).to(dtype)
    bias = torch.randn(Cout, generator=g) * 0.5
    add = torch.randn(B, Cout, H // add_scale, W // add_scale, generator=g).to(dtype) if mode == G.CONV_ADD_NEAREST else None
    ref = G.conv3x3_ref(x.double(), w.double(), bias.double(), mode, None if add is None else add.double(), add_scale)
    return (x, w, bias, mode, add, add_scale), ref


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode,add_scale", [(0, 1), (1, 1), (2, 1), (3, 1), (3, 2), (3, 4)])
@pytest.mark.parametrize("Cin,Cout", [(3, 16), (20, 48)])
def test_conv3x3_bound_holds_for_the_kernel_emulation(dtype, mode, add_scale, Cin, Cout):
    args, (ref, S) = conv_case(dtype, 2, Cin, Cout, 8, 12 if add_scale != 4 else 16, mode, seed=Cin + Cout + mode, add_scale=add_scale)
    assert violations(emulate_conv3x3(*args, dtype=dtype), ref, S, dtype) == 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fault,mode", [("tap_shifted", G.CONV_PLAIN), ("tap_shifted", G.CONV_UNSHUFFLE2),
                                        ("shuffle_bits_swapped", G.CONV_SHUFFLE2)])
def test_conv3x3_bound_catches_a_wrong_emulation(dtype, fault, mode):
    args, (ref, S) = conv_case(dtype, 2, 20, 48, 8, 12, mode, seed=3)
    assert violations(emulate_conv3x3(*args, dtype=dtype), ref, S, dtype) == 0
    assert violations(emulate_conv3x3(*args, dtype=dtype, fault=fault), ref, S, dtype) > 0
