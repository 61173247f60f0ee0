"""float64 references of the two dense GEMM kernels -- vmb_pixlin (1x1 convolution with its LayerNorm / gate prologue and bias /
SiLU range / residual epilogue) and vmb_conv3x3 (3x3 convolution with its store permutations) -- each with the rounding magnitude
its error is bounded by.

Each reference computes in float64 with torch on the device of its inputs (the bench-geometry cases run on the GPU: a 3 GFLOP
float64 contraction is slow on a host with a small CPU quota, and DGEMM's own error is ~1e8 times below the bounds) and returns
the exact value of the operation on the kernel's inputs together with S, the same expression evaluated over absolute values.
An output element is then bounded on its own (bound()):

    |got - ref| <= u_out * |ref|  +  16 * eps_fp32 * S  +  T  +  TINY

u_out * |ref| is the final rounding to the output dtype; 16 * eps_fp32 * S covers the fp32 accumulation (a sum of n terms of
random sign errs by ~0.2 eps * S), the fp32 LayerNorm statistics and the approximate exp / reciprocal of the SiLU; it stays about
1e-4 below any O(1) mistake (a dropped K row, a wrong statistic, a missing bias, a wrong tap or store index).

T is the prologue's rounding straddle (pixlin only).  With a LayerNorm or gate prologue and 16-bit inputs the kernel rounds its
*fp32* x' to bf16 / fp16 before the contraction, the reference rounds the *float64* x'.  Both round to the same value unless x'
lies within the fp32 error e of x' of a rounding midpoint; there the two can differ by one ulp of the input dtype, so

    T[m, p] = sum_k |w[m, k]| * ulp_in(x'[k, p]) * [dist(x'[k, p], nearest midpoint) <= e[k, p]]

with e = 16 eps_fp32 times the magnitude of the fp32 computation of x' (for LayerNorm that magnitude carries the (1 + rho)
conditioning factor of the variance, rho = sum_k (|x| + |mu|)^2 / sum_k (x - mu)^2).  T is zero for all but a few elements, so it
does not loosen the bound where a dropped K row would show.
"""
import torch
import torch.nn.functional as F

EPS32 = 2.0 ** -23
K_EPS = 16
U_OUT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY = {torch.float32: 0.0, torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}  # half the fp16 subnormal spacing
LN_EPS = 1e-5

CONV_PLAIN, CONV_UNSHUFFLE2, CONV_SHUFFLE2, CONV_ADD_NEAREST = 0, 1, 2, 3


def bound(ref, S, out_dtype, T=None):
    """the element-wise bound of the module docstring"""
    b = U_OUT[out_dtype] * ref.abs() + K_EPS * EPS32 * S + TINY[out_dtype]
    return b if T is None else b + T


def _neighbour(r, x, dtype):
    """the dtype value next to r (x rounded to dtype, float64) on x's side, as float64"""
    bits = r.to(dtype).view(torch.int16)
    up = (x.abs() >= r.abs()).to(torch.int16)  # away from zero when |x| >= |r| (sign-magnitude: +1 grows the magnitude)
    return (bits + 2 * up - 1).view(dtype).double()


def straddle(xp, e, dtype):
    """(ulp, mask): the spacing of dtype at xp (float64) towards xp's nearest rounding midpoint, and whether that midpoint lies
    within e of xp (the fp32 and float64 roundings of xp may then differ by that ulp)"""
    r = xp.to(dtype).double()
    nb = _neighbour(r, xp, dtype)
    ulp = (nb - r).abs()
    return ulp, (xp - 0.5 * (r + nb)).abs() <= e


def _ln64(x, mode, lw, lb):
    """LayerNorm over K of x (B, K, P) -> (x', magnitude of its fp32 evaluation)"""
    mu = x.mean(1, keepdim=True)
    d = x - mu
    rstd = (d.square().mean(1, keepdim=True) + LN_EPS).rsqrt()
    rho = (x.abs() + mu.abs()).square().sum(1, keepdim=True) / d.square().sum(1, keepdim=True).clamp_min(1e-300)
    lw = lw.view(1, -1, 1)
    if mode == 1:
        lb = lb.view(1, -1, 1)
        return d * rstd * lw + lb, (x.abs() + mu.abs()) * rstd * lw.abs() * (1 + rho) + lb.abs()
    return x * rstd * lw, x.abs() * rstd * lw.abs() * (1 + rho)


def pixlin_ref(x, w, bias=None, residual=None, ln=None, gate=None, gate_mode=0, act=(0, 0), in_dtype=torch.float32):
    """out[b, m, p] = epi(sum_k w[m, k] pro(x)[b, k, p]) in the kernel's order of operations -> (ref, S, T).

    x (B, K, P), w (M, K), bias (M), residual (B, M, P), gate (B, K): float64, holding the kernel's (dtype-rounded) inputs.
    ln = (mode, ln_w, ln_b): mode 1 WithBias, 2 BiasFree (x / sqrt(var + 1e-5), the variance about the mean).
    gate_mode 1: x (1 + g), 2: x + g, applied after the LayerNorm.  act = [act_from, act_to): SiLU on those output channels.
    in_dtype: bf16 / fp16 round the prologue output to it before the contraction (T is their straddle term); fp32 does not."""
    xp, mag = x, x.abs()
    if ln is not None and ln[0]:
        xp, mag = _ln64(x, ln[0], ln[1], ln[2])
    if gate is not None and gate_mode:
        g = gate.unsqueeze(-1)
        xp, mag = (xp * (1 + g), mag * (1 + g.abs())) if gate_mode == 1 else (xp + g, mag + g.abs())
    pro = xp is not x
    wa = w.abs()
    T = torch.zeros((), dtype=torch.float64, device=x.device)
    if pro and in_dtype != torch.float32:
        ulp, near = straddle(xp, K_EPS * EPS32 * mag, in_dtype)
        T = torch.einsum("mk,bkp->bmp", wa, ulp * near)
        xp = xp.to(in_dtype).double()
        mag = xp.abs()  # the rounded x' is exact: only the contraction's accumulation remains
    y = torch.einsum("mk,bkp->bmp", w, xp)
    S = torch.einsum("mk,bkp->bmp", wa, mag)
    if bias is not None:
        y, S = y + bias.view(1, -1, 1), S + bias.abs().view(1, -1, 1)
    a0, a1 = max(act[0], 0), min(act[1], w.shape[0])
    if a0 < a1:
        t = y[:, a0:a1]
        y = torch.cat([y[:, :a0], t * torch.sigmoid(t), y[:, a1:]], 1)
        # |silu'| <= 1.1: an error d of t becomes <= 1.1 d; the kernel's ex2.approx / rcp.approx add a few eps of |t|
        S = torch.cat([S[:, :a0], 1.1 * S[:, a0:a1] + t.abs(), S[:, a1:]], 1)
        if T.dim():
            T = torch.cat([T[:, :a0], 1.1 * T[:, a0:a1], T[:, a1:]], 1)
    if residual is not None:
        y, S = y + residual, S + residual.abs()
    return y, S, T


def conv_store(v, mode, add=None, add_scale=1):
    """the store permutation of vmb_conv3x3 on a (B, Cout, H, W) conv result (+ bias)"""
    if mode == CONV_UNSHUFFLE2:
        return F.pixel_unshuffle(v, 2)      # out[b, 4m + 2 (y % 2) + x % 2, y / 2, x / 2]
    if mode == CONV_SHUFFLE2:
        return F.pixel_shuffle(v, 2)        # out[b, m / 4, 2y + (m / 2) % 2, 2x + m % 2]
    if mode == CONV_ADD_NEAREST:
        return v + add.repeat_interleave(add_scale, 2).repeat_interleave(add_scale, 3)
    return v


def conv3x3_ref(x, w, bias=None, mode=CONV_PLAIN, add=None, add_scale=1):
    """3x3 convolution (stride 1, zero padding 1) of x (B, Cin, H, W) with w (Cout, Cin, 3, 3), + bias, then the store of `mode`
    (add: (B, Cout, H / s, W / s), mode CONV_ADD_NEAREST) -> (ref, S); all float64"""
    y = F.conv2d(x, w, bias, padding=1)
    S = F.conv2d(x.abs(), w.abs(), None if bias is None else bias.abs(), padding=1)
    if mode == CONV_ADD_NEAREST:
        return conv_store(y, mode, add, add_scale), conv_store(S, mode, add.abs(), add_scale)
    return conv_store(y, mode), conv_store(S, mode)
