"""Element-wise error bound of the selective-scan kernels against the float64 oracle (oracle/cscan.py, oracle/csrc/scan_ref.c).

scan_fwd_mag / scan_bwd_mag return, beside each float64 result, its magnitude S: the same recurrences with every product replaced
by the product of absolute values and every sum by the sum of absolute terms, plus the terms through which a rounding error of an
earlier quantity reaches this one (the `E` value-plus-magnitude idea of oracle/channel_ref.py).  An element is then bounded on its
own:

    |got - ref| <= u_out * |ref|  +  K * eps_fp32 * S  +  TINY

u_out * |ref| is the final rounding to the output dtype (fp32 for dA, dD and ddelta_bias whatever the input dtype).

Why K = 16.  Each fp32 operation of the kernel rounds with a relative error of at most u = eps_fp32 / 2; S counts every term once,
so K * eps_fp32 * S = 2K u S allows each term 2K = 32 roundings.  That covers:
  * the state update h = a h + b: one product and one sum per position, plus exp(x) evaluated as ex2(x log2 e) with MUFU.EX2
    (~2 ulp) on an exponent that itself carries the roundings of dt * A * log2e -- hence the (1 + r |x|) a Mh term of S;
  * dt = softplus(delta + bias), evaluated as max(x, 0) + log1p(exp(-|x|)): its relative error grows with |x| (the r = 1 + |x|
    multiplier of the oracle) and enters every b = dt u B and every exponent;
  * the chunked parallel scans (carry * prod a + local state, up to 32 lanes and the checkpoint segments): a carry propagated over
    k positions picks up k roundings of the product, and S grows by one a Mh per position, i.e. by k copies of the carried
    magnitude;
  * the sums over the state (y, du, ddelta), over positions and rows (dA, dB, dC, dD, dbias) in any order: a sum of n terms of
    random sign errs by about sqrt(n) u max|term|, far below u * sum|term|;
  * ddelta's softplus derivative, formed as 1 - exp(-dt): an absolute (not relative) error of a few u, which the oracle adds as
    (2 + r dt) * sum Mdh Mv.
On the CPU the sequential fp32 evaluations (scan_ref_fwd_f32, scan_ref_bwd_f32) use at most ~0.05 of the bound
(tests/test_scan_ref_cpu.py); the kernels' approximate ex2 / lg2 / rcp and their reassociation take a few times more.  K stays
~1e-4 relative below any O(1) fault: a dropped carry, a neighbour's dt, the wrong group's B / C, a missing tail term.

fp32 atomics.  dA, dD and ddelta_bias receive one fp32 atomic addition per contributing CTA or warp, dB and dC (through the fp32
scratch) one per contributing warp or CTA of the group; the deterministic kernels instead add the same partial sums in a fixed
order.  Each of those P additions rounds its running sum, whose magnitude is at most the sum of the absolute terms, itself <= S.
atomic(S, P) adds that P * u * S = P / (2K) * K eps_fp32 S to the element's magnitude.
"""
import torch

EPS32 = 2.0 ** -23
K_EPS = 16
U_OUT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY = {torch.float32: 0.0, torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}  # half the fp16 subnormal spacing


def bound(ref, S, out_dtype):
    """the element-wise bound of the module docstring"""
    return U_OUT[out_dtype] * ref.abs() + K_EPS * EPS32 * S + TINY[out_dtype]


def atomic(S, P):
    """S of a sum that reaches memory as P fp32 additions of partial sums (module docstring)"""
    return S * (1.0 + P / (2.0 * K_EPS))
