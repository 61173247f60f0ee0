"""The channel-direction OSS kernels against the float64 reference of oracle/channel_ref.py, on every path the launchers pick:
- forward: channel_branch_v2_kernel (default) and channel_branch_kernel (v1: taken when v2's shared memory does not fit), each
  through ops.channel_branch;
- backward: channel_branch_bwd_kernel through ops.channel_branch_bwd, where ops.channel_branch_bwd_supported says it fits;
- end to end: fused_train.channel_gate, which runs the two kernels (the _Channel Function) where the backward fits and torch autograd
  over SS2D_1.cforward_pooled (the flat scan) above that.

Widths: the bench net's levels (48, 96, 192, 384), both sides of every shared-memory limit below, loop tails (C % 4 != 0,
C % 8 != 0, C < 32), realsr with fewer than 16 states (its state lanes are masked), and SS2D_1 at ssm_ratio 2 (C = E; realsr's
rank comes from d_model).  Batches 1, 3 and 8: one CTA per image, parameter gradients combined with atomics across CTAs.  Parameters
come from real SS2D_1 modules in both regimes of channel_ref.make_module, pooled sums are those of L = 64 or 4096 pixels.

Every element is bounded on its own: |got - ref| <= 2^-24 |ref| + K eps_fp32 S, S the magnitude the reference computes next to each
value (channel_ref.bound; tests/test_channel_ref_cpu.py shows it breaks for a dropped last position, a dropped state lane and a
bf16-rounded mean).  Every output tensor is also held to a norm-wise tolerance (NORM_TOL below): the element-wise bound alone cannot
resolve the gradients whose terms cancel.  test_bound_resolves asserts, per case and per output, that the two together reject an
all-zero result and a parameter gradient missing its largest single image's contribution.

Which path a case takes is derived from mirrors of the launchers' shared-memory formulas (fwd_v2 / bwd_kernel below), and asserted:
the backward mirror against ops.channel_branch_bwd_supported and the library's vmb_channel_branch_bwd_smem_bytes; the forward mirror
against the kernel a torch.profiler trace names.  With 227 KB of shared memory per block the mirrors give:
  forward v2:        sisr / mamber32 C <= 255, mamber33 C <= 383, realsr C <= 384   (v1 above, up to C = 593 / 665 / 451)
  backward kernel:   sisr / mamber32 C <= 245, mamber33 C <= 370, realsr C <= 377   (the torch fallback above)
(realsr at ssm_ratio 1 and N = 16, Rc = ceil(C / 16); a smaller rank or N moves its limits up.)

These tests found no kernel bug.  The largest err / element-wise bound over all cases (RATIOS, printed at the end of the module with
pytest -s), measured on an H100 80GB HBM3 at its 700 W power limit: forward v1 0.006, forward v2 0.006, backward kernel 0.06,
channel_gate on the kernels 0.06, on the torch fallback 0.046 (the backward's fp32 atomics move the last digit from run to run).
"""
import functools

import pytest
import torch

from oracle import channel_ref as cr
from tests.test_enhance_gpu import kernel_census, kernel_names
from vmambair_b200 import _lib, fused_train, ops

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

SMEM_LIMIT = 227 * 1024


# ----------------------------------------------------------------------------- mirrors of the launchers' path choices
def fwd_smem(C, dc, Rc, N, v2):
    """oss_ops.cu channel_launch: v1's shared memory, and v2's (v1's plus the h * C staging)"""
    RN, CP = Rc + 2 * N, C | 1
    base = 4 * (dc * C + 2 * RN * CP + 4 * dc * C + C + 64 + 2 * RN * dc + 2 * dc * Rc + 2 * dc + 3 * dc + 1)
    return base + 4 * 2 * dc * 16 * CP if v2 else base


def fwd_v2(C, dc, Rc, N):
    return 2 * dc * 16 <= 512 and fwd_smem(C, dc, Rc, N, True) <= SMEM_LIMIT


def bwd_smem(C, dc, Rc, N):
    """channel_bwd.cu channel_bwd_smem"""
    RN, CP, rows = Rc + 2 * N, C | 1, 2 * dc
    return 4 * (dc * C + 2 * RN * CP + 3 * rows * C + 2 * C + 64 + 2 * RN * dc + 2 * dc * Rc + 2 * dc + 3 * dc + 1 + rows * 16 * CP)


def bwd_kernel(C, dc, Rc, N):
    return N <= 16 and 2 * dc * 16 <= 512 and bwd_smem(C, dc, Rc, N) <= SMEM_LIMIT


# ----------------------------------------------------------------------------- cases
NATIVE = {"sisr": "randn", "mamber32": "randn", "mamber33": "randn", "realsr": "dtinit"}
OTHER = {"randn": "dtinit", "dtinit": "randn"}
VARIANTS = list(NATIVE)


def _cases():
    out = []  # (variant, C, ssm_ratio, d_state, regime)
    for v in VARIANTS:
        for C in (48, 96, 192, 384):  # the bench net's levels, in both regimes
            out += [(v, C, 1, 16, NATIVE[v]), (v, C, 1, 16, OTHER[NATIVE[v]])]
    for v, Cs in (("sisr", (245, 246)), ("mamber32", (255, 256)), ("mamber33", (370, 371, 383, 384)), ("realsr", (377, 378, 385))):
        out += [(v, C, 1, 16, NATIVE[v]) for C in Cs]  # both sides of a shared-memory limit
    for i, C in enumerate((5, 13, 30, 37, 251)):  # loop tails
        out += [(v, C, 1, 16, NATIVE[v] if (i + j) % 2 == 0 else OTHER[NATIVE[v]]) for j, v in enumerate(VARIANTS)]
    out += [("realsr", C, 1, N, r) for C, N, r in ((37, 8, "dtinit"), (64, 11, "randn"), (200, 8, "randn"), (251, 11, "dtinit"))]
    out += [(v, 96, 2, 16, NATIVE[v]) for v in VARIANTS]  # ssm_ratio 2: C = E = 2 d_model
    out += [("realsr", 192, 2, 16, "dtinit"), ("realsr", 40, 2, 8, "randn"), ("mamber33", 250, 2, 16, "dtinit")]
    return [(*c, (1, 3, 8)[i % 3], (64, 4096)[i % 2]) for i, c in enumerate(out)]  # + batch, pixels per image


CASES = _cases()
IDS = [f"{v}-C{C}-r{r}-N{N}-{reg}-B{B}-L{L}" for v, C, r, N, reg, B, L in CASES]


@functools.lru_cache(maxsize=None)
def reference(case):
    """module (CPU), prm (CPU fp32), pooled sums and dc_out (CPU) and the float64 reference of one case: c, dpooled, the parameter
    gradients, and for B > 1 each parameter gradient without its largest single image's contribution (a lost CTA)"""
    variant, C, ratio, N, regime, B, L = case
    a = cr.make_module(variant, C // ratio, ratio, N, regime, seed=C * 3 + B + N)
    assert a.d_inner == C and a.dc_state == N
    if variant == "realsr":
        assert a.dtc_rank == -(-(C // ratio) // 16)
    prm = cr.module_prm(a)
    g = torch.Generator().manual_seed(C + B)
    pooled = (L * (0.5 * torch.randn(B, C, generator=g) + 0.3 * torch.randn(B, 1, generator=g))).float()
    dc_out = torch.randn(B, C, generator=g)
    c, ctx = cr.forward(pooled.double(), 1.0 / L, cr.prm64(prm))
    dpooled, grads = cr.backward(ctx, dc_out.double())
    missing = {}
    if B > 1:  # the backward is linear in dc_out: image b's share of a parameter gradient is the backward of dc_out zero but row b
        shares = []
        for b in range(B):
            gb = torch.zeros(B, C, dtype=torch.float64)
            gb[b] = dc_out[b].double()
            shares.append(cr.backward(ctx, gb)[1])
        for k, ref in grads.items():
            big = max(shares, key=lambda sh: float(sh[k].v.norm()))
            missing[k] = ref.v - big[k].v
    return a, prm, pooled, dc_out, c, dpooled, grads, missing


@functools.lru_cache(maxsize=None)
def setup(case):
    """reference(case) with prm, pooled and dc_out on the GPU"""
    a, prm, pooled, dc_out, c, dpooled, grads, _ = reference(case)
    prm = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in prm.items()}
    return a, prm, pooled.cuda(), dc_out.cuda(), c, dpooled, grads


# Norm-wise criterion, per output tensor: ||got - ref||_2 <= NORM_TOL * ||ref||_2.  The element-wise bound alone cannot resolve the
# parameter gradients whose terms cancel: after the LayerNorm, sum_l dout = 0 and dout is orthogonal to the normalised output, and
# with D u dominating the scan (dt ~ 1e-3) the output is nearly affine in the pooled mean, so the gradients of Dsc, conv_cout,
# conv_cin and the dtc projection are small differences of large terms.  K eps S then keeps the cancelled mass and can exceed the
# gradient itself.  The norm-wise tolerances are set from measurement (largest ||err|| / ||ref|| over all cases, H100 80GB HBM3 at
# 700 W: Dsc 1.1e-2, conv_cout.weight 3.9e-3, conv_cin 1.1e-4, every other output <= 3e-5) with headroom, and test_bound_resolves
# asserts that each one, with the element-wise bound, still rejects an all-zero result and one image's contribution left out.
NORM_TOL = {"Dsc": 2e-2, "cout_w": 1e-2}
NORM_TOL_DEFAULT = 1e-3
# conv_cout.bias: d cout_b = sum_{b,l} dout = 0 exactly (the LayerNorm's backward sums to zero over C), so it has no relative error
# to bound; the element-wise bound holds it to rounding size around zero
STRUCTURAL_ZERO = ("cout_b",)

RATIOS = {}  # kernel -> the largest err / bound seen in this session; printed at the end of the module (pytest -s shows it)


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    print("\nlargest err / element-wise bound per kernel:", {k: round(v, 4) for k, v in sorted(RATIOS.items())})


def fails(got, ref, key, pre=None):
    """None if `got` (CPU float64) passes both criteria against the E `ref` (+ prefill `pre`), else a message"""
    val, bound = ref.v, cr.bound(ref)
    if pre is not None:
        val, bound = val + pre, bound + cr.U_OUT * pre.abs() + cr.K * cr.EPS32 * pre.abs()
    err = (got - val).abs()
    ratio = err / bound.clamp_min(1e-300)
    if not bool((ratio <= 1).all()):
        i = int(ratio.flatten().argmax())
        return (f"{int((err > bound).sum())} of {err.numel()} elements out of bound; worst at flat index {i}: "
                f"got {float(got.flatten()[i])}, ref {float(val.flatten()[i])}, bound {float(bound.flatten()[i])}")
    if key not in STRUCTURAL_ZERO:
        tol = NORM_TOL.get(key, NORM_TOL_DEFAULT)
        if not float(err.norm()) <= tol * float(ref.v.norm()):
            return f"||err|| = {float(err.norm()):.3g} > {tol} ||ref|| = {tol * float(ref.v.norm()):.3g}"
    return None


def check(got, ref, what, kernel, key=None, pre=None):
    """element-wise bound (module docstring) and, for a named output, the norm-wise criterion; pre: a prefill the result was added to"""
    got = got.detach().double().cpu().reshape(ref.v.shape)
    pre = None if pre is None else pre.double().cpu().reshape(ref.v.shape)
    val = ref.v if pre is None else ref.v + pre
    bound = cr.bound(ref) if pre is None else cr.bound(ref) + cr.U_OUT * pre.abs() + cr.K * cr.EPS32 * pre.abs()
    RATIOS[kernel] = max(RATIOS.get(kernel, 0.0), float(((got - val).abs() / bound.clamp_min(1e-300)).max()))
    msg = fails(got, ref, key, pre)
    assert msg is None, f"{what}: {msg}"


def dims(prm):
    return prm["dc"], prm["Rc"], prm["N"]


# ----------------------------------------------------------------------------- resolution
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_bound_resolves(case):
    """on the reference side, the criteria check() applies reject, for dpooled and every parameter gradient of this case: an all-zero
    result, and (B > 1) the gradient without its largest single image's contribution, as if one CTA's atomics were lost.
    conv_cout.bias is exactly zero (STRUCTURAL_ZERO) and has nothing to resolve."""
    _, _, _, _, _, dp_ref, g_ref, missing = reference(case)
    outputs = {"dpooled": dp_ref, **g_ref}
    for k, ref in outputs.items():
        if k in STRUCTURAL_ZERO:
            continue
        assert fails(torch.zeros_like(ref.v), ref, k) is not None, f"{k}: an all-zero result passes"
        if k in missing:
            assert fails(missing[k], ref, k) is not None, f"{k}: the gradient without one image's contribution passes"


# ----------------------------------------------------------------------------- forward
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_channel_branch_forward_on_mirrored_kernel(case):
    """ops.channel_branch against float64; the kernel a profiler trace names is the one the shared-memory mirror fwd_v2 predicts
    (v1 runs only where v2 does not fit)"""
    C, L = case[1], case[6]
    a, prm, pooled, _, c_ref, _, _ = setup(case)
    census, c = kernel_census(lambda: ops.channel_branch(pooled, 1.0 / L, prm, C))
    v2 = fwd_v2(C, *dims(prm))
    assert kernel_names(census) == {"channel_branch_v2_kernel" if v2 else "channel_branch_kernel": 1}, census
    check(c, c_ref, "c", "forward v2" if v2 else "forward v1", "c")


# ----------------------------------------------------------------------------- backward kernel
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_channel_branch_backward(case):
    """ops.channel_branch_bwd against float64 (dpooled and every parameter gradient) wherever the kernel is supported, fresh and
    into prefilled accumulators; everywhere: ops.channel_branch_bwd_supported == the mirror, whose smem == the library's"""
    C, L = case[1], case[6]
    a, prm, pooled, dc_out, _, dp_ref, g_ref = setup(case)
    assert bwd_smem(C, *dims(prm)) == _lib.lib().vmb_channel_branch_bwd_smem_bytes(C, *dims(prm))
    sup = ops.channel_branch_bwd_supported(C, prm)
    assert sup == bwd_kernel(C, *dims(prm))
    if not sup:
        return  # fused_train.channel_gate takes the torch fallback here: test_channel_gate_end_to_end
    assert set(g_ref) == {k for k in cr.KEYS if prm[k] is not None}
    dpooled, g = ops.channel_branch_bwd(pooled, 1.0 / L, prm, C, dc_out)
    check(dpooled, dp_ref, "dpooled", "backward", "dpooled")
    for k, ref in g_ref.items():
        check(g[k], ref, f"d {k}", "backward", k)
    if prm["cin_w"] is None:  # realsr: the kernel got null conv_cin / conv_cout gradient pointers and wrote nothing there
        assert not any(g[k].any() for k in ("cin_w", "cin_b", "cout_w", "cout_b"))
    # into=: every other accumulator prefilled and passed in; those receive prefill + gradient, the rest are returned fresh
    into_keys = list(g_ref)[::2]
    pre = {k: torch.randn(g[k].numel(), device="cuda") for k in into_keys}
    into = {k: t.clone() for k, t in pre.items()}
    dpooled2, g2 = ops.channel_branch_bwd(pooled, 1.0 / L, prm, C, dc_out, into=into)
    check(dpooled2, dp_ref, "dpooled (into=)", "backward", "dpooled")
    for k, ref in g_ref.items():
        if k in into:
            assert g2[k].data_ptr() == into[k].data_ptr()
            check(into[k], ref, f"d {k} (into=, prefilled)", "backward", k, pre=pre[k])
        else:
            check(g2[k], ref, f"d {k} (into=, fresh)", "backward", k)


# ----------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_channel_gate_end_to_end(case):
    """fused_train.channel_gate forward + backward: the _Channel Function exactly where the backward kernel fits, torch autograd
    over cforward_pooled above; c, pooled.grad and every parameter's .grad against float64"""
    C, L = case[1], case[6]
    a, prm, pooled, dc_out, c_ref, dp_ref, g_ref = setup(case)
    m = a.cuda()
    try:
        m.zero_grad(set_to_none=True)
        pp = pooled.clone().requires_grad_()
        c = fused_train.channel_gate(m, pp, L)
        fused = "_Channel" in type(c.grad_fn).__name__
        assert fused == bwd_kernel(C, *dims(prm)), type(c.grad_fn).__name__
        kernel = "channel_gate (kernels)" if fused else "channel_gate (torch fallback)"
        c.backward(dc_out)
        check(c, c_ref, "c", kernel, "c")
        check(pp.grad, dp_ref, "pooled.grad", kernel, "dpooled")
        params = dict(m.named_parameters())
        for name, k in cr.PARAM_KEYS.items():
            if k in g_ref:
                check(params[name].grad, g_ref[k], f"{name}.grad", kernel, k)
            else:
                assert name not in params
    finally:
        a.cpu()
