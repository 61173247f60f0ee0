"""The float64 channel-branch reference (oracle/channel_ref.py) that tests/test_channel_branch_gpu.py holds the kernels to:
its analytic backward against autograd of its own forward, its forward against the fp32 oracle's channel section
(oracle.oss_ref.channel), and the resolution of its bound: a reference with a plausible kernel bug in it must break the bound."""
import pytest
import torch

from oracle import channel_ref as cr
from oracle import oss_ref

CASES = [  # (variant, d_model, ssm_ratio, d_state, regime, B, L)
    ("sisr", 13, 1, 16, "randn", 2, 64),
    ("mamber32", 37, 1, 16, "dtinit", 3, 4096),
    ("mamber33", 30, 1, 16, "randn", 1, 64),
    ("mamber33", 24, 2, 16, "dtinit", 2, 4096),
    ("realsr", 40, 1, 8, "dtinit", 2, 64),
    ("realsr", 21, 2, 11, "randn", 3, 4096),
]


def pooled_sums(B, C, L, seed):
    g = torch.Generator().manual_seed(seed)
    return (L * (0.5 * torch.randn(B, C, generator=g) + 0.2)).float()


@pytest.mark.parametrize("variant,d_model,ratio,N,regime,B,L", CASES)
def test_analytic_backward_matches_autograd(variant, d_model, ratio, N, regime, B, L):
    a = cr.make_module(variant, d_model, ratio, N, regime, seed=d_model)
    C = a.d_inner
    prm = cr.prm64(cr.module_prm(a))
    leaves = {k: v.clone().requires_grad_() for k, v in prm.items() if torch.is_tensor(v)}
    pooled = pooled_sums(B, C, L, 1).double().requires_grad_()
    c, ctx = cr.forward(pooled, 1.0 / L, {**prm, **leaves})
    g = torch.randn(B, C, dtype=torch.float64)
    auto = torch.autograd.grad(c.v, [pooled, *leaves.values()], g)
    dpooled, gr = cr.backward(ctx, g)
    for name, got, want in zip(["pooled", *leaves], [dpooled, *(gr[k] for k in leaves)], auto):
        err = (got.v.detach() - want).abs()
        assert bool((err <= 1e-10 * got.s.detach()).all()), (name, float(err.max()), float(want.abs().max()))


@pytest.mark.parametrize("variant,d_model,ratio,N,regime,B,L", CASES)
def test_forward_matches_fp32_oracle(variant, d_model, ratio, N, regime, B, L):
    a = cr.make_module(variant, d_model, ratio, N, regime, seed=d_model + 1)
    C = a.d_inner
    pooled = pooled_sums(B, C, L, 2)
    c, _ = cr.forward(pooled.double(), 1.0 / L, cr.prm64(cr.module_prm(a)))
    sd = {k: v.detach().float() for k, v in a.state_dict().items()}
    got = oss_ref.channel(sd, "", pooled * (1.0 / L)).double()
    err = (got - c.v).abs()
    bound = cr.bound(c)
    assert bool((err <= bound).all()), float((err / bound).max())


RES_CASES = [  # (variant, d_model, d_state, regime): both regimes, a width with v1's 4-position and v2's 8-position tails
    ("sisr", 48, 16, "randn"), ("mamber33", 37, 16, "dtinit"), ("realsr", 96, 16, "dtinit"), ("realsr", 30, 11, "randn"),
]


@pytest.mark.parametrize("perturb", ["drop_last_bu", "drop_last_state", "bf16_mean"])
@pytest.mark.parametrize("variant,d_model,N,regime", RES_CASES)
def test_bound_resolves_plausible_bugs(perturb, variant, d_model, N, regime):
    """the bound the GPU tests apply, forward (c) and backward (dpooled and every parameter gradient), is broken somewhere by a
    reference with one of these bugs: the last position's B u term dropped (a loop-tail bug), the last state lane dropped (a lane
    masking bug), the pooled mean rounded to bf16 (a precision bug)"""
    a = cr.make_module(variant, d_model, 1, N, regime, seed=d_model + 2)
    C, B, L = a.d_inner, 3, 64
    prm = cr.prm64(cr.module_prm(a))
    pooled = pooled_sums(B, C, L, 3).double()
    g = torch.randn(B, C, dtype=torch.float64)
    c, ctx = cr.forward(pooled, 1.0 / L, prm)
    cp, ctxp = cr.forward(pooled, 1.0 / L, prm, perturb=perturb)
    assert bool(((cp.v - c.v).abs() > cr.bound(c)).any()), "forward"
    dp, gr = cr.backward(ctx, g)
    dpp, grp = cr.backward(ctxp, g)
    broken = [k for k in gr if ((grp[k].v - gr[k].v).abs() > cr.bound(gr[k])).any()]
    assert ((dpp.v - dp.v).abs() > cr.bound(dp)).any() or broken, "backward"
