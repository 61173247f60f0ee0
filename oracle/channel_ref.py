"""Float64 reference of the channel-direction OSS, forward and backward, with a rounding-error magnitude next to every value.
TEST INFRASTRUCTURE ONLY.

The operation is SS2D_1.cforward_pooled (vmambair_b200/archs.py) on the pooled sums, as vmb_channel_branch / vmb_channel_branch_bwd
compute it (csrc/oss_ops.cu, csrc/channel_bwd.cu): pooled mean -> conv_cin affine (absent for realsr) -> two directions (natural,
flipped) -> xc_proj -> dtc_proj + bias + softplus -> selective scan over L = C with A = -exp(Ac_logs), D = Dsc -> un-flip + sum ->
conv_cout (absent for realsr) -> channel_norm (WithBias LayerNorm over C).  The backward is written analytically, phase by phase as
channel_bwd.cu runs it (channel_norm, conv_cout + merge, Dsc, the reverse scan, dtc_proj, xc_proj, conv_cin, pool).

Every intermediate is an E: its float64 value v and a magnitude s, built by the same expression over absolute values
(s(a + b) = s(a) + s(b), s(a b) = s(a) |b| + |a| s(b), s(f(x)) = |f'(x)| s(x) + |f(x)|; inputs and parameters start at s = |v|).
eps_fp32 * s is then a first-order bound, up to a constant, on the error an fp32 evaluation of the same expressions makes, whatever
the order of its sums.  Two consequences are deliberate:
- the scan's magnitude is weighted by its effective memory length: s(h_l) = a_l s(h_{l-1}) + ..., so with a ~ 1 (the realsr dt init:
  dt ~ 1e-3..1e-1, A = -(1..16)) the rounding of every earlier step stays in s(h_l), as it stays in the fp32 state;
- the LayerNorm's rstd carries an extra relative (1 + rho), rho = sum_l (|x| + |mu|)^2 / sum_l (x - mu)^2 per image: the condition
  number of the variance, which the statistic's own rounding error is relative to (as in tests/test_train_ops_gpu.py).
bound() turns s into the element-wise test bound u_out |ref| + K eps_fp32 s.
"""
from __future__ import annotations

import torch

EPS32 = torch.finfo(torch.float32).eps
U_OUT = 2.0 ** -24  # the kernels' outputs are fp32
# K: the fp32 sums here err by about 0.2 eps per unit of s; MUFU ex2 / the fast reciprocal square root add a few eps, the fp32 atomics
# of the parameter gradients a few more.  16 leaves room for those.  Where a value is a sum whose terms cancel (the parameter gradients
# the LayerNorm's null space nearly removes: Dsc, conv_cout.weight, conv_cin, the dtc projection), s keeps the cancelled mass and
# K eps s can exceed the value itself; tests/test_channel_branch_gpu.py adds a norm-wise criterion for those.
K = 16
KEYS = ("cin_w", "cin_b", "xc_proj", "dtc_w", "dtc_b", "Ac_logs", "Dsc", "cout_w", "cout_b", "cn_w", "cn_b")


class E:
    """float64 value v and its rounding magnitude s (module docstring)"""
    __slots__ = ("v", "s")

    def __init__(self, v, s=None):
        self.v = v
        self.s = v.abs() if s is None else s

    def __add__(a, b):
        b = _e(b)
        return E(a.v + b.v, a.s + b.s)

    __radd__ = __add__

    def __sub__(a, b):
        b = _e(b)
        return E(a.v - b.v, a.s + b.s)

    def __rsub__(a, b):
        return _e(b) - a

    def __neg__(a):
        return E(-a.v, a.s)

    def __mul__(a, b):
        b = _e(b)
        return E(a.v * b.v, a.s * b.v.abs() + a.v.abs() * b.s)

    __rmul__ = __mul__

    def __getitem__(a, i):
        return E(a.v[i], a.s[i])

    def map(a, f):
        """a shape-only function (view, flip, unsqueeze, ...) applied to both parts"""
        return E(f(a.v), f(a.s))

    def sum(a, *dims, keepdim=False):
        return E(a.v.sum(dims, keepdim=keepdim), a.s.sum(dims, keepdim=keepdim))

    def mean(a, dim, keepdim=False):
        return E(a.v.mean(dim, keepdim=keepdim), a.s.mean(dim, keepdim=keepdim))


def _e(x):
    if isinstance(x, E):
        return x
    x = torch.as_tensor(x, dtype=torch.float64)
    return E(x)


def stack(es, dim):
    return E(torch.stack([e.v for e in es], dim), torch.stack([e.s for e in es], dim))


def cat(es, dim):
    return E(torch.cat([e.v for e in es], dim), torch.cat([e.s for e in es], dim))


def ein(spec, a, b):
    return E(torch.einsum(spec, a.v, b.v), torch.einsum(spec, a.s, b.v.abs()) + torch.einsum(spec, a.v.abs(), b.s))


def exp(x):
    v = x.v.exp()
    return E(v, v * (x.s + 1))


def softplus(x):
    v = torch.logaddexp(x.v, torch.zeros_like(x.v))
    return E(v, torch.sigmoid(x.v) * x.s + v)


def sigmoid(x):
    v = torch.sigmoid(x.v)
    return E(v, v * (1 - v) * x.s + v)


def rsqrt(x):
    v = x.v.rsqrt()
    return E(v, 0.5 * v / x.v * x.s + v)


def bound(ref):
    """element-wise bound of an fp32 result against the E `ref`"""
    return U_OUT * ref.v.abs() + K * EPS32 * ref.s


def prm64(prm):
    """a launcher's prm dict (fp32 tensors on any device, cin / cout None for realsr) -> the same as float64 CPU"""
    return {k: (v.detach().double().cpu() if torch.is_tensor(v) else v) for k, v in prm.items()}


def module_prm(a):
    """the channel parameters of SS2D_1 `a` as fused_train._Channel hands them to the launchers (flat, cin / cout None for realsr)"""
    has_cio = hasattr(a, "conv_cin")
    flat = lambda t: t.detach().float().reshape(-1)
    return dict(cin_w=flat(a.conv_cin.weight) if has_cio else None, cin_b=flat(a.conv_cin.bias) if has_cio else None,
                xc_proj=flat(a.xc_proj_weight), dtc_w=flat(a.dtc_projs_weight), dtc_b=flat(a.dtc_projs_bias), Ac_logs=flat(a.Ac_logs),
                Dsc=flat(a.Dsc), cout_w=flat(a.conv_cout.weight) if has_cio else None, cout_b=flat(a.conv_cout.bias) if has_cio else None,
                cn_w=flat(a.channel_norm.body.weight), cn_b=flat(a.channel_norm.body.bias), dc=a.dc_inner, Rc=a.dtc_rank, N=a.dc_state)


def make_module(variant, d_model, ratio=1, d_state=16, regime="randn", seed=0):
    """SS2D_1 on the CPU with its channel parameters in one of two regimes, then moved off their init constants (as
    tests/test_ss2d_fused_gpu.make does): "randn" -- the sisr / mamber init (randn Ac_logs, dtc weight and bias: short, varied
    memory); "dtinit" -- the realsr init (dt ~ 1e-3..1e-1 through softplus^-1 biases, A = -(1..N): a ~ 1, memory up to the whole
    sequence)"""
    from vmambair_b200 import archs
    torch.manual_seed(seed)
    a = archs.SS2D_1(d_model=d_model, ssm_ratio=ratio, d_state=d_state, variant=variant)
    dc, Rc, N = a.dc_inner, a.dtc_rank, a.dc_state
    with torch.no_grad():
        if regime == "randn":
            a.Ac_logs.copy_(torch.randn(2 * dc, N))
            a.dtc_projs_weight.copy_(torch.randn(2, dc, Rc))
            a.dtc_projs_bias.copy_(torch.randn(2, dc))
        else:
            dts = [archs.SS2D_1.dt_init(Rc, dc) for _ in range(2)]
            a.dtc_projs_weight.copy_(torch.stack([t.weight for t in dts], 0))
            a.dtc_projs_bias.copy_(torch.stack([t.bias for t in dts], 0))
            a.Ac_logs.copy_(archs.SS2D_1.A_log_init(N, dc, copies=2))
        for n, p in a.named_parameters():
            if n.endswith(("body.weight", "body.bias", "Ds", "Dsc", "A_logs", "Ac_logs")):
                p.add_(0.1 * torch.randn_like(p))
    return a


# module parameter name -> prm key
PARAM_KEYS = {"conv_cin.weight": "cin_w", "conv_cin.bias": "cin_b", "xc_proj_weight": "xc_proj", "dtc_projs_weight": "dtc_w",
              "dtc_projs_bias": "dtc_b", "Ac_logs": "Ac_logs", "Dsc": "Dsc", "conv_cout.weight": "cout_w", "conv_cout.bias": "cout_b",
              "channel_norm.body.weight": "cn_w", "channel_norm.body.bias": "cn_b"}


def forward(pooled, inv_count, prm, perturb=None):
    """pooled (B, C) sums and prm (prm64) -> (c E (B, C), ctx for backward()).

    perturb (resolution checks only): "drop_last_bu" -- the last position's B u term of every scan row left out;
    "drop_last_state" -- the last state lane left out of the scan (of y here, and of dh, dB, dC and d Ac_logs in backward());
    "bf16_mean" -- the pooled mean rounded to bf16 first."""
    dc, Rc, N = prm["dc"], prm["Rc"], prm["N"]
    RN = Rc + 2 * N
    P = {k: (E(v) if torch.is_tensor(v) else None) for k, v in prm.items() if k in KEYS}
    B_, C = pooled.shape
    m = E(pooled) * inv_count
    if perturb == "bf16_mean":
        m = E(m.v.to(torch.bfloat16).double(), m.s)
    if P["cin_w"] is not None:
        seq = m.map(lambda t: t[:, None, :]) * P["cin_w"].map(lambda t: t.view(1, dc, 1)) + P["cin_b"].map(lambda t: t.view(1, dc, 1))
    else:
        seq = m.map(lambda t: t[:, None, :])
    xs = stack([seq, seq.map(lambda t: t.flip(-1))], 1)                       # (B, 2, dc, C)
    xp = P["xc_proj"].map(lambda t: t.view(2, RN, dc))
    dbl = ein("bkjl,kcj->bkcl", xs, xp)                                        # (B, 2, RN, C)
    dtw = P["dtc_w"].map(lambda t: t.view(2, dc, Rc))
    pre = ein("bkrl,kjr->bkjl", dbl[:, :, :Rc], dtw) + P["dtc_b"].map(lambda t: t.view(1, 2, dc, 1))
    dt = softplus(pre)                                                          # (B, 2, dc, C)
    A = -exp(P["Ac_logs"]).map(lambda t: t.view(1, 2, dc, N))
    D = P["Dsc"].map(lambda t: t.view(1, 2, dc))
    Bm, Cm = dbl[:, :, Rc:Rc + N], dbl[:, :, Rc + N:]                           # (B, 2, N, C)
    lanes = N - 1 if perturb == "drop_last_state" else N
    z = torch.zeros(B_, 2, dc, N, dtype=torch.float64)
    h = E(z, z)
    hs, as_, ys = [], [], []
    for l in range(C):
        dtl, ul = dt[..., l], xs[..., l]
        a = exp(dtl.map(lambda t: t[..., None]) * A)
        bu = (dtl * ul).map(lambda t: t[..., None]) * Bm[..., l].map(lambda t: t[:, :, None, :])
        if perturb == "drop_last_bu" and l == C - 1:
            bu = E(torch.zeros_like(bu.v), bu.s)
        h = a * h + bu
        hc = h * Cm[..., l].map(lambda t: t[:, :, None, :])
        ys.append(D * ul + hc[..., :lanes].sum(-1))
        hs.append(h)
        as_.append(a)
    y = stack(ys, -1)                                                           # (B, 2, dc, C)
    ym = y[:, 0] + y[:, 1].map(lambda t: t.flip(-1))                            # (B, dc, C)
    if P["cout_w"] is not None:
        out = (ym * P["cout_w"].map(lambda t: t.view(1, dc, 1))).sum(1) + P["cout_b"]
    else:
        out = ym[:, 0]
    mu = out.mean(-1, keepdim=True)
    d = out - mu
    var = (d * d).mean(-1, keepdim=True)
    rho = (out.v.abs() + mu.v.abs()).square().sum(-1, keepdim=True) / d.v.square().sum(-1, keepdim=True).clamp_min(1e-300)
    rstd = rsqrt(var + 1e-5)
    rstd = E(rstd.v, rstd.s + rho * rstd.v)
    xh = d * rstd
    c = xh * P["cn_w"] + P["cn_b"]
    ctx = dict(P=P, dims=(B_, C, dc, Rc, N), lanes=lanes, inv_count=inv_count, m=m, xs=xs, dbl=dbl, dtw=dtw, pre=pre, dt=dt, A=A, D=D,
               Bm=Bm, Cm=Cm, hs=hs, as_=as_, ym=ym, rstd=rstd, xh=xh)
    return c, ctx


def backward(ctx, dc_out):
    """analytic backward of forward() at dc_out (B, C) float64 -> (dpooled E (B, C), {key: E} flat like the launcher's prm)"""
    P, (B_, C, dc, Rc, N) = ctx["P"], ctx["dims"]
    xs, dbl, dt, A, D, Bm, Cm = (ctx[k] for k in ("xs", "dbl", "dt", "A", "D", "Bm", "Cm"))
    rstd, xh, hs, as_ = ctx["rstd"], ctx["xh"], ctx["hs"], ctx["as_"]
    g = E(dc_out)
    gr = {}
    # channel_norm
    gr["cn_w"], gr["cn_b"] = (g * xh).sum(0), g.sum(0)
    gw = g * P["cn_w"]
    dout = rstd * (gw - gw.mean(-1, keepdim=True) - xh * (gw * xh).mean(-1, keepdim=True))  # (B, C)
    # conv_cout + merge
    if P["cout_w"] is not None:
        gr["cout_b"] = dout.sum(0, 1).map(lambda t: t.view(1))
        gr["cout_w"] = (dout.map(lambda t: t[:, None, :]) * ctx["ym"]).sum(0, 2)
        cw = P["cout_w"].map(lambda t: t.view(1, dc, 1))
        dy = stack([dout.map(lambda t: t[:, None, :]) * cw, dout.map(lambda t: t.flip(-1)[:, None, :]) * cw], 1)
    else:
        dy = stack([dout.map(lambda t: t[:, None, :]), dout.map(lambda t: t.flip(-1)[:, None, :])], 1)  # (B, 2, dc, C)
    gr["Dsc"] = (dy * xs).sum(0, 3).map(lambda t: t.reshape(-1))
    # reverse scan
    z = torch.zeros(B_, 2, dc, N, dtype=torch.float64)
    dh = E(z, z)
    lane = (torch.arange(N) < ctx["lanes"]).double()  # 0 on a state lane the forward left out
    dpre, du, dAs, dB, dC = [None] * C, [None] * C, [], [None] * C, [None] * C
    for l in range(C - 1, -1, -1):
        dyl, dtl, ul = dy[..., l], dt[..., l], xs[..., l]
        Bl, Cl = Bm[..., l].map(lambda t: t[:, :, None, :]), Cm[..., l].map(lambda t: t[:, :, None, :])
        dh = (Cl * dyl.map(lambda t: t[..., None]) + (as_[l + 1] * dh if l + 1 < C else dh)) * lane
        hprev = hs[l - 1] if l > 0 else E(z, z)
        ahp = as_[l] * hprev
        t1 = (dh * Bl).sum(-1)
        t2 = (A * dh * ahp).sum(-1)
        dpre[l] = (ul * t1 + t2) * sigmoid(ctx["pre"][..., l])
        du[l] = dtl * t1 + D * dyl
        dAs.append(dh * dtl.map(lambda t: t[..., None]) * ahp)
        dB[l] = (dh * (dtl * ul).map(lambda t: t[..., None])).sum(2)            # (B, 2, N): summed over the rows of a direction
        dC[l] = (dyl.map(lambda t: t[..., None]) * hs[l] * lane).sum(2)
    gr["Ac_logs"] = (A.map(lambda t: t[0]) * stack(dAs, 0).sum(0, 1)).map(lambda t: t.reshape(-1))
    dpre, du, dB, dC = stack(dpre, -1), stack(du, -1), stack(dB, -1), stack(dC, -1)
    # dtc_proj
    gr["dtc_w"] = ein("bkjl,bkrl->kjr", dpre, dbl[:, :, :Rc]).map(lambda t: t.reshape(-1))
    gr["dtc_b"] = dpre.sum(0, 3).map(lambda t: t.reshape(-1))
    ddbl = cat([ein("bkjl,kjr->bkrl", dpre, ctx["dtw"]), dB, dC], 2)           # (B, 2, RN, C)
    # xc_proj
    gr["xc_proj"] = ein("bkcl,bkjl->kcj", ddbl, xs).map(lambda t: t.reshape(-1))
    dxs = du + ein("bkcl,kcj->bkjl", ddbl, P["xc_proj"].map(lambda t: t.view(2, Rc + 2 * N, dc)))
    dseq = dxs[:, 0] + dxs[:, 1].map(lambda t: t.flip(-1))                     # (B, dc, C)
    # conv_cin, pool
    if P["cin_w"] is not None:
        gr["cin_w"] = (dseq * ctx["m"].map(lambda t: t[:, None, :])).sum(0, 2)
        gr["cin_b"] = dseq.sum(0, 2)
        dpooled = (dseq * P["cin_w"].map(lambda t: t.view(1, dc, 1))).sum(1) * ctx["inv_count"]
    else:
        dpooled = dseq[:, 0] * ctx["inv_count"]
    return dpooled, gr
