"""Each backward / weight-preparation stage of the training path (vmambair_b200.fused_train) through its ops.* wrapper against a
float64 CPU reference of the same operation, on every dispatch path of its launcher, plus the fused training step of a whole block
at image sizes where those paths change (odd H*W, W % 8 != 0, C*L not a multiple of the vector width).

The references take the same dtype-rounded inputs as the kernels; the parameter-gradient phases take the kernel's own data-phase
outputs (stats, dv) as inputs, so that errors do not compound.  Every element is bounded on its own (check()):

    |got - ref| <= u_out * |ref|  +  K * eps_fp32 * S

u_out is the unit roundoff of the output dtype, S the sum of the absolute values of the terms that produced the element (computed
next to each reference).  Terms scaled by a LayerNorm statistic carry the factor (1 + rho), rho = sum_c (|x| + |mu|)^2 / sum_c (x - mu)^2
per pixel: the condition number of the variance, which the statistic's own rounding error is relative to.

No kernel has a path switch: each path is reached by the layout of its inputs alone (the conditions are those of the launchers in
csrc/train_ops.cu, csrc/wgrad.cu and ops.py, mirrored by the *_fast() helpers, which the tests assert so that a layout cannot drift
onto the other path unnoticed).  Where both paths can take the same values they run on the same values.

Bugs these tests found:
- ops.sum4_add rejected C*L not a multiple of the 16 B vector width (any fused training step at dim 30 on 7x9 in fp32): it now falls
  back to a torch sum there, like pixlin_wgrad.
- ops.pixlin_wgrad's torch fallback for 16-bit rows that are not 16 B aligned rounded dW to bf16 / fp16: it now accumulates in fp32.
"""
import pytest
import torch
import torch.nn.functional as F

import vmambair_b200.archs as archs
from vmambair_b200 import ops

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
U_OUT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY = {torch.float32: 0.0, torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}  # half the fp16 subnormal spacing
EPS32 = torch.finfo(torch.float32).eps
# K: fp32 sums of n random-signed terms err by about 0.2 eps * S; the per-pixel statistics, the approximate exp / reciprocal of the
# activations and the fp32 atomics of the parameter gradients add a few eps more.  16 leaves room for those and is still ~1e-4 of
# any O(1) mistake (a dropped bias, a wrong tap, a wrong statistic).
K = 16


def check(got, ref, S, dtype, what):
    """element-wise bound of the module docstring; got: kernel output (any device / dtype), ref / S: float64 CPU"""
    got = got.detach().double().cpu()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    bound = U_OUT[dtype] * ref.abs() + K * EPS32 * S + TINY[dtype]
    bad = ~(err <= bound)
    if bad.any():
        i = int((err / bound.clamp_min(1e-300)).flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements out of bound; worst at flat index {i}: "
                             f"got {float(got.flatten()[i])}, ref {float(ref.flatten()[i])}, bound {float(bound.flatten()[i])}")
    return bound


def check_pair(a, b, bound_a, bound_b, what):
    """the two dispatch paths of one launcher on the same values: within the sum of their bounds of the fp64 reference"""
    assert bool(((a.detach().double().cpu() - b.detach().double().cpu()).abs() <= bound_a + bound_b).all()), what


def rnd(dtype, *shape, scale=1.0, shift=None):
    """random CUDA tensor rounded to dtype (the kernels' inputs) and its float64 CPU copy (the references' inputs)"""
    t = torch.randn(*shape, device="cuda") * scale
    if shift is not None:
        t = t + shift
    t = t.to(dtype)
    return t, t.double().cpu()


# ----------------------------------------------------------------------------- layouts: the same values on either path
def offset_view(t, c0=4):
    """t in channels c0.. of a wider buffer: batch stride != C*L, as xz[:, C:] is in the block (c0 = 4 keeps 8 B alignment)"""
    B, C_, L = t.shape
    buf = torch.randn(B, C_ + c0, L, device=t.device).to(t.dtype)
    buf[:, c0:] = t
    return buf[:, c0:]


def odd_stride(t):
    """t as buf[..., :L] of a (B, C, L + 1) buffer: channel stride L + 1"""
    B, C_, L = t.shape
    buf = torch.randn(B, C_, L + 1, device=t.device).to(t.dtype)
    buf[..., :L] = t
    return buf[..., :L]


def misaligned(t):
    """contiguous t starting one element into its storage: not 16 B aligned"""
    flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = flat[1:].view(t.shape)
    v.copy_(t)
    return v


def ln_fast(C_, L, *ts):
    """train_ops.cu ln_fwd_launch / ln_bwd_launch: the channel-split px kernels"""
    return L >= 2 and L % 2 == 0 and C_ >= 8 and all(t.stride(0) % 2 == 0 and t.stride(1) % 2 == 0 and t.data_ptr() % 8 == 0 for t in ts)


def ln_params_fast(L, *ts):
    """train_ops.cu ln_bwd_dwdb_kernel: the pixel-pair loop"""
    return L % 2 == 0 and all(t.stride(0) % 2 == 0 and t.stride(1) % 2 == 0 and t.data_ptr() % 8 == 0 for t in ts)


def merge_fast(C_, L, stats_ptr, z, dz):
    """train_ops.cu merge_bwd_launch: merge_bwd_dx_px_kernel (dy2 / dm are fresh contiguous tensors)"""
    return L >= 2 and L % 2 == 0 and C_ >= 8 and stats_ptr % 16 == 0 and \
        all(t.stride(0) % 2 == 0 and t.stride(1) % 2 == 0 and t.data_ptr() % 8 == 0 for t in (z, dz))


def dw_fast(W, *ts):
    """train_ops.cu vmb_dwconv3x3_bwd vec_ok: 8-pixel strips with 16 B loads"""
    return W % 8 == 0 and all(t.data_ptr() % 16 == 0 and t.stride(0) % 8 == 0 and t.stride(1) % 8 == 0 for t in ts)


# ----------------------------------------------------------------------------- float64 references
def ln_stats64(x):
    """x (B,C,L) float64 -> mu, d = x - mu, rstd, rho (each (B,1,L) but d)"""
    mu = x.mean(1, keepdim=True)
    d = x - mu
    rstd = (d.square().mean(1, keepdim=True) + 1e-5).rsqrt()
    rho = ((x.abs() + mu.abs()).square().sum(1, keepdim=True) / d.square().sum(1, keepdim=True).clamp_min(1e-300))
    return mu, d, rstd, rho


def ln_fwd64(x, mode, w, b):
    mu, d, rstd, rho = ln_stats64(x)
    w, A = w.view(1, -1, 1), x.abs() + mu.abs()
    if mode == 1:
        return d * rstd * w + b.view(1, -1, 1), A * rstd * w.abs() * (1 + rho) + b.abs().view(1, -1, 1)
    return x * rstd * w, x.abs() * rstd * w.abs() * (1 + rho)


def ln_bwd_dx64(x, g, mode, w, add):
    """-> (dx, S, mu, rstd, S_rstd)"""
    C_ = x.shape[1]
    mu, d, rstd, rho = ln_stats64(x)
    gw, agw, A = g * w.view(1, -1, 1), (g * w.view(1, -1, 1)).abs(), x.abs() + mu.abs()
    if mode == 1:
        dx = rstd * (gw - gw.mean(1, keepdim=True) - d * rstd.square() * (gw * d).mean(1, keepdim=True))
        S = rstd * (agw + agw.mean(1, keepdim=True) + A * rstd.square() * (agw * A).mean(1, keepdim=True)) * (1 + rho)
    else:
        dx = rstd * gw - rstd ** 3 * d * (gw * x).sum(1, keepdim=True) / C_
        S = rstd * (agw + A * rstd.square() * (agw * x.abs()).mean(1, keepdim=True)) * (1 + rho)
    if add is not None:
        dx, S = dx + add, S + add.abs()
    return dx, S, mu, rstd, rstd * (1 + rho)


def ln_params64(x, g, mode, stats):
    """dw / db from the kernel's (mu, rstd) per pixel"""
    mu, rstd = stats[..., 0].unsqueeze(1), stats[..., 1].unsqueeze(1)
    xh = (x - mu) * rstd if mode == 1 else x * rstd
    A = (x.abs() + (mu.abs() if mode == 1 else 0)) * rstd
    return (g * xh).sum((0, 2)), (g.abs() * A).sum((0, 2)), g.sum((0, 2)), g.abs().sum((0, 2))


# ----------------------------------------------------------------------------- LayerNorm
LN_C = [5, 8, 12, 48, 384]  # C = 5: per-pixel kernel by C; C = 12: uneven channel slices q * C / 8
LN_L = [2, 70, 4096]        # L = 70: the tail CTA of the px kernels clamps to the last pixel pair
LN_MODES = [(1, False), (1, True), (2, False), (2, True)]  # (1 WithBias / 2 BiasFree, residual-branch gradient `add` given)


def ln_batch(C_, L):
    return 3 if C_ * L <= 2 ** 18 else 1  # batch > 1 with channel-offset views; the largest plane once, to keep the fp64 side small


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("C_", LN_C)
@pytest.mark.parametrize("L", LN_L)
def test_layernorm_fwd(dtype, mode, C_, L):
    """vmb_layernorm_fwd: ln_fwd_px_kernel (channel-offset view) and ln_fwd_kernel (the same values at channel stride L + 1)"""
    torch.manual_seed(C_ * 7 + L + mode)
    B = ln_batch(C_, L)
    x, x64 = rnd(dtype, B, C_, L, shift=torch.randn(B, 1, L, device="cuda"))
    w = 1 + 0.5 * torch.randn(C_, device="cuda")
    b = 0.5 * torch.randn(C_, device="cuda") if mode == 1 else None
    ref, S = ln_fwd64(x64, mode, w.double().cpu(), b.double().cpu() if b is not None else None)
    xa, xb = offset_view(x), odd_stride(x)
    assert ln_fast(C_, L, xa) == (C_ >= 8) and not ln_fast(C_, L, xb)
    ya, yb = ops.layernorm_fwd(xa, mode, w, b), ops.layernorm_fwd(xb, mode, w, b)
    check_pair(ya, yb, check(ya, ref, S, dtype, "y (px)"), check(yb, ref, S, dtype, "y (per pixel)"), "y: px vs per pixel")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode,has_add", LN_MODES)
@pytest.mark.parametrize("C_", LN_C)
@pytest.mark.parametrize("L", LN_L)
def test_layernorm_bwd(dtype, mode, has_add, C_, L):
    """vmb_layernorm_bwd data phase (ln_bwd_dx_px_kernel / ln_bwd_dx_kernel: dx and the (mu, rstd) statistics) and params phase
    (ln_bwd_dwdb_kernel pixel-pair / scalar loop), each fed the statistics of the OTHER data path as well as its own"""
    torch.manual_seed(C_ * 11 + L + mode + 2 * has_add)
    B = ln_batch(C_, L)
    x, x64 = rnd(dtype, B, C_, L, shift=torch.randn(B, 1, L, device="cuda"))
    g, g64 = rnd(dtype, B, C_, L)
    add, add64 = rnd(dtype, B, C_, L) if has_add else (None, None)
    w = 1 + 0.5 * torch.randn(C_, device="cuda")
    dx_ref, S, mu_ref, rstd_ref, S_rstd = ln_bwd_dx64(x64, g64, mode, w.double().cpu(), add64)
    lay = {"px": offset_view, "per pixel": odd_stride}
    res = {}
    for name, f in lay.items():
        xx, gg, aa = f(x), f(g), (f(add) if add is not None else None)
        assert ln_fast(C_, L, *[t for t in (xx, gg, aa) if t is not None]) == (name == "px" and C_ >= 8)
        dx, st = ops.layernorm_bwd(xx, gg, mode, w, add=aa, phase="data")
        bd = check(dx, dx_ref, S, dtype, f"dx ({name})")
        check(st[..., 0], mu_ref[:, 0], (x64.abs().mean(1) + mu_ref[:, 0].abs()), torch.float32, f"mu ({name})")
        check(st[..., 1], rstd_ref[:, 0], S_rstd[:, 0], torch.float32, f"rstd ({name})")
        res[name] = (dx, bd, st, xx, gg)
    check_pair(res["px"][0], res["per pixel"][0], res["px"][1], res["per pixel"][1], "dx: px vs per pixel")
    for data_path in lay:  # the parameter phase of either layout on the statistics of either data path
        st = res[data_path][2]
        dw_ref, S_dw, db_ref, S_db = ln_params64(x64, g64, mode, st.double().cpu())
        for name in lay:
            xx, gg = res[name][3], res[name][4]
            assert ln_params_fast(L, xx, gg) == (name == "px" and L % 2 == 0)
            dw, db = ops.layernorm_bwd(xx, gg, mode, w, phase="params", stats=st)
            check(dw, dw_ref, S_dw, torch.float32, f"dw ({name} loop, stats of the {data_path} path)")
            if mode == 1:
                check(db, db_ref, S_db, torch.float32, f"db ({name} loop, stats of the {data_path} path)")
            else:
                assert db is None


# ----------------------------------------------------------------------------- out_norm + SiLU gate
def _silu64(z):
    s = torch.sigmoid(z)
    return z * s, s * (1 + z * (1 - s)), s


MERGE_CASES = [  # (B, C, H, W, producer of the forward workspace: "single" kernel (16-bit, H, W % 16 == 0, C <= 96, H W >= 128 x 128)
    #             / "two" kernels)
    (2, 48, 128, 128, "single"), (2, 48, 16, 16, "two"),
    (2, 5, 128, 128, "single"), (2, 5, 16, 32, "two"),   # C = 5: per-pixel kernel by C
    (2, 12, 7, 9, "two"),                                 # odd L
    (1, 9, 2, 3, "two"),                                  # B*C*L % 4 != 0: statistics not 16 B aligned
    (1, 96, 128, 128, "single"),
]


@pytest.mark.parametrize("dtype,B,C_,H,W,producer", [(dt, *c) for dt in DTYPES for c in MERGE_CASES
                                                     if not (dt == torch.float32 and c[4] == "single")])
@pytest.mark.parametrize("has_dpool", [False, True])
def test_merge_norm_gate_bwd(dtype, B, C_, H, W, producer, has_dpool):
    """vmb_merge_norm_gate_bwd on the workspace of either forward producer: dm, dz through merge_bwd_dx_px_kernel (z, dz channel-offset
    views) and merge_bwd_dx_kernel (the same z at channel stride L + 1), and d ln_w / d ln_b"""
    torch.manual_seed(C_ * 5 + H + W + has_dpool)
    L = H * W
    ys = torch.randn(B, 4, C_, L, device="cuda").to(dtype)
    z, z64 = rnd(dtype, B, C_, L, scale=2.0)
    lw = 1 + 0.5 * torch.randn(C_, device="cuda")
    lb = 0.5 * torch.randn(C_, device="cuda")
    _, _, ws = ops.merge_norm_gate(ys, z, lw, lb, C_, H, W, z_preact=True, return_ws=True)
    dy2, dy2_64 = rnd(dtype, B, C_, L)
    dpool = torch.randn(B, C_, device="cuda") * 3 if has_dpool else None
    # reference: the forward's merged fp32 values are the input; its statistics are recomputed here (this checks the producer's too)
    m64 = ws.view(torch.float32)[:B * C_ * L].view(B, C_, L).double().cpu()
    mu, d, rstd, rho = ln_stats64(m64)
    A = m64.abs() + mu.abs()
    w64, b64 = lw.double().cpu().view(1, -1, 1), lb.double().cpu().view(1, -1, 1)
    t = dy2_64 + (dpool.double().cpu().unsqueeze(-1) if has_dpool else 0)
    at = dy2_64.abs() + (dpool.double().cpu().abs().unsqueeze(-1) if has_dpool else 0)
    sz, dsz, sg = _silu64(z64)
    gw, agw = t * sz * w64, at * sz.abs() * w64.abs()
    dm_ref = rstd * (gw - gw.mean(1, keepdim=True) - d * rstd.square() * (gw * d).mean(1, keepdim=True))
    S_dm = rstd * (agw + agw.mean(1, keepdim=True) + A * rstd.square() * (agw * A).mean(1, keepdim=True)) * (1 + rho)
    n = d * rstd * w64 + b64
    dz_ref = t * n * dsz
    S_dz = at * (A * rstd * w64.abs() * (1 + rho) + b64.abs()) * sg * (1 + 3 * z64.abs())
    dn, adn = t * sz, at * sz.abs()
    dw_ref, S_dw = (dn * d * rstd).sum((0, 2)), (adn * A * rstd * (1 + rho)).sum((0, 2))
    db_ref, S_db = dn.sum((0, 2)), adn.sum((0, 2))
    stats_ptr = ws.data_ptr() + 4 * B * C_ * L
    res = {}
    for name, f in (("px", offset_view), ("per pixel", odd_stride)):
        zz = f(z)
        dz = f(torch.zeros_like(z))
        assert merge_fast(C_, L, stats_ptr, zz, dz) == (name == "px" and merge_fast(C_, L, stats_ptr, z, z))
        dm = ops.merge_norm_gate_bwd(ws, zz, dy2, dpool, lw, lb, C_, L, dz_out=dz, phase="data")
        res[name] = (dm, check(dm, dm_ref, S_dm, dtype, f"dm ({name})"), dz, check(dz, dz_ref, S_dz, dtype, f"dz ({name})"))
        dw, db = ops.merge_norm_gate_bwd(ws, zz, dy2, dpool, lw, lb, C_, L, dz_out=None, phase="params")
        check(dw, dw_ref, S_dw, torch.float32, f"d ln_w ({name} z)")
        check(db, db_ref, S_db, torch.float32, f"d ln_b ({name} z)")
    (a, ba, za, bza), (b_, bb, zb, bzb) = res["px"], res["per pixel"]
    check_pair(a, b_, ba, bb, "dm: px vs per pixel")
    check_pair(za, zb, bza, bzb, "dz: px vs per pixel")


# ----------------------------------------------------------------------------- depthwise 3x3 + SiLU / GELU gate
DW_SHAPES = [  # (B, c_out, H, W)
    (2, 6, 8, 16),   # 8-pixel strips
    (2, 5, 1, 8),    # strips, one row: every pixel is in a border strip
    (3, 4, 3, 3),    # scalar: W % 8 != 0, every pixel on the border
    (2, 5, 5, 12),   # scalar: W = 12
    (2, 3, 9, 1),    # scalar: W = 1
]


def _gelu64(v):
    cdf = 0.5 * (1 + torch.erf(v * 0.5 ** 0.5))
    return v * cdf, cdf + v * torch.exp(-0.5 * v * v) / (2 * torch.pi) ** 0.5


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("has_bias", [False, True])
@pytest.mark.parametrize("B,Co,H,W", DW_SHAPES)
def test_dwconv3x3_bwd(dtype, mode, has_bias, B, Co, H, W):
    """vmb_dwconv3x3_bwd: dv (dwconv_bwd_pre_kernel) and dw9 / dbias (dwconv_wgrad_kernel, fed the kernel's own dv), on 8-pixel
    strips (aligned, W % 8 == 0) and per pixel (the same values one element into their storage)"""
    torch.manual_seed(B * 13 + Co + H * W + mode + 2 * has_bias)
    ch, L = Co * (2 if mode else 1), H * W
    x, x64 = rnd(dtype, B, ch, L)
    g, g64 = rnd(dtype, B, Co, L)
    w9 = 0.5 * torch.randn(ch, 9, device="cuda")
    bias = 0.5 * torch.randn(ch, device="cuda") if has_bias else None
    w64, b64 = w9.double().cpu().view(ch, 1, 3, 3), (bias.double().cpu() if has_bias else None)
    conv = lambda t, w, b: F.conv2d(t.view(B, ch, H, W), w, b, padding=1, groups=ch).view(B, ch, L)
    v = conv(x64, w64, b64)
    a = conv(x64.abs(), w64.abs(), b64.abs() if has_bias else None)  # sum of |terms| of each conv output
    if mode == 0:
        sg = torch.sigmoid(v)
        dv_ref, S_dv = g64 * sg * (1 + v * (1 - sg)), g64.abs() * (1 + a)
    else:
        v1, v2, a1, a2 = v[:, :Co], v[:, Co:], a[:, :Co], a[:, Co:]
        gl, dgl = _gelu64(v1)
        dv_ref = torch.cat([g64 * v2 * dgl, g64 * gl], 1)
        S_dv = torch.cat([g64.abs() * (a2 + v2.abs() * (1 + a1)), g64.abs() * 2 * a1], 1)
    res = {}
    for name, f in (("strips", lambda t: t), ("per pixel", misaligned)):
        xx, gg = f(x), f(g)
        assert dw_fast(W, xx, gg) == (name == "strips" and W % 8 == 0)
        dv = ops.dwconv3x3_bwd(xx, w9, bias, gg, Co, H, W, mode, phase="data")
        res[name] = (dv, check(dv, dv_ref, S_dv, dtype, f"dv ({name})"))
        # parameter gradients against the sums over this path's own dv
        dv64 = dv.double().cpu()
        xp, axp = F.pad(x64.view(B, ch, H, W), (1, 1, 1, 1)), F.pad(x64.abs().view(B, ch, H, W), (1, 1, 1, 1))
        d4, ad4 = dv64.view(B, ch, H, W), dv64.abs().view(B, ch, H, W)
        dw_ref = torch.stack([(d4 * xp[:, :, i // 3:i // 3 + H, i % 3:i % 3 + W]).sum((0, 2, 3)) for i in range(9)], 1)
        S_dw = torch.stack([(ad4 * axp[:, :, i // 3:i // 3 + H, i % 3:i % 3 + W]).sum((0, 2, 3)) for i in range(9)], 1)
        dw, db = ops.dwconv3x3_bwd(xx, w9, bias, None, Co, H, W, mode, phase="params", dv=dv)
        check(dw, dw_ref, S_dw, torch.float32, f"dw9 ({name})")
        if has_bias:
            check(db, dv64.sum((0, 2)), ad4.sum((0, 2, 3)), torch.float32, f"dbias ({name})")
        else:
            assert db is None
    check_pair(res["strips"][0], res["per pixel"][0], res["strips"][1], res["per pixel"][1], "dv: strips vs per pixel")


# ----------------------------------------------------------------------------- channel gate, sum4_add
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("B,C_,L", [(3, 7, 70), (2, 48, 4096)])
def test_channel_gate_bwd(dtype, mode, B, C_, L):
    """vmb_channel_gate_bwd: y2 * (1 + c) (mode 1) / y2 + c (mode 2) -> dy2 and the per-(image, channel) gate gradient"""
    torch.manual_seed(B + C_ + L + mode)
    dyg, dyg64 = rnd(dtype, B, C_, L)
    y2, y2_64 = rnd(dtype, B, C_, L)
    gate = torch.randn(B, C_, device="cuda")
    g64 = gate.double().cpu().unsqueeze(-1)
    dy2, dg = ops.channel_gate_bwd(dyg, y2, gate, mode)
    if mode == 1:
        check(dy2, dyg64 * (1 + g64), dyg64.abs() * (1 + g64.abs()), dtype, "dy2")
        check(dg, (dyg64 * y2_64).sum(2), (dyg64 * y2_64).abs().sum(2), torch.float32, "dgate")
    else:
        assert torch.equal(dy2, dyg)
        check(dg, dyg64.sum(2), dyg64.abs().sum(2), torch.float32, "dgate")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,C_,L,layout", [
    (2, 8, 64, "contiguous"),    # the vector kernel
    (3, 30, 63, "contiguous"),   # C*L = 1890: not a multiple of 4 or 8 -> torch
    (2, 36, 63, "contiguous"),   # C*L = 2268: the fp32 kernel; 16-bit -> torch
    (2, 8, 64, "misaligned"),    # one element into the storage -> torch
])
def test_sum4_add(dtype, B, C_, L, layout):
    """ops.sum4_add: add + the four direction gradients of each image (x4 indexed per batch), on the kernel and on the torch fallback"""
    torch.manual_seed(B + C_ + L)
    x4, x4_64 = rnd(dtype, B, 4, C_, L)
    add, add64 = rnd(dtype, B, C_, L)
    if layout == "misaligned":
        add = misaligned(add)
    out = ops.sum4_add(x4, add)
    check(out, add64 + x4_64.sum(1), add64.abs() + x4_64.abs().sum(1), dtype, "sum4_add")


# ----------------------------------------------------------------------------- 1x1-conv weight gradient
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,M,Kc,L", [(2, 70, 40, 96), (3, 16, 130, 520), (2, 24, 20, 63)])  # M, K tails; pixel splits; L % 8 != 0
@pytest.mark.parametrize("per_batch,with_bias,prefill", [(False, False, False), (False, True, True), (True, True, False), (True, False, True)])
def test_pixlin_wgrad(dtype, B, M, Kc, L, per_batch, with_bias, prefill):
    """ops.pixlin_wgrad: dW = sum_{b,p} dy x^T (ADDED into `out`), dbias = sum_{b,p} dy (added), per image or summed; the mma.sync
    kernel (16-bit, 16 B aligned rows) and the torch fallback (fp32, or L % 8 != 0) hold the same fp32 contract"""
    torch.manual_seed(B * 3 + M + Kc + L)
    dy = offset_view(torch.randn(B, M, L, device="cuda").to(dtype), 8)  # a channel-offset view, like d z_pre in dxz
    x, x64 = rnd(dtype, B, Kc, L)
    dy64 = dy.double().cpu()
    shape = (B, M, Kc) if per_batch else (M, Kc)
    out = torch.randn(shape, device="cuda") if prefill else torch.zeros(shape, device="cuda")
    pre = out.double().cpu()
    dbias = torch.randn(M, device="cuda") if with_bias else None
    pre_b = dbias.double().cpu() if with_bias else None
    got = ops.pixlin_wgrad(dy, x, per_batch=per_batch, out=out, dbias=dbias)
    assert got.data_ptr() == out.data_ptr()
    ref = torch.einsum("bmp,bkp->bmk", dy64, x64)
    S = torch.einsum("bmp,bkp->bmk", dy64.abs(), x64.abs())
    if not per_batch:
        ref, S = ref.sum(0), S.sum(0)
    check(got, pre + ref, pre.abs() + S, torch.float32, "dW")
    if with_bias:
        check(dbias, pre_b + dy64.sum((0, 2)), pre_b.abs() + dy64.abs().sum((0, 2)), torch.float32, "dbias")


# ----------------------------------------------------------------------------- per-step weight preparation
@pytest.mark.parametrize("dtype", DTYPES)
def test_prep_block_weights(dtype):
    """vmb_prep_block_weights, one launch of every job type: 0 convert and 1 convert + transpose (padding columns zero) and 4 flipped
    taps bit for bit; 3 A = -exp and 2 the folded x_proj / dt_proj matrix and its transpose within fp32 rounding of float64"""
    torch.manual_seed(1)
    C_, R, N, M0, K0 = 30, 2, 16, 37, 21
    Mb = 4 * (C_ + 2 * N)
    p16 = lambda n: (n + 15) // 16 * 16
    src = torch.randn(M0, K0, device="cuda")
    xw, dtw = torch.randn(4, R + 2 * N, C_, device="cuda"), torch.randn(4, C_, R, device="cuda")
    A_logs, taps = torch.randn(4 * C_, N, device="cuda"), torch.randn(C_, 9, device="cuda")
    fill = lambda *s, dt=dtype: torch.full(s, 7.0, device="cuda", dtype=dt)  # the kernel must overwrite padding too
    d0, d1, big, bigT = fill(M0, p16(K0)), fill(K0, p16(M0)), fill(Mb, p16(C_)), fill(C_, p16(Mb))
    dA, dflip = fill(4 * C_, N, dt=torch.float32), fill(C_, 9, dt=torch.float32)
    ops.prep_block_weights([(0, src, None, d0, None, M0, K0, 0, p16(K0), 0), (1, src, None, d1, None, M0, K0, 0, p16(M0), 0),
                            (2, xw, dtw, big, bigT, C_, R, 2 * N, p16(C_), p16(Mb)), (3, A_logs, None, dA, None, 4 * C_, N, 0, 0, 0),
                            (4, taps, None, dflip, None, C_, 9, 0, 0, 0)], dtype)
    assert torch.equal(d0[:, :K0], src.to(dtype)) and not d0[:, K0:].any()
    assert torch.equal(d1[:, :M0], src.t().to(dtype)) and not d1[:, M0:].any()
    assert torch.equal(dflip, taps.flip(-1))
    a64 = A_logs.double().cpu()
    check(dA, -a64.exp(), a64.exp(), torch.float32, "A = -exp(A_logs)")
    xw64, dtw64 = xw.double().cpu(), dtw.double().cpu()
    ref = torch.cat([torch.cat([dtw64[k] @ xw64[k, :R], xw64[k, R:]], 0) for k in range(4)], 0)
    S = torch.cat([torch.cat([dtw64[k].abs() @ xw64[k, :R].abs(), xw64[k, R:].abs()], 0) for k in range(4)], 0)
    check(big[:, :C_], ref, S, dtype, "folded x_proj / dt_proj")
    assert torch.equal(bigT[:, :Mb], big[:, :C_].t()) and not big[:, C_:].any() and not bigT[:, Mb:].any()


# ----------------------------------------------------------------------------- the fused training step at odd geometries
@pytest.mark.parametrize("variant,dim,H,W", [
    ("sisr", 32, 7, 9), ("sisr", 32, 10, 12), ("mamber32", 32, 7, 9), ("mamber32", 32, 10, 12),  # odd L; W % 8 != 0
    ("sisr", 30, 7, 9), ("mamber32", 30, 7, 9),  # C*L = 1890: sum4_add off its vector kernel
])
def test_block_fused_training_path_at_odd_geometries(variant, dim, H, W):
    """fp32 fused training step (the per-pixel / scalar kernel paths above, inside a block) vs torch autograd over the composed path"""
    torch.manual_seed(dim + H * W)
    blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant=variant).cuda()
    x = torch.randn(2, dim, H, W, device="cuda")
    dout = torch.randn(2, dim, H, W, device="cuda")
    grads = {}
    try:
        for path in ("fused", "compose"):
            archs.set_train_path(path)
            blk.zero_grad(set_to_none=True)
            xx = x.clone().requires_grad_()
            y = blk(xx)
            if path == "fused":
                assert "Tail" in type(y.grad_fn).__name__, "the fused training path did not run"
            y.backward(dout)
            grads[path] = [xx.grad.clone()] + [p.grad.clone() for p in blk.parameters()]
    finally:
        archs.set_train_path("fused")
    names = ["x"] + [n for n, _ in blk.named_parameters()]
    for n, a, b in zip(names, grads["fused"], grads["compose"]):
        tol = 2e-2 if n.endswith("conv_cout.bias") else 3e-3 * float(b.abs().max().clamp_min(1e-6)) + 1e-5
        assert float((a - b).abs().max()) <= tol, (n, float((a - b).abs().max()), float(b.abs().max()))
