"""The selective-scan kernels -- flat (vmb_selective_scan_fwd / _bwd) and direction-aware (vmb_selective_scan_fwd_grouped /
_bwd_grouped) -- against the float64 oracle (oracle/cscan.py), element by element, on every launch configuration of their pickers:

    |got - ref| <= u_out * |ref|  +  16 * eps_fp32 * S  +  TINY      (S: the oracle's magnitude, oracle/scan_bound.py)

with S of dA, dD and ddelta_bias, dB and dC widened by the P fp32 additions of partial sums that reach each of them.

fwd_path() / bwd_path() restate the pickers of csrc/scan_fwd_tma.cu (scan_fwd_tma_pick), csrc/scan_fwd.cu (pick_cfg),
csrc/scan_bwd.cu (pick_rb_bwd), csrc/scan_bwd_tma.cu (bwd_tma_ss, grouped_ss) and the vec_ok rules of csrc/api.cu.  A path label
is the kernel family (gen / tma / grp-tma) with RB and WPC or SS, the MODE (0 plain, 1 checkpoints, 2 grouped, 3 grouped +
checkpoints), det / atomic, and the in / out dtypes.  Each case names the path it intends and asserts that the mirror agrees;
test_every_path_is_covered asserts that the cases reach every label.  The knobs VMB_SCAN_TMA, VMB_SCAN_SS, VMB_SCAN_RB,
VMB_SCAN_WPC, VMB_SCAN_BWD_TMA, VMB_SCAN_SS_BWD and VMB_SCAN_RB_BWD are read on every launch, so monkeypatch.setenv forces a path
in this process.  The grouped oracle flips the reversed groups into sequence order, runs the flat oracle with one group per
direction and flips the results back.  The worst err / bound per path is printed at the end of the module.
"""
import os
from collections import namedtuple

import pytest
import torch

from oracle import cscan
from oracle import scan_bound as SB
from tests.test_scan_gpu import make_inputs
from vmambair_b200 import ops

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
DTYPES = [F32, BF16, F16]
T, CKPT = 16, 64  # kScanT, kScanCkpt (csrc/scan_params.h)
RATIOS = {}  # path -> largest err / bound seen
KNOBS = ("VMB_SCAN_TMA", "VMB_SCAN_SS", "VMB_SCAN_RB", "VMB_SCAN_WPC", "VMB_SCAN_BWD_TMA", "VMB_SCAN_SS_BWD", "VMB_SCAN_RB_BWD",
         "VMB_SCAN_BWD_TMA_F32")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dname(dt):
    return {F32: "f32", BF16: "bf16", F16: "f16"}[dt]


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    cscan.use_host_threads()
    yield
    if RATIOS:
        print("\nlargest err / bound per path: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(RATIOS.items())))


@pytest.fixture(autouse=True)
def _clean_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def _env(name, default=None):
    v = os.environ.get(name)
    return default if v is None else int(v)


# ============================================================================= path mirror
def fwd_path(batch, dim, L, N, G, dtype, vec_ok, grouped, ckpt, out_f32=False):
    """label of the forward launch (scan_fwd_launch)"""
    npad, rpg, rows = -(-N // 16) * 16, dim // G, batch * dim
    mode = (2 if grouped else 0) + (1 if ckpt else 0)
    io = dname(dtype) + ("-f32out" if out_f32 else "")
    # scan_fwd_tma_pick
    tma = _env("VMB_SCAN_TMA", 1) != 0 and vec_ok and npad == 16 and L >= 512 and not (grouped and N != 16)
    if tma:
        ss = 1
        while ss < 4 and rows // 2 * ss < 8 * sms():
            ss <<= 1
        if _env("VMB_SCAN_SS") in (1, 2, 4):
            ss = _env("VMB_SCAN_SS")
        if rpg % (2 * 4 // ss) == 0:
            return f"fwd-tma-ss{ss}-m{mode}-{io}"
    if grouped:
        assert vec_ok and npad == 16, "the grouped generic forward needs aligned rows and dstate <= 16"
    # pick_cfg
    rb = 1 if rows < 1536 else 2 if rows < 8192 else 4 if rows < 32768 else 8
    while rb > 1 and rpg % rb:
        rb >>= 1
    while rb < 8 and rpg % (rb * 2) == 0 and (32 // rb) * T >= 2 * L:
        rb *= 2
    e = _env("VMB_SCAN_RB", 0)
    if 0 < e <= 8 and e & (e - 1) == 0 and rpg % e == 0:
        rb = e
    if grouped and ckpt and rb > 2:
        rb = 2
    wpc = 4
    while wpc > 1 and rpg % (rb * wpc):
        wpc >>= 1
    e = _env("VMB_SCAN_WPC", 0)
    if e > 0 and e & (e - 1) == 0 and rpg % (rb * e) == 0 and e <= 4:
        wpc = e
    return f"fwd-gen-rb{rb}-wpc{wpc}-m{mode}-{io}"


def bwd_tma_ss(batch, dim):
    rows, ss = batch * dim, 1
    while ss < 4 and rows // (2 * 4 // ss) * 2 <= 2 * sms():
        ss <<= 1
    if _env("VMB_SCAN_SS_BWD") in (1, 2, 4):
        ss = _env("VMB_SCAN_SS_BWD")
    return ss


def bwd_path(batch, dim, L, N, G, dtype, vec_ok, grouped, ckpt, det, dout_f32=False):
    """(label, rows per contributor) of the backward launch (scan_bwd_launch / scan_bwd_grouped_launch)"""
    npad, rpg = -(-N // 16) * 16, dim // G
    io = dname(dtype) + ("-f32dout" if dout_f32 else "")
    d = "det" if det else "atomic"
    if grouped:  # grouped_ss
        ss = bwd_tma_ss(batch, dim)
        while ss < 4 and rpg % (2 * 4 // ss):
            ss <<= 1
        return f"bwd-grp-tma-ss{ss}-{d}-{io}", 8 // ss
    tma = (_env("VMB_SCAN_BWD_TMA", 1) != 0 and not (dtype == F32 and _env("VMB_SCAN_BWD_TMA_F32", 1) == 0) and vec_ok and
           npad == 16 and L >= 512 and ckpt)
    if tma:
        ss = bwd_tma_ss(batch, dim)
        if rpg % (2 * 4 // ss) == 0:
            return f"bwd-tma-ss{ss}-{d}-{io}", 8 // ss
    rb = 0
    e = _env("VMB_SCAN_RB_BWD", 0)
    if 0 < e <= 8 and e & (e - 1) == 0 and rpg % e == 0:
        rb = e
    if not rb:
        rows = batch * dim
        rb = 2 if rows < 1536 else 4 if rows < 6144 else 8
        while rb > 1 and rpg % rb:
            rb >>= 1
    return f"bwd-gen-rb{rb}-{d}-{io}", rb


def aligned16(t):
    return t.data_ptr() % 16 == 0


def flat_vec_ok(ts, dtype, f32_ts=()):
    """api.cu: 16 B aligned base pointers, batch / row strides in whole 16 B vectors (in each tensor's own element type)"""
    v = 16 // torch.tensor([], dtype=dtype).element_size()
    ok = all(aligned16(t) and all(s % v == 0 for s in t.stride()[:-1]) for t in ts)
    return ok and all(aligned16(t) and all(s % 4 == 0 for s in t.stride()[:-1]) for t in f32_ts)


def all_paths():
    """every label the pickers can produce"""
    out = set()
    for dt in DTYPES:
        ios = [dname(dt)] + ([dname(dt) + "-f32out"] if dt != F32 else [])
        gios = [dname(dt)] + ([dname(dt) + "-f32dout"] if dt != F32 else [])
        for io in ios:
            out |= {f"fwd-gen-rb{rb}-wpc{w}-m{m}-{io}" for rb in (1, 2, 4, 8) for w in (1, 2, 4) for m in (0, 1)}
            out |= {f"fwd-tma-ss{ss}-m{m}-{io}" for ss in (1, 2, 4) for m in (0, 1)}
        out |= {f"fwd-gen-rb{rb}-wpc{w}-m2-{dname(dt)}" for rb in (1, 2, 4, 8) for w in (1, 2, 4)}
        out |= {f"fwd-gen-rb{rb}-wpc{w}-m3-{dname(dt)}" for rb in (1, 2) for w in (1, 2, 4)}
        out |= {f"fwd-tma-ss{ss}-m{m}-{dname(dt)}" for ss in (1, 2, 4) for m in (2, 3)}
        for d in ("det", "atomic"):
            for io in gios:
                out |= {f"bwd-gen-rb{rb}-{d}-{io}" for rb in (1, 2, 4, 8)}
                out |= {f"bwd-tma-ss{ss}-{d}-{io}" for ss in (1, 2, 4)}
            out |= {f"bwd-grp-tma-ss{ss}-{d}-{dname(dt)}" for ss in (1, 2, 4)}
    return out


# ============================================================================= cases
# kind: "flat" / "grouped"; bwd: also run the backward on the forward's checkpoints (None: forward only, else det 0 / 1)
# layout: "dense" / "strided" (u, delta, dout channel slices of wider buffers, B and C halves of one (B, G, 2N, L) buffer) /
#         "misaligned" (flat: u one element into its storage -> no 16 B rows)
# env: knobs; expect: (forward label, backward label or None) the case is written for, None where the natural path is recorded
Case = namedtuple("Case", "kind dtype b D L N G env bwd layout out_f32 model expect")
Case.__new__.__defaults__ = ("dense", False, False, None)


def case_id(c):
    env = "-".join(f"{k[9:].lower()}{v}" for k, v in sorted(c.env.items()))
    return (f"{c.kind}-{dname(c.dtype)}{'-f32out' if c.out_f32 else ''}-b{c.b}-D{c.D}-L{c.L}-N{c.N}-G{c.G}-{c.layout}"
            f"{'-model' if c.model else ''}{'' if c.bwd is None else ('-det' if c.bwd else '-atomic')}{'-' + env if env else ''}")


def matrix():
    cs = []
    Ls = [520, 1000, 4104, 512]
    Ns = [16, 15, 17, 1]
    for dt in DTYPES:
        ofs = [False] + ([True] if dt != F32 else [])
        for of in ofs:
            io = dname(dt) + ("-f32out" if of else "")
            gio = dname(dt) + ("-f32dout" if of else "")
            # generic forward: every (RB, WPC), MODE 0 and 1; MODE 1 runs the generic backward at the same RB
            i = 0
            for rb in (1, 2, 4, 8):
                for wpc in (1, 2, 4):
                    for ck in (0, 1):
                        i += 1
                        det = (rb + wpc + ck) % 2
                        L, N = (Ls[i % 4], Ns[i % 4]) if not of else (1000, 16)
                        env = dict(VMB_SCAN_TMA=0, VMB_SCAN_RB=rb, VMB_SCAN_WPC=wpc, VMB_SCAN_BWD_TMA=0, VMB_SCAN_RB_BWD=rb)
                        exp_b = f"bwd-gen-rb{rb}-{'det' if det else 'atomic'}-{gio}" if ck else None
                        cs.append(Case("flat", dt, 1, 64, L, N, 2, env, det if ck else None, "strided" if i % 3 == 0 else "dense",
                                       of, i % 5 == 0, (f"fwd-gen-rb{rb}-wpc{wpc}-m{ck}-{io}", exp_b)))
            # generic backward with the atomic / det mode the loop above did not give each RB
            for rb in (1, 2, 4, 8):
                for det in (0, 1):
                    env = dict(VMB_SCAN_TMA=0, VMB_SCAN_RB=2, VMB_SCAN_WPC=1, VMB_SCAN_BWD_TMA=0, VMB_SCAN_RB_BWD=rb)
                    cs.append(Case("flat", dt, 2, 32, 65 if rb % 2 else 511, 16, 4, env, det, "dense", of, False,
                                   (f"fwd-gen-rb2-wpc1-m1-{io}", f"bwd-gen-rb{rb}-{'det' if det else 'atomic'}-{gio}")))
            # TMA forward: SS 1 / 2 / 4, MODE 0 and 1; MODE 1 runs the TMA backward at the same SS, atomic and det
            for ss in (1, 2, 4):
                env = dict(VMB_SCAN_SS=ss, VMB_SCAN_SS_BWD=ss)
                L = (512, 4104, 1000)[ss // 2]
                cs.append(Case("flat", dt, 2, 48, L, 16, 2, env, None, "dense", of, ss == 2, (f"fwd-tma-ss{ss}-m0-{io}", None)))
                for det in (0, 1):
                    cs.append(Case("flat", dt, 2, 48, (520, 4104)[det], 16, 2, env, det, "strided" if det else "dense", of,
                                   ss == 4, (f"fwd-tma-ss{ss}-m1-{io}", f"bwd-tma-ss{ss}-{'det' if det else 'atomic'}-{gio}")))
        # grouped, generic forward: every (RB, WPC) at MODE 2, RB <= 2 at MODE 3 (clamped there: RB 4 / 8 are not instantiated)
        for rb in (1, 2, 4, 8):
            for wpc in (1, 2, 4):
                env = dict(VMB_SCAN_TMA=0, VMB_SCAN_RB=rb, VMB_SCAN_WPC=wpc)
                L = (64, 520, 1000)[(rb + wpc) % 3]
                cs.append(Case("grouped", dt, 1, 4 * 32, L, 16 if wpc != 2 else 15, 4, env, None, "strided", False, rb == 4,
                               (f"fwd-gen-rb{rb}-wpc{wpc}-m2-{dname(dt)}", None)))
                if rb <= 4:
                    rbe = min(rb, 2)
                    det = (rb + wpc) % 2
                    ss = 4 if wpc == 4 else 2
                    env = dict(env, VMB_SCAN_SS_BWD=ss)
                    cs.append(Case("grouped", dt, 1, 4 * 32, (520, 1000, 64)[wpc // 2], 16, 4, env, det, "strided", False, False,
                                   (f"fwd-gen-rb{rbe}-wpc{wpc}-m3-{dname(dt)}", f"bwd-grp-tma-ss{ss}-{'det' if det else 'atomic'}-{dname(dt)}")))
        # grouped, TMA forward: SS 1 / 2 / 4, MODE 2 and 3, with the grouped backward at the same SS (atomic and det)
        for ss in (1, 2, 4):
            env = dict(VMB_SCAN_SS=ss, VMB_SCAN_SS_BWD=ss)
            cs.append(Case("grouped", dt, 1, 4 * 16, (512, 1000, 4104)[ss // 2], 16, 4, env, None, "strided", False, ss == 1,
                           (f"fwd-tma-ss{ss}-m2-{dname(dt)}", None)))
            for det in (0, 1):
                cs.append(Case("grouped", dt, 2, 4 * 8, (4104, 520)[det], 16, 4, env, det, "strided", False, det == 1,
                               (f"fwd-tma-ss{ss}-m3-{dname(dt)}", f"bwd-grp-tma-ss{ss}-{'det' if det else 'atomic'}-{dname(dt)}")))
        # the grouped backward at short L (always the TMA kernel, zero-filled boxes past the end) and its natural SS
        for det in (0, 1):
            cs.append(Case("grouped", dt, 1, 4 * 6, 64, 16, 4, {}, det, "strided", False, False, None))
            cs.append(Case("grouped", dt, 3, 4 * 6, 8 if dt != F32 else 4, 16, 4, {}, det, "strided", False, True, None))
    return cs


def edges():
    """every declared edge on its natural path: L across the TMA tail, the checkpoint boundary and the 256-position chunk (+ 8);
    dstate up to the declared 256; odd rows per group; strided and misaligned rows; batch 1 and a batch that reaches SS = 1"""
    cs = []
    Ns = [1, 15, 16, 17, 64, 256]
    for i, L in enumerate([1, 63, 64, 65, 511, 512, 520, 1000, 4104]):
        dt = DTYPES[i % 3]
        cs.append(Case("flat", dt, 2, 24, L, Ns[i % 6], 2, {}, i % 2, "strided" if i % 2 else "dense", False, i % 4 == 0))
    for i, N in enumerate(Ns):
        dt = DTYPES[(i + 1) % 3]
        cs.append(Case("flat", dt, 1, 16, 1000 if N < 64 else 300, N, 2, {}, i % 2, "dense", dt != F32 and i % 2 == 0, i % 3 == 0))
    for rb in (1, 2, 4, 8):  # dstate 256 on every generic RB, forward and backward
        cs.append(Case("flat", BF16, 1, 16, 200, 256, 2, dict(VMB_SCAN_RB=rb, VMB_SCAN_RB_BWD=rb), 1, "dense", False, True, None))
    cs += [Case("flat", BF16, 2, 18, 1000, 16, 3, {}, 0, "dense", False, False, None),         # 6 rows per group: TMA at SS 4
           Case("flat", F16, 1, 9, 1000, 16, 3, {}, 1, "strided", False, False, None),         # 3 rows per group (odd): generic
           Case("flat", F32, 1, 15, 4104, 16, 5, {}, 0, "dense", False, True, None),           # 3 rows per group, long
           Case("flat", BF16, 2, 16, 1000, 16, 2, {}, 1, "misaligned", False, False, None),    # no 16 B rows: generic
           Case("flat", F16, 2, 16, 1001, 16, 2, {}, 0, "dense", False, False, None),          # odd L: no 16 B rows
           Case("flat", BF16, 8, 384, 1000, 16, 4, {}, 1, "dense", False, True, None),         # SS = 1 by the SM count
           Case("grouped", BF16, 8, 4 * 96, 1000, 16, 4, {}, 0, "strided", False, True, None)]
    return cs


CASES = matrix() + edges()


# ============================================================================= running one case
def _place(t, layout, extra=8):
    """t (B, R, L) in the requested layout: dense, or channels [extra, extra + R) of a wider buffer"""
    if layout != "strided":
        return t.contiguous()
    buf = torch.randn(t.shape[0], t.shape[1] + extra, t.shape[2], device=t.device).to(t.dtype)
    buf[:, extra:] = t
    return buf[:, extra:]


def _misaligned(t):
    flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = flat[1:].view(t.shape)
    v.copy_(t)
    return v


def check(got, ref, S, dtype, what, paths):
    got = got.detach().double().cpu()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    b = SB.bound(ref, S, dtype)
    r = err / b.clamp_min(1e-300)
    worst = float(r.max()) if r.numel() else 0.0
    for p in paths:
        RATIOS[p] = max(RATIOS.get(p, 0.0), worst)
    bad = ~(err <= b)
    if bad.any():
        i = int(r.flatten().argmax())
        idx = [int(x) for x in torch.unravel_index(torch.tensor(i), r.shape)]
        raise AssertionError(f"{what} [{'/'.join(paths)}]: {int(bad.sum())} of {err.numel()} elements out of bound; worst at {idx}: "
                             f"got {float(got.flatten()[i])}, ref {float(ref.flatten()[i])}, bound {float(b.flatten()[i])}")


def _inputs(c, seed):
    b, D, L, N, G = c.b, c.D, c.L, c.N, c.G
    u, delta, A, Bm, Cm, Dv, bias = make_inputs(b, D, L, N, G, c.dtype, seed=seed, model_like=c.model)
    g = torch.Generator().manual_seed(seed + 1)
    dout = torch.randn(b, D, L, generator=g)
    dout = dout if c.out_f32 else dout.to(c.dtype)
    return u, delta, A, Bm, Cm, Dv, bias, dout


def check_grads(got, ref, S, dtype, P_bc, P_prm, paths):
    names = ("du", "ddelta", "dA", "dB", "dC", "dD", "dbias")
    for k, (n, x, y, s) in enumerate(zip(names, got, ref, S)):
        if n in ("dB", "dC"):
            s = SB.atomic(s, P_bc)
        elif n in ("dA", "dD", "dbias"):
            s = SB.atomic(s, P_prm)
        check(x, y, s, dtype if k in (0, 1, 3, 4) else F32, n, paths)


def run_flat(c, monkeypatch, seed):
    for k, v in c.env.items():
        monkeypatch.setenv(k, str(v))
    u, delta, A, Bm, Cm, Dv, bias, dout = _inputs(c, seed)
    sp = True
    dev = "cuda"
    if c.layout == "strided":
        ud, dd, gd = (_place(t.to(dev), "strided") for t in (u, delta, dout))
        bc = torch.cat([Bm, Cm], 2).to(dev)  # (B, G, 2N, L): B and C are its halves, as the training path's bc buffer
        Bd, Cd = bc[:, :, :c.N], bc[:, :, c.N:]
    else:
        ud, dd, gd, Bd, Cd = (t.to(dev).contiguous() for t in (u, delta, dout, Bm, Cm))
        if c.layout == "misaligned":
            ud = _misaligned(ud)
    Ad, Dd, bd = A.to(dev), Dv.to(dev), bias.to(dev)
    need_ck = c.bwd is not None
    out, ck = ops.selective_scan_fwd(ud, dd, Ad, Bd, Cd, Dd, bd, sp, need_ckpt=need_ck, out_float=c.out_f32)
    vec = flat_vec_ok([ud, dd, Bd, Cd], c.dtype, [out] if c.out_f32 else []) and (c.out_f32 or flat_vec_ok([out], c.dtype))
    fp = fwd_path(c.b, c.D, c.L, c.N, c.G, c.dtype, vec, False, need_ck, c.out_f32)
    if c.expect is not None:
        assert fp == c.expect[0], (fp, c.expect[0])
    ref, S = cscan.scan_fwd_mag(u, delta, A, Bm, Cm, Dv, bias, sp)
    check(out, ref, S, F32 if c.out_f32 else c.dtype, "out", [fp])
    if c.bwd is None:
        return
    grads = ops.selective_scan_bwd(ud, dd, Ad, Bd, Cd, Dd, bd, gd, ck, sp, dout_float=c.out_f32, deterministic=bool(c.bwd))
    bvec = vec and flat_vec_ok([gd], F32 if c.out_f32 else c.dtype)
    bp, per = bwd_path(c.b, c.D, c.L, c.N, c.G, c.dtype, bvec, False, True, c.bwd, c.out_f32)
    if c.expect is not None and c.expect[1] is not None:
        assert bp == c.expect[1], (bp, c.expect[1])
    g, s = cscan.scan_bwd_mag(u, delta, A, Bm, Cm, Dv, bias, dout, sp)
    check_grads(grads, g, s, c.dtype, (c.D // c.G) // per, 4 * c.b, [bp])


def _seq(t, rev):
    return t.flip(-1) if rev else t


def run_grouped(c, monkeypatch, seed):
    """four directions like the OSS block: 0 / 2 read x, 1 / 3 its (W, H) transpose; 2 / 3 walk backwards.  delta, B and C are
    channel slices of one (B, 2, R + 2N, L) buffer per source, as the block's fused x_proj / dt_proj GEMM writes them."""
    for k, v in c.env.items():
        monkeypatch.setenv(k, str(v))
    G, R, L, N, b = c.G, c.D // c.G, c.L, c.N, c.b
    u, delta, A, Bm, Cm, Dv, bias, dout = _inputs(c, seed)  # sequence order, one group per direction
    revs = [0, 0, 1, 1][:G] if G >= 3 else [0, 1][:G]
    src = [g % 2 for g in range(G)]  # source tensor of each direction (0: x, 1: the transposed copy)
    slot = [g // 2 for g in range(G)]
    dev = "cuda"
    us_mem = [_seq(u[:, g * R:(g + 1) * R], revs[g]) for g in range(G)]  # each direction's operands in its source's memory order
    # the directions that share a source share its u: make the reversed one the flipped copy of the forward one
    for g in range(G):
        if slot[g] == 1:
            us_mem[g] = us_mem[g - 2]
            u[:, g * R:(g + 1) * R] = _seq(us_mem[g], revs[g])
    x = [torch.zeros(b, R, L, dtype=c.dtype) for _ in range(2)]
    big = [torch.zeros(b, 2, R + 2 * N + 8, L, dtype=c.dtype) for _ in range(2)]
    for g in range(G):
        x[src[g]].copy_(us_mem[g])
        big[src[g]][:, slot[g], :R] = _seq(delta[:, g * R:(g + 1) * R], revs[g])
        big[src[g]][:, slot[g], R:R + N] = _seq(Bm[:, g], revs[g])
        big[src[g]][:, slot[g], R + N:R + 2 * N] = _seq(Cm[:, g], revs[g])
    xd = [t.to(dev) for t in x]
    bigd = [t.to(dev) for t in big]
    us = [xd[src[g]] for g in range(G)]
    ds = [bigd[src[g]][:, slot[g], :R] for g in range(G)]
    Bs = [bigd[src[g]][:, slot[g], R:R + N] for g in range(G)]
    Cs = [bigd[src[g]][:, slot[g], R + N:R + 2 * N] for g in range(G)]
    Ad, Dd, bd = A.to(dev), Dv.to(dev), bias.to(dev)
    need_ck = c.bwd is not None
    r = ops.selective_scan_fwd_grouped(us, ds, Bs, Cs, revs, Ad, Dd, bd, True, need_ckpt=need_ck)
    ys, ck = r if need_ck else (r, None)
    vec = flat_vec_ok(us + ds + Bs + Cs + [ys], c.dtype) and L % (16 // ys.element_size()) == 0
    fp = fwd_path(b, c.D, L, N, G, c.dtype, vec, True, need_ck)
    if c.expect is not None:
        assert fp == c.expect[0], (fp, c.expect[0])
    ref, S = cscan.scan_fwd_mag(u, delta, A, Bm, Cm, Dv, bias, True)
    ref, S = ref.view(b, G, R, L), S.view(b, G, R, L)
    for g in range(G):
        check(ys[:, g], _seq(ref[:, g], revs[g]), _seq(S[:, g], revs[g]), c.dtype, f"out[{g}]", [fp])
    if c.bwd is None:
        return
    gbuf = torch.randn(b, G, R + 8, L).to(c.dtype)
    for g in range(G):
        gbuf[:, g, 8:] = _seq(dout[:, g * R:(g + 1) * R], revs[g])
    gd = gbuf.to(dev)
    douts = [gd[:, g, 8:] for g in range(G)]
    dus, dds, dA, dBs, dCs, dD, dbias = ops.selective_scan_bwd_grouped(us, ds, Bs, Cs, douts, revs, Ad, Dd, bd, ck, True,
                                                                        deterministic=bool(c.bwd))
    bp, per = bwd_path(b, c.D, L, N, G, c.dtype, True, True, True, c.bwd)
    if c.expect is not None and c.expect[1] is not None:
        assert bp == c.expect[1], (bp, c.expect[1])
    gr, s = cscan.scan_bwd_mag(u, delta, A, Bm, Cm, Dv, bias, dout, True)
    P_bc, P_prm = R // per, 4 * b
    rows = lambda t, g: t[:, g * R:(g + 1) * R]
    for g in range(G):
        rv = revs[g]
        check(dus[g], _seq(rows(gr[0], g), rv), _seq(rows(s[0], g), rv), c.dtype, f"du[{g}]", [bp])
        check(dds[g], _seq(rows(gr[1], g), rv), _seq(rows(s[1], g), rv), c.dtype, f"ddelta[{g}]", [bp])
        check(dBs[g], _seq(gr[3][:, g], rv), SB.atomic(_seq(s[3][:, g], rv), P_bc), c.dtype, f"dB[{g}]", [bp])
        check(dCs[g], _seq(gr[4][:, g], rv), SB.atomic(_seq(s[4][:, g], rv), P_bc), c.dtype, f"dC[{g}]", [bp])
    check(dA, gr[2], SB.atomic(s[2], P_prm), F32, "dA", [bp])
    check(dD, gr[5], SB.atomic(s[5], P_prm), F32, "dD", [bp])
    check(dbias, gr[6], SB.atomic(s[6], P_prm), F32, "dbias", [bp])


def run_case(c, monkeypatch, seed):
    (run_grouped if c.kind == "grouped" else run_flat)(c, monkeypatch, seed)


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_scan_path(c, monkeypatch):
    run_case(c, monkeypatch, seed=1 + CASES.index(c))


def test_every_path_is_covered():
    """the case list reaches every label of the mirror's table (predicted with each case's knobs, as the run asserts)"""
    reached = set()
    for c in CASES + BENCH:
        if c.expect is not None:
            reached |= {p for p in c.expect if p is not None}
    missing = all_paths() - reached
    assert not missing, sorted(missing)


# ============================================================================= the scans the bench launches
def bench_sites():
    """the scans of the bench's default net (MambaSISR6, class defaults), from its modules: inference at the engine's per-launch
    batch (8: bench.py's InferenceEngine has chains = lowres_chains = 1 by default, so every level runs the whole batch) through
    the direction-aware forward; the training step at B = 4 through the flat forward with checkpoints and its backward"""
    from vmambair_b200 import archs
    net = archs.MambaSISR6()
    H = 64
    sites = {}
    for stage, hw in [(net.encoder_level1, H), (net.encoder_level2, H // 2), (net.encoder_level3, H // 4), (net.latent, H // 8),
                      (net.decoder_level3, H // 4), (net.decoder_level2, H // 2), (net.decoder_level1, H), (net.refinement, H)]:
        a = stage[0].attn
        sites[(a.d_inner, a.d_state, hw * hw)] = None
    cs = []
    for (C_, N, L) in sites:
        cs.append(Case("grouped", BF16, 8, 4 * C_, L, N, 4, {}, None, "strided", False, True, None))
        cs.append(Case("flat", BF16, 4, 4 * C_, L, N, 4, {}, 0, "dense", False, True, None))
    return cs


BENCH = bench_sites()


def _natural(c):
    """the path a bench site takes on this GPU, by the mirror (no knob set)"""
    rows_vec = c.L % 8 == 0
    fp = fwd_path(c.b, c.D, c.L, c.N, c.G, c.dtype, rows_vec, c.kind == "grouped", c.bwd is not None)
    bp = None if c.bwd is None else bwd_path(c.b, c.D, c.L, c.N, c.G, c.dtype, rows_vec, False, True, c.bwd)[0]
    return fp, bp


@pytest.mark.parametrize("c", BENCH, ids=case_id)
def test_bench_site(c, monkeypatch):
    run_case(c._replace(expect=_natural(c)), monkeypatch, seed=101 + BENCH.index(c))
