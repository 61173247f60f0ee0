"""vmb_pixlin (every 1x1 convolution, in inference and training) and vmb_conv3x3 (every dense 3x3 convolution of the U-Net trunk)
against their float64 references (oracle/gemm_ref.py), element by element, on every dispatch path of their launchers.

    |got - ref| <= u_out * |ref|  +  16 * eps_fp32 * S  +  T  +  TINY      (T: the prologue's rounding straddle, see gemm_ref)

Neither launcher has a path switch: the path follows from the SM count, the grid, the shared-memory size, pointer alignment and
stride divisibility.  pixlin_path() / conv_path() mirror csrc/pixlin.cu (pixlin_launch, kstream_applicable, launch_mma, launch2) and
csrc/conv3x3.cu (conv3x3_launch, launch_16, launch_tma) with vec_ok / w_vec / pair_ok of csrc/api.cu and the kernels; every case
asserts the path it intends, so that a case cannot drift onto another path when the card or a heuristic changes, and
test_every_path_is_covered asserts that the case list reaches every path.  Where two paths can take the same values they run on
the same values (check_pair: within the sum of their two bounds).

The worst err / bound per path is printed at the end of the module.  It sits just below 1 wherever a term of the bound is an exact
allowance rather than slack: the final round-to-nearest of a 16-bit output uses up to u_out * |ref|, and an x' whose fp32 and
float64 values round to neighbouring 16-bit values differs by exactly the T of that element.  The fp32 accumulation term is the
slack: the fp32 paths, which have neither, use 0.07 - 0.14 of it on the H100.
"""
import zlib
from collections import namedtuple

import pytest
import torch

from oracle import gemm_ref as G
from vmambair_b200 import ops

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
DT16 = [BF16, F16]
RATIOS = {}  # path -> largest err / bound seen (printed at the end of the module)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    if RATIOS:
        print("\nlargest err / bound per path: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(RATIOS.items())))


def check(got, ref, S, dtype, what, paths=(), T=None):
    """element-wise bound of the module docstring (all on the GPU); records the worst ratio under each path label"""
    got = got.detach().double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    b = G.bound(ref, S, dtype, T)
    r = err / b.clamp_min(1e-300)
    worst = float(r.max()) if r.numel() else 0.0
    for p in paths:
        RATIOS[p] = max(RATIOS.get(p, 0.0), worst)
    bad = ~(err <= b)
    if bad.any():
        i = int(r.flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements out of bound; worst at flat index {i}: "
                             f"got {float(got.flatten()[i])}, ref {float(ref.flatten()[i])}, bound {float(b.flatten()[i])}")
    return b


def check_pair(a, b, bound_a, bound_b, what, bitwise=False):
    """two dispatch paths on the same values: within the sum of their bounds of the float64 reference; bitwise: identical (the two
    paths issue the same mma.sync sequence in the same k order and round once, as measured on the H100)"""
    if bitwise:
        assert torch.equal(a, b), what
    assert bool(((a.detach().double() - b.detach().double()).abs() <= bound_a + bound_b).all()), what


def misaligned(t):
    """contiguous copy of t starting one element into its storage: not 16 B (nor 4 B) aligned"""
    flat = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = flat[1:].view(t.shape)
    v.copy_(t)
    return v


def aligned16(t):
    return t.data_ptr() % 16 == 0


# ============================================================================= pixlin: path mirror
PL2_KC, PL_KC_F32, KS_MT = 384, 384, 128


def ceil16(k):
    return (k + 15) // 16 * 16


def pixlin_smem(K, elt, PT=64, wtiles=2):
    kpad = ceil16(K)
    if elt == 2:
        KC = min(kpad, PL2_KC)
        return 2 * (KC * (PT + 8) + wtiles * 64 * (KC + 8)) + 4 * (8 * 16 * (PT // 4 + 4) + 1024)
    KC = min(kpad, PL_KC_F32)
    return 4 * (KC * 68 + 64 * (KC + 1) + 64 * 68 + 128)


def pixlin_vec_ok(x, out, residual, dtype, out_dtype):
    """api.cu vmb_pixlin: 16 B rows of x, out and the residual"""
    vm = max(16 // torch.tensor([], dtype=dtype).element_size(), 16 // torch.tensor([], dtype=out_dtype).element_size())
    ts = [x, out] + ([residual] if residual is not None else [])
    return all(aligned16(t) and t.stride(0) % vm == 0 and t.stride(1) % vm == 0 for t in ts) and x.shape[2] % vm == 0


def pixlin_w_vec(w, K, dtype):
    """api.cu vmb_pixlin: weight rows 16 B aligned and padded to ceil16(K)"""
    v = 16 // torch.tensor([], dtype=dtype).element_size()
    return aligned16(w) and w.stride(0) % v == 0 and w.stride(0) >= ceil16(K)


def pixlin_path(B, K, M, P, dtype, out_dtype, pro, vec_ok, w_vec):
    """the set of path labels pixlin_launch takes"""
    kpad = ceil16(K)
    if dtype == F32:
        return {"f32-resident" if kpad <= PL_KC_F32 else "f32-chunked"}
    if out_dtype == dtype and not pro and vec_ok and w_vec and K > PL2_KC and M <= 2 * KS_MT:
        return {"kstream"}
    n = sms()
    big = cdiv(P, 128) * B >= n and pixlin_smem(K, 2, 128, 2) <= 100 * 1024
    ptiles, mtiles = cdiv(P, 128 if big else 64), cdiv(M, 64)
    msplit = 1
    while msplit < mtiles and ptiles * B * msplit < 3 * n // 2:
        msplit += 1
    w_all = False
    if kpad <= PL2_KC and w_vec:
        ms = msplit
        while ms < mtiles and cdiv(mtiles, ms) * 64 * (kpad + 8) * 2 > 64 * 1024:
            ms += 1
        w_all = cdiv(mtiles, ms) * 64 * (kpad + 8) * 2 <= 64 * 1024
    paths = {"w_all" if w_all else "ring", "epi-vec" if (out_dtype != F32 and vec_ok) else "epi-patch"}
    if kpad <= PL2_KC:
        paths.add("mma-resident-PT128" if big else "mma-resident-PT64")
    else:
        paths.add("mma-chunked-vecW" if w_vec else "mma-chunked-scalarW")
    if out_dtype == F32:
        paths.add("mma-f32-out-PT128" if big else "mma-f32-out-PT64")
    return paths


PIXLIN_PATHS = {"kstream", "mma-resident-PT64", "mma-resident-PT128", "mma-chunked-vecW", "mma-chunked-scalarW", "epi-vec",
                "epi-patch", "w_all", "ring", "mma-f32-out-PT64", "mma-f32-out-PT128", "f32-resident", "f32-chunked"}


# ============================================================================= pixlin: one case
# B: an int, or "big" = the smallest batch at which the 128-pixel tiles fill the GPU (ceil(P / 128) * B >= SMs)
# x: "dense" / "offset" (channels c0.. of a wider buffer, as xz[:, C:]) / "misaligned" (one element into its storage)
# out: "dense" / "group" (out and residual are channel groups of (B, 4, M, P) buffers, as in cross_scan.py's backward)
# act: True (a SiLU range inside M) / False / (act_from, act_to); bias, res: with a bias / residual
# w: "padded" (pad_weight: vector staging) / "unpadded" (row stride K) / "misaligned" (padded, one element into its storage) /
#    "wide" (columns [0, K) of a wider random matrix: the kernel must not use the columns beyond K)
Pix = namedtuple("Pix", "dtype B K M P pro out_f32 x out w act bias res expect")
Pix.__new__.__defaults__ = (None, False, "dense", "dense", "padded", True, True, True, None)


def batch_of(c):
    return cdiv(sms(), cdiv(c.P, 128)) if c.B == "big" else c.B


def pix_id(c):
    pro = "" if not c.pro else f"-{c.pro[0]}{c.pro[1]}"
    act = "" if c.act is True else ("-noact" if c.act is False else f"-act{c.act[0]}_{c.act[1]}")
    return (f"{str(c.dtype)[6:]}-B{c.B}-K{c.K}-M{c.M}-P{c.P}{pro}{'-f32out' if c.out_f32 else ''}-x_{c.x}-out_{c.out}-w_{c.w}"
            f"{act}{'' if c.bias else '-nobias'}{'' if c.res else '-nores'}")


def make_pixlin(c, seed, with_ref=True):
    """operands of one case in their layouts + float64 reference (ref, S, T) (None unless with_ref) + the predicted paths"""
    torch.manual_seed(seed)
    dt, B, K, M, P = c.dtype, batch_of(c), c.K, c.M, c.P
    out_dtype = F32 if c.out_f32 else dt
    dev = "cuda"
    shift = torch.randn(B, 1, P, device=dev) if c.pro and c.pro[0] == "ln" else 0
    x = (torch.randn(B, K, P, device=dev) + shift).to(dt)
    w = (torch.randn(M, K, device=dev) * K ** -0.5).to(dt)
    bias = 0.5 * torch.randn(M, device=dev) if c.bias else None
    res = torch.randn(B, M, P, device=dev).to(dt) if c.res else None
    ln = gate = None
    gate_mode = 0
    if c.pro and c.pro[0] == "ln":
        ln = (c.pro[1], 1 + 0.5 * torch.randn(K, device=dev), 0.5 * torch.randn(K, device=dev) if c.pro[1] == 1 else None)
    elif c.pro and c.pro[0] == "gate":
        gate, gate_mode = torch.randn(B, K, device=dev), c.pro[1]
    act = c.act if isinstance(c.act, tuple) else ((M // 3, M - M // 4) if c.act else (0, 0))
    # layouts
    if c.x == "offset":
        buf = torch.randn(B, K + 8, P, device=dev).to(dt)
        buf[:, 8:] = x
        xx = buf[:, 8:]
    elif c.x == "misaligned":
        xx = misaligned(x)
    else:
        xx = x
    if c.out == "group":
        obuf = torch.full((B, 4, M, P), float("nan"), device=dev, dtype=out_dtype)
        out = obuf[:, 1]
        rr = None
        if res is not None:
            rbuf = torch.randn(B, 4, M, P, device=dev).to(dt)
            rbuf[:, 2] = res
            rr = rbuf[:, 2]
    else:
        out, rr = None, res
    if c.w == "padded":
        ww = ops.pad_weight(w)
    elif c.w == "unpadded":
        ww = w.contiguous()
    elif c.w == "misaligned":
        ww = misaligned(ops.pad_weight(w))
    else:  # wide
        wb = torch.randn(M, ceil16(K) + 24, device=dev).to(dt)
        wb[:, :K] = w
        ww = wb[:, :K]
    d = lambda t: None if t is None else t.double()
    ref = None
    if with_ref:
        ref = G.pixlin_ref(d(x), d(w), d(bias), d(res), None if ln is None else (ln[0], d(ln[1]), d(ln[2])), d(gate), gate_mode, act,
                           dt)
    out_probe = out if out is not None else torch.empty((B, M, P), dtype=out_dtype, device=dev)
    vec_ok = pixlin_vec_ok(xx, out_probe, rr, dt, out_dtype)
    paths = pixlin_path(B, K, M, P, dt, out_dtype, bool(c.pro), vec_ok, pixlin_w_vec(ww, K, dt))
    call = dict(x=xx, w=ww, bias=bias, residual=rr, ln=ln, gate=gate, gate_mode=gate_mode, act=act, out_dtype=out_dtype, out=out)
    return call, ref, paths, out_dtype


def run_pixlin(c, seed=0):
    call, (ref, S, T), paths, out_dtype = make_pixlin(c, seed)
    if c.expect is not None:
        assert set(c.expect) <= paths, (sorted(c.expect), sorted(paths))
    got = ops.pixlin(**call)
    if call["out"] is not None:
        assert got.data_ptr() == call["out"].data_ptr()
    b = check(got, ref, S, out_dtype, pix_id(c), paths, T)
    return got, b, paths


# ============================================================================= pixlin: the case list
def _pix_cases():
    cs = []
    for dt in DT16:
        # K-streamed GEMM: K > 384 with no prologue, M <= 256 (partial 128-row M tiles at 96 and 200), K not a multiple of 32
        for K, M, P in [(400, 96, 256), (510, 200, 512), (1021, 256, 128)]:
            cs.append(Pix(dt, 2, K, M, P, expect={"kstream"}))
        cs.append(Pix(dt, 2, 1021, 96, 128, w="wide", expect={"kstream"}))          # kw = min(w_ld, ceil16(K)) < w_ld
        cs.append(Pix(dt, 2, 510, 96, 256, act=False, out="group", expect={"kstream"}))
        # resident K on the mma kernel: PT 64 / 128 x {w_all, ring} x {vec epilogue, smem patch (misaligned x), fp32 output}
        for B, P in [(2, 256), ("big", 1024)]:
            pt = "mma-resident-PT64" if B == 2 else "mma-resident-PT128"
            for w, wm in [("padded", "w_all"), ("misaligned", "ring")]:
                cs.append(Pix(dt, B, 48, 200, P, w=w, expect={pt, wm, "epi-vec"}))
                cs.append(Pix(dt, B, 48, 200, P, w=w, x="misaligned", expect={pt, wm, "epi-patch"}))
                cs.append(Pix(dt, B, 48, 200, P, w=w, out_f32=True, expect={pt, wm, "epi-patch"}))
        cs.append(Pix(dt, "big", 144, 70, 1024, w="misaligned", expect={"mma-resident-PT128", "ring"}))  # K = 144: the PT 128 limit
        cs.append(Pix(dt, 2, 20, 70, 200, w="unpadded", expect={"mma-resident-PT64", "ring"}))
        cs.append(Pix(dt, 2, 48, 96, 256, w="wide", expect={"mma-resident-PT64", "w_all"}))
        # prologues on the resident path
        for K in [5, 20, 48, 96, 144, 384]:
            for pro in [("ln", 1), ("ln", 2), ("gate", 1), ("gate", 2)]:
                cs.append(Pix(dt, 2, K, 70, 192, pro=pro, expect={"mma-resident-PT64"}))
        for pro in [("ln", 1), ("gate", 2)]:
            cs.append(Pix(dt, "big", 144, 96, 1024, pro=pro, expect={"mma-resident-PT128"}))
            cs.append(Pix(dt, "big", 48, 96, 1024, pro=pro, out_f32=True, expect={"mma-resident-PT128", "epi-patch"}))
        # K-chunked mma: K > 384 with M > 256 (kstream takes M <= 256), vector and scalar weight staging
        for K in [400, 1021]:
            cs.append(Pix(dt, 2, K, 300, 128, expect={"mma-chunked-vecW", "ring", "epi-vec"}))
            cs.append(Pix(dt, 2, K, 300, 128, w="misaligned" if K % 8 == 0 else "unpadded", expect={"mma-chunked-scalarW", "ring"}))
        cs.append(Pix(dt, 2, 510, 300, 128, out_f32=True, expect={"mma-chunked-vecW", "epi-patch"}))
        cs.append(Pix(dt, 2, 400, 96, 128, x="misaligned", expect={"mma-chunked-vecW", "epi-patch"}))  # kstream needs vec_ok
        # operand layouts the library passes
        cs.append(Pix(dt, 2, 48, 96, 256, x="offset", pro=("ln", 1), expect={"epi-vec"}))
        cs.append(Pix(dt, 2, 80, 160, 256, x="offset", out="group", expect={"epi-vec"}))
        cs.append(Pix(dt, 2, 48, 96, 63, expect={"epi-patch"}))                          # P % 8 != 0
        cs.append(Pix(dt, 2, 510, 96, 63, expect={"mma-chunked-vecW", "epi-patch"}))     # P % 8 != 0: not kstream
        cs.append(Pix(dt, 3, 48, 96, 63, pro=("gate", 1), out_f32=True, expect={"epi-patch"}))
    # fp32 FFMA kernel: resident (with LayerNorm, gate, act range) and K-chunked, with the msplit grid split (one pixel tile)
    cs += [Pix(F32, 2, 48, 96, 200, pro=("ln", 1), expect={"f32-resident"}),
           Pix(F32, 2, 384, 70, 64, pro=("ln", 2), expect={"f32-resident"}),
           Pix(F32, 2, 20, 70, 63, pro=("gate", 1), x="misaligned", expect={"f32-resident"}),
           Pix(F32, 1, 96, 300, 64, pro=("gate", 2), out="group", expect={"f32-resident"}),
           Pix(F32, 1, 1021, 300, 64, expect={"f32-chunked"}),
           Pix(F32, 2, 400, 96, 200, w="unpadded", x="offset", expect={"f32-chunked"})]
    return cs


PIX_CASES = _pix_cases()


@pytest.mark.parametrize("c", PIX_CASES, ids=pix_id)
def test_pixlin(c):
    run_pixlin(c, seed=zlib.crc32(pix_id(c).encode()) % 10007)


@pytest.mark.parametrize("dtype", [F32, BF16, F16])
@pytest.mark.parametrize("pro", [("ln", 1), ("gate", 1)])
def test_pixlin_prologue_needs_resident_k(dtype, pro):
    c = Pix(dtype, 1, 400, 32, 64, pro=pro)
    call = make_pixlin(c, 0, with_ref=False)[0]
    with pytest.raises(RuntimeError, match="pixlin"):
        ops.pixlin(**call)
        torch.cuda.synchronize()


# ----------------------------------------------------------------------------- pixlin: the same values on two paths
@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("pro", [None, ("ln", 1)])
def test_pixlin_pt64_vs_pt128(dtype, pro):
    """image 0 alone (64-pixel tiles) and inside a batch that fills the GPU with 128-pixel tiles.  Bitwise identical without a
    prologue; with the LayerNorm prologue the per-pixel statistics are reduced over 8 (PT 64) or 4 (PT 128) K slices, so the fp32
    statistics -- and rarely the rounded x' -- differ: within the bounds"""
    c = Pix(dtype, "big", 96, 200, 1024, pro=pro)
    call, (ref, S, T), paths, od = make_pixlin(c, 5)
    assert "mma-resident-PT128" in paths
    one = {k: (v[:1] if isinstance(v, torch.Tensor) and v.dim() == 3 else v) for k, v in call.items()}
    if call["gate"] is not None:
        one["gate"] = call["gate"][:1]
    B = batch_of(c)
    assert "mma-resident-PT64" in pixlin_path(1, 96, 200, 1024, dtype, od, bool(pro), True, True)
    a, b = ops.pixlin(**one), ops.pixlin(**call)
    ba = check(a, ref[:1], S[:1], od, "PT 64", T=T[:1] if T.dim() else None)
    bb = check(b, ref, S, od, f"PT 128 (B = {B})", T=T if T.dim() else None)
    check_pair(a, b[:1], ba, bb[:1], "PT 64 vs PT 128", bitwise=pro is None)


@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("K", [48, 510])
def test_pixlin_vec_vs_patch_epilogue(dtype, K):
    """the same x, aligned (epilogue straight from the accumulators) and one element into its storage (smem-patch epilogue):
    bitwise identical"""
    c = Pix(dtype, 2, K, 300, 256)
    call, (ref, S, T), paths, od = make_pixlin(c, 6)
    assert "epi-vec" in paths
    a = ops.pixlin(**call)
    call2 = dict(call, x=misaligned(call["x"]), residual=misaligned(call["residual"]))
    assert not pixlin_vec_ok(call2["x"], a, call2["residual"], dtype, od)
    b = ops.pixlin(**call2)
    check_pair(a, b, check(a, ref, S, od, "vec epilogue"), check(b, ref, S, od, "patch epilogue"), "vec vs patch epilogue",
               bitwise=True)


@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("K", [48, 144])
def test_pixlin_w_all_vs_ring(dtype, K):
    """a padded weight (all weight tiles of a CTA resident) against a misaligned copy of it (the double-buffered ring): bitwise
    identical"""
    c = Pix(dtype, 1, K, 300, 512, pro=("ln", 1))
    call, (ref, S, T), paths, od = make_pixlin(c, 7)
    assert "w_all" in paths
    w2 = misaligned(call["w"])
    assert "ring" in pixlin_path(1, K, 300, 512, dtype, od, True, True, pixlin_w_vec(w2, K, dtype))
    a, b = ops.pixlin(**call), ops.pixlin(**dict(call, w=w2))
    check_pair(a, b, check(a, ref, S, od, "w_all", T=T), check(b, ref, S, od, "ring", T=T), "w_all vs ring", bitwise=True)


# ============================================================================= conv3x3: path mirror
kTH, kTW = 8, 16


def conv_path(x, Cout, nhwc, out):
    """(kernel, pair_ok) that conv3x3_launch takes for input x (the view passed to ops.conv3x3) and destination out"""
    B, Cin, H, W = x.shape
    if x.dtype == F32:
        return ("simt-nhwc" if nhwc else "simt-nchw"), None
    tiles = cdiv(W, kTW) * cdiv(H, kTH) * B
    n = sms()
    if nhwc:
        k = "tma-nhwc-16" if Cout <= 16 else "tma-nhwc-64"
    else:
        aligned = W % 8 == 0 and x.stride(0) % 8 == 0 and x.stride(1) % 8 == 0 and aligned16(x) and x.stride(1) >= H * W and x.stride(0) > 0
        if not aligned:
            return ("generic-16" if Cout <= 16 else "generic-64"), None
        if Cout > 32 and tiles * cdiv(Cout, 64) >= n:
            k = "tma-nchw-64"
        elif Cout > 16 and tiles * cdiv(Cout, 32) >= n:
            k = "tma-nchw-32"
        else:
            k = "tma-nchw-16"
    pair_ok = W % 4 == 0 and out.stride(0) % 2 == 0 and out.stride(1) % 2 == 0 and out.data_ptr() % 4 == 0
    return k, pair_ok


CONV_PATHS = {"tma-nchw-64", "tma-nchw-32", "tma-nchw-16", "tma-nhwc-16", "tma-nhwc-64", "generic-16", "generic-64", "simt-nchw",
              "simt-nhwc", "pair_ok", "pair-elementwise"}
MODES = [G.CONV_PLAIN, G.CONV_UNSHUFFLE2, G.CONV_SHUFFLE2, G.CONV_ADD_NEAREST]
OUT_SHAPE = {G.CONV_PLAIN: lambda B, C, H, W: (B, C, H, W), G.CONV_UNSHUFFLE2: lambda B, C, H, W: (B, 4 * C, H // 2, W // 2),
             G.CONV_SHUFFLE2: lambda B, C, H, W: (B, C // 4, 2 * H, 2 * W), G.CONV_ADD_NEAREST: lambda B, C, H, W: (B, C, H, W)}


# B: an int or "mt64" / "mt32" = the smallest batch at which that output-channel tile fills the GPU
# x: "dense" / "offset" (channels of a wider buffer) / "misaligned" / "nhwc"
# out: "dense" / "slice" (a channel slice of a wider destination, as the decoder's concatenation buffer) / "odd" (one element into
#      its storage: 32-bit pair stores are not aligned -> element-wise stores)
Conv = namedtuple("Conv", "dtype B Cin Cout H W mode scale x out expect")
Conv.__new__.__defaults__ = ("dense", "dense", None)


def conv_batch(c):
    if c.B == "mt64":
        return cdiv(sms(), cdiv(c.W, kTW) * cdiv(c.H, kTH) * cdiv(c.Cout, 64))
    if c.B == "mt32":
        return cdiv(sms(), cdiv(c.W, kTW) * cdiv(c.H, kTH) * cdiv(c.Cout, 32))
    return c.B


def conv_id(c):
    return f"{str(c.dtype)[6:]}-B{c.B}-{c.Cin}to{c.Cout}-{c.H}x{c.W}-mode{c.mode}-s{c.scale}-x_{c.x}-out_{c.out}"


def make_conv(c, seed, with_ref=True):
    torch.manual_seed(seed)
    dt, B, Cin, Cout, H, W = c.dtype, conv_batch(c), c.Cin, c.Cout, c.H, c.W
    dev = "cuda"
    x = torch.randn(B, Cin, H, W, device=dev).to(dt)
    w = (torch.randn(Cout, Cin, 3, 3, device=dev) * (9 * Cin) ** -0.5).to(dt)
    bias = 0.5 * torch.randn(Cout, device=dev)
    add = torch.randn(B, Cout, H // c.scale, W // c.scale, device=dev).to(dt) if c.mode == G.CONV_ADD_NEAREST else None
    if c.x == "offset":
        buf = torch.randn(B, Cin + 8, H, W, device=dev).to(dt)
        buf[:, 8:] = x
        xx = buf[:, 8:]
    elif c.x == "misaligned":
        xx = misaligned(x)
    elif c.x == "nhwc":
        xx = x.contiguous(memory_format=torch.channels_last)
    else:
        xx = x
    shape = OUT_SHAPE[c.mode](B, Cout, H, W)
    if c.out == "slice":
        obuf = torch.full((shape[0], shape[1] + 6) + shape[2:], float("nan"), device=dev, dtype=dt)
        out = obuf[:, 2:2 + shape[1]]
    elif c.out == "odd":
        out = misaligned(torch.full(shape, float("nan"), device=dev, dtype=dt))
    else:
        out = torch.empty(shape, device=dev, dtype=dt)
    ref = S = None
    if with_ref:
        ref, S = G.conv3x3_ref(x.double(), w.double(), bias.double(), c.mode, None if add is None else add.double(), c.scale)
    k, pair_ok = conv_path(xx, Cout, c.x == "nhwc", out)
    paths = {k} | ({"pair_ok" if pair_ok else "pair-elementwise"} if pair_ok is not None else set())
    call = dict(x=xx, wp=ops.pack_conv3x3_weight(w, dt), bias=bias, c_out=Cout, mode=c.mode, out=out, add=add, add_scale=c.scale,
                nhwc=c.x == "nhwc")
    return call, ref, S, paths


def run_conv(c, seed=0):
    call, ref, S, paths = make_conv(c, seed)
    if c.expect is not None:
        assert set(c.expect) <= paths, (sorted(c.expect), sorted(paths))
    got = ops.conv3x3(**call)
    assert got.data_ptr() == call["out"].data_ptr()
    return got, check(got, ref, S, c.dtype, conv_id(c), paths), paths


def _conv_cases():
    cs = []
    for dt in DT16:
        for mode, sc in [(m, 1) for m in MODES] + [(G.CONV_ADD_NEAREST, 2)]:
            for out in ("dense", "slice", "odd"):
                # TMA NCHW, output-channel tile 64 / 32 / 16 (Cout not a multiple of the tile), Cin chunk tails 20 / 5 / 3
                cs.append(Conv(dt, "mt64", 20, 80, 32, 32, mode, sc, out=out, expect={"tma-nchw-64"}))
                cs.append(Conv(dt, "mt32", 5, 48, 32, 32, mode, sc, out=out, expect={"tma-nchw-32"}))
                cs.append(Conv(dt, 2, 3, 20, 10, 24, mode, sc, out=out, expect={"tma-nchw-16"}))
                # TMA NHWC, tile 16 / 64
                cs.append(Conv(dt, 2, 16, 12, 10, 24, mode, sc, x="nhwc", out=out, expect={"tma-nhwc-16"}))
                cs.append(Conv(dt, 2, 24, 72, 10, 24, mode, sc, x="nhwc", out=out, expect={"tma-nhwc-64"}))
                # generic (unaligned) kernel, tile 16 / 64: a misaligned base, W % 8 != 0
                cs.append(Conv(dt, 2, 20, 16, 10, 24, mode, sc, x="misaligned", out=out, expect={"generic-16"}))
                cs.append(Conv(dt, 2, 5, 72, 10, 12, mode, sc, out=out, expect={"generic-64"}))
        # partial 8 x 16 tiles and halo borders: H = 1, 9; W = 8, 24; the channel-offset input view; add_scale 1 / 4
        for H, W in [(1, 8), (9, 24), (9, 8), (1, 24)]:
            cs.append(Conv(dt, 3, 20, 36, H, W, G.CONV_PLAIN, 1, x="offset", expect={"tma-nchw-16", "pair_ok"}))
            cs.append(Conv(dt, 2, 8, 20, H, W, G.CONV_SHUFFLE2, 1, x="nhwc", out="odd", expect={"tma-nhwc-64", "pair-elementwise"}))
        cs.append(Conv(dt, 2, 20, 36, 8, 24, G.CONV_ADD_NEAREST, 4, expect={"tma-nchw-16"}))
        cs.append(Conv(dt, 2, 96, 3, 16, 32, G.CONV_ADD_NEAREST, 4, x="nhwc", expect={"tma-nhwc-16"}))
        cs.append(Conv(dt, 2, 20, 36, 8, 24, G.CONV_ADD_NEAREST, 1, out="odd", expect={"tma-nchw-16", "pair-elementwise"}))
    # fp32: the SIMT kernel, NCHW and NHWC, every store mode
    for mode in MODES:
        for x in ("dense", "nhwc"):
            cs.append(Conv(F32, 2, 5, 20, 10, 24, mode, 2 if mode == G.CONV_ADD_NEAREST else 1, x=x, out="slice",
                           expect={"simt-nhwc" if x == "nhwc" else "simt-nchw"}))
        cs.append(Conv(F32, 2, 20, 36, 9 if mode != G.CONV_UNSHUFFLE2 else 10, 12, mode, 1, x="offset", out="odd",
                       expect={"simt-nchw"}))
    return cs


CONV_CASES = _conv_cases()


@pytest.mark.parametrize("c", CONV_CASES, ids=conv_id)
def test_conv3x3(c):
    run_conv(c, seed=zlib.crc32(conv_id(c).encode()) % 10007)


# ----------------------------------------------------------------------------- conv3x3: the same values on two paths
@pytest.mark.parametrize("dtype", DT16)
def test_conv3x3_mt16_vs_mt32_vs_mt64(dtype):
    """image 0 alone (tile 16) and inside batches that fill the GPU with the 32- and 64-channel tiles: bitwise identical"""
    c = Conv(dtype, "mt64", 20, 48, 32, 32, G.CONV_PLAIN, 1)
    call, ref, S, paths = make_conv(c, 9)
    assert "tma-nchw-64" in paths
    B32 = cdiv(sms(), 8 * 2)
    outs = {}
    for B, want in [(1, "tma-nchw-16"), (B32, "tma-nchw-32"), (conv_batch(c), "tma-nchw-64")]:
        xb, ob = call["x"][:B], torch.empty((B, 48, 32, 32), dtype=dtype, device="cuda")
        assert conv_path(xb, 48, False, ob)[0] == want
        got = ops.conv3x3(**dict(call, x=xb, out=ob))
        outs[want] = (got[:1], check(got, ref[:B], S[:B], dtype, want)[:1])
    (a, ba), (b, bb), (d, bd) = outs.values()
    check_pair(a, b, ba, bb, "MT 16 vs MT 32", bitwise=True)
    check_pair(a, d, ba, bd, "MT 16 vs MT 64", bitwise=True)


@pytest.mark.parametrize("dtype", DT16)
@pytest.mark.parametrize("mode", MODES)
def test_conv3x3_tma_vs_generic(dtype, mode):
    """the same input aligned (TMA) and one element into its storage (the generic kernel); paired and element-wise stores: bitwise
    identical"""
    c = Conv(dtype, 2, 20, 36, 16, 32, mode, 1)
    call, ref, S, paths = make_conv(c, 10)
    assert "tma-nchw-16" in paths and "pair_ok" in paths
    a = ops.conv3x3(**call)
    ba = check(a, ref, S, dtype, "TMA")
    xm, om = misaligned(call["x"]), misaligned(torch.empty_like(call["out"]))
    assert conv_path(xm, 36, False, om)[0] == "generic-64"
    b = ops.conv3x3(**dict(call, x=xm, out=om))
    check_pair(a, b, ba, check(b, ref, S, dtype, "generic"), "TMA vs generic", bitwise=True)
    oo = misaligned(torch.empty_like(call["out"]))
    assert conv_path(call["x"], 36, False, oo)[1] is False
    e = ops.conv3x3(**dict(call, out=oo))
    check_pair(a, e, ba, check(e, ref, S, dtype, "TMA, element-wise stores"), "paired vs element-wise stores",
               bitwise=True)


# ============================================================================= the bench net's call sites (B = 8, 64 x 64 LQ)
def bench_sites():
    """(pixlin cases, conv cases) of the bench's default net (MambaSISR6, class defaults) at B = 8, 64 x 64, from its modules"""
    from vmambair_b200 import archs
    net = archs.MambaSISR6()
    B, H = 8, 64
    pix, conv = [], []
    for stage, hw in [(net.encoder_level1, H), (net.encoder_level2, H // 2), (net.decoder_level1, H), (net.latent, H // 8)]:
        blk = stage[0]
        a, f = blk.attn, blk.ffn
        D, C, N = a.d_model, a.d_inner, a.d_state
        gm = 1 if a.gate == "mul" else 2
        L = hw * hw
        has_b = lambda m: m.bias is not None
        pix += [Pix(BF16, B, D, 2 * C, L, pro=("ln", 1), act=(C, 2 * C), bias=has_b(a.in_conv), res=False),  # norm1 + in_conv, SiLU(z)
                Pix(BF16, B, C, 2 * (C + 2 * N), L, act=False, bias=False, res=False),  # x_proj + dt_proj of two directions
                Pix(BF16, B, C, D, L, pro=("gate", gm), act=False, bias=has_b(a.out_conv)),  # channel gate + out_conv + residual
                Pix(BF16, B, D, f.project_in.out_channels, L, pro=("ln", 1), act=False, bias=has_b(f.project_in), res=False),
                Pix(BF16, B, f.project_out.in_channels, D, L, act=False, bias=has_b(f.project_out))]  # project_out + residual
    for m, hw in [(net.reduce_chan_level2, H // 2), (net.reduce_chan_level3, H // 4)]:
        pix.append(Pix(BF16, B, m.in_channels, m.out_channels, hw * hw, act=False, bias=m.bias is not None, res=False))
    for m, hw, mode in [(net.patch_embed.proj, H, G.CONV_PLAIN), (net.down1_2.body[0], H, G.CONV_UNSHUFFLE2),
                        (net.down2_3.body[0], H // 2, G.CONV_UNSHUFFLE2), (net.down3_4.body[0], H // 4, G.CONV_UNSHUFFLE2),
                        (net.up4_3.body[0], H // 8, G.CONV_SHUFFLE2), (net.up3_2.body[0], H // 4, G.CONV_SHUFFLE2),
                        (net.up2_1.body[0], H // 2, G.CONV_SHUFFLE2)]:
        conv.append(Conv(BF16, B, m.in_channels, m.out_channels, hw, hw, mode, 1, out="slice" if mode == G.CONV_SHUFFLE2 else "dense"))
    last = net.tail[1]  # conv_last on the NHWC features at 4x, + the nearest-upsampled LQ image
    conv.append(Conv(BF16, B, last.in_channels, last.out_channels, 4 * H, 4 * H, G.CONV_ADD_NEAREST, 4, x="nhwc"))
    return pix, conv


BENCH_PIX, BENCH_CONV = bench_sites()


@pytest.mark.parametrize("c", BENCH_PIX, ids=pix_id)
def test_bench_pixlin_site(c):
    run_pixlin(c, seed=11)


@pytest.mark.parametrize("c", BENCH_CONV, ids=conv_id)
def test_bench_conv3x3_site(c):
    run_conv(c, seed=12)


# ============================================================================= coverage of the path table
def test_every_path_is_covered():
    hit = set()
    for c in PIX_CASES + BENCH_PIX:
        hit |= make_pixlin(c, 0, with_ref=False)[2]
    for c in CONV_CASES + BENCH_CONV:
        hit |= make_conv(c, 0, with_ref=False)[3]
    assert hit == PIXLIN_PATHS | CONV_PATHS, (sorted(PIXLIN_PATHS | CONV_PATHS - hit), sorted(hit - PIXLIN_PATHS - CONV_PATHS))
