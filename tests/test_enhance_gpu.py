"""RealESRGANer.enhance on the library's kernels (vmambair_b200.enhance, csrc/image_io.cu) against the reference's outputs
(tests/golden/enhance_ref.npz), and every image kernel against OpenCV's results (enhance_cv2.npz) and the numpy restatements of
vmambair_b200.image_ref, bit for bit."""
import collections
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from vmambair_b200 import archs, image_ref, ops
from vmambair_b200.enhance import RealESRGANer, pad_plan
from vmambair_b200.tiling import TiledInference

pytestmark = pytest.mark.gpu
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def _load(name):
    with np.load(os.path.join(GOLDEN, name)) as f:
        return {k: f[k] for k in f.files}


@pytest.fixture(scope="module")
def cv():
    return _load("enhance_cv2.npz")


@pytest.fixture(scope="module")
def ref():
    return _load("enhance_ref.npz")


@pytest.fixture(scope="module")
def weights(tmp_path_factory):
    """the tiny reference networks' weights as BasicSR checkpoints ({"params_ema": state_dict})"""
    out = {}
    for tag in ("realsr", "sisr"):
        sd = {k: torch.from_numpy(v.astype(np.float32)) for k, v in _load(f"enhance_net_{tag}.npz").items()}
        path = str(tmp_path_factory.mktemp("w") / f"{tag}.pth")
        torch.save({"params_ema": sd}, path)
        out[tag] = path
    return out


def _net(tag):
    ctor = archs.MambaRealSR11 if tag == "realsr" else archs.MambaSISR6
    return ctor(dim=8, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1)


def _cases(ref):
    return sorted({k.split("/")[0] for k in ref})


def _upsampler(ref, weights, name, **kw):
    pre_pad, tile, tile_pad, outscale, net_alpha = ref[f"{name}/params"]
    tag = str(ref[f"{name}/net"])
    up = RealESRGANer(4, weights[tag], model=_net(tag), tile=int(tile), tile_pad=int(tile_pad), pre_pad=int(pre_pad), **kw)
    return up, (None if outscale < 0 else float(outscale)), ("realesrgan" if net_alpha else "bilinear")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---------------------------------------------------------------- kernels

@pytest.mark.parametrize("i", range(6))
@pytest.mark.parametrize("depth", ["uint8", "uint16"])
def test_lanczos4_kernel_matches_opencv(cv, i, depth):
    src, dst = cv[f"lanczos{i}_{depth}/src"], cv[f"lanczos{i}_{depth}/dst"]
    got = ops.resize_lanczos4(_dev(src), dst.shape[1], dst.shape[0]).cpu().numpy()
    np.testing.assert_array_equal(got, dst)


@pytest.mark.parametrize("depth", [np.uint8, np.uint16])
@pytest.mark.parametrize("c", [1, 3, 4])
@pytest.mark.parametrize("size,f", [((37, 53), 1.7), ((64, 31), 0.5), ((5, 7), 3.5), ((129, 67), 0.3)])
def test_lanczos4_kernel_on_strided_views_matches_the_restatement(depth, c, size, f):
    rng = np.random.default_rng(hash((c, size)) % 1000)
    h, w = size
    hi = 256 if depth == np.uint8 else 65536
    big = rng.integers(0, hi, (h + 3, w + 5, c)).astype(depth)
    view = big[2:2 + h, 3:3 + w] if c > 1 else big[2:2 + h, 3:3 + w, 0]  # row stride > width: a crop of a wider image
    dw, dh = int(w * f), int(h * f)
    want = image_ref.resize_lanczos4(np.ascontiguousarray(view), (dw, dh))
    t = _dev(big)
    tv = t[2:2 + h, 3:3 + w] if c > 1 else t[2:2 + h, 3:3 + w, 0]
    np.testing.assert_array_equal(ops.resize_lanczos4(tv, dw, dh).cpu().numpy(), want)


def _planes_ref(img, max_range, ph, pw, alpha_plane):
    """image_to_planes in torch on the host: float32 division, BGR -> RGB / gray x 3, three reflect pads"""
    x = torch.from_numpy(np.ascontiguousarray(img).astype(np.float32)) / torch.tensor(max_range, dtype=torch.float32)
    x = x[:, :, None] if x.dim() == 2 else x
    rgb = x[:, :, [0, 0, 0]] if x.shape[2] == 1 else x[:, :, [2, 1, 0]]
    ims = [rgb] + ([x[:, :, [3, 3, 3]]] if alpha_plane else [])
    p = torch.stack(ims).permute(0, 3, 1, 2)
    for a, b in zip(ph, pw):
        if a or b:
            p = F.pad(p, (0, b, 0, a), "reflect")
    return p


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("c,alpha", [(1, False), (3, False), (4, False), (4, True)])
@pytest.mark.parametrize("depth", [np.uint8, np.uint16])
def test_image_to_planes_matches_torch(dtype, c, alpha, depth):
    rng = np.random.default_rng(c)
    h, w = 19, 13
    max_range = 255 if depth == np.uint8 else 65535
    img = rng.integers(0, max_range + 1, (h, w, c)).astype(depth)
    ph, pw = pad_plan(h, w, 10, 2)  # (10, 1, 2), (10, 1, 0): pre_pad, the mod pad of scale 2 and the pad to 8
    # channels-planar storage seen as HWC: pixel stride 1, channel stride H*W (a non-contiguous view)
    planar = _dev(np.moveaxis(img, 2, 0).copy()).permute(1, 2, 0)
    src = planar if c > 1 else planar[:, :, 0]
    got = ops.image_to_planes(src, max_range, ph, pw, alpha_plane=alpha, dtype=dtype)
    want = _planes_ref(img if c > 1 else img[:, :, 0], max_range, ph, pw, alpha).to(dtype)
    assert got.shape == want.shape == (1 + alpha, 3, h + sum(ph), w + sum(pw))
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("depth", [np.uint8, np.uint16])
def test_image_max(depth):
    rng = np.random.default_rng(3)
    hi = 256 if depth == np.uint8 else 40000
    img = rng.integers(0, hi // 2, (33, 70, 4)).astype(depth)
    img[31, 66, 3] = hi - 1  # in the alpha channel, near the bottom-right corner
    assert int(ops.image_max(_dev(img)).item()) == hi - 1
    assert int(ops.image_max(_dev(img)[:30, :60]).item()) == img[:30, :60].max()


def _image_ref(planes, H, W, channels, max_range, out_dtype, alpha_src=None):
    """planes_to_image restated with numpy and vmambair_b200.image_ref"""
    p = np.clip(planes.float().cpu().numpy()[:, :, :H, :W], 0, 1).astype(np.float32)
    bgr = np.transpose(p[0, [2, 1, 0]], (1, 2, 0))
    if channels == 1:
        v = image_ref.bgr2gray(bgr)
    else:
        v = bgr
        if channels == 4:
            if alpha_src is None:
                a = image_ref.bgr2gray(np.transpose(p[1, [2, 1, 0]], (1, 2, 0)))
            else:
                a = image_ref.resize_linear((alpha_src.astype(np.float32) / np.float32(max_range)).astype(np.float32), (W, H))
            v = np.concatenate([v, a[:, :, None]], 2)
    r = np.rint((v * np.float32(max_range)).astype(np.float32))
    return np.clip(r, 0, np.iinfo(out_dtype).max).astype(out_dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("c,linear", [(1, False), (3, False), (4, False), (4, True)])
@pytest.mark.parametrize("depth", [np.uint8, np.uint16])
def test_planes_to_image_matches_the_restatement(dtype, c, linear, depth):
    torch.manual_seed(c)
    H, W = 4 * 11, 4 * 9
    max_range = 255 if depth == np.uint8 else 65535
    planes = (torch.rand(2, 3, H + 12, W + 20) * 1.2 - 0.1).to(DEV, dtype)  # values outside [0, 1] are clamped
    planes = planes[:, :, 5:, 3:]  # a cropped view: row stride > width, offset start
    alpha_src = np.random.default_rng(c).integers(0, max_range + 1, (11, 9)).astype(depth) if linear else None
    src = torch.from_numpy(np.stack([alpha_src] * 4, 2)).to(DEV)[:, :, 3] if linear else None  # a channel of an RGBA image
    got = ops.planes_to_image(planes, H, W, c, max_range, torch.uint8 if depth == np.uint8 else torch.uint16, alpha_src=src)
    want = _image_ref(planes, H, W, c, max_range, depth, alpha_src)
    np.testing.assert_array_equal(got.cpu().numpy(), want)


def test_gray_and_linear_kernels_match_opencv(cv):
    """BGR2GRAY and INTER_LINEAR through planes_to_image against cv2: gray bit-exact after x 255 / 65535 and rounding; the linear alpha
    within 1 LSB (OpenCV runs float INTER_LINEAR through IPP, test_enhance_cpu.py::test_linear_restatement_within_one_ulp)"""
    g = cv["gray/src"]
    planes = torch.from_numpy(np.ascontiguousarray(np.transpose(g[:, :, [2, 1, 0]], (2, 0, 1))))[None].to(DEV)
    for m, dt in ((255, torch.uint8), (65535, torch.uint16)):
        got = ops.planes_to_image(planes, g.shape[0], g.shape[1], 1, m, dt).cpu().numpy()
        want = np.rint(np.clip(cv["gray/dst"], 0, 1) * np.float32(m)).astype(got.dtype)
        np.testing.assert_array_equal(got, want)
    for i in range(3):
        src, dst = cv[f"linear{i}/src"], cv[f"linear{i}/dst"]
        a8 = np.rint(src * 255).astype(np.uint8)  # the fixtures' sources are k / 255
        H, W = dst.shape
        got = ops.planes_to_image(torch.zeros(1, 3, H, W, device=DEV), H, W, 4, 255, torch.uint8, alpha_src=_dev(a8))
        d = np.abs(got.cpu().numpy()[:, :, 3].astype(int) - np.rint(dst * np.float32(255)).astype(int))
        assert d.max() <= 1


def test_kernels_replay_in_a_cuda_graph():
    rng = np.random.default_rng(9)
    img = _dev(rng.integers(0, 65536, (24, 40, 4)).astype(np.uint16))
    ph, pw = pad_plan(24, 40, 10, 4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())

    def run():
        m = ops.image_max(img)
        p = ops.image_to_planes(img, 65535, ph, pw, alpha_plane=True, dtype=torch.bfloat16)
        o = ops.planes_to_image(p, 24, 40, 4, 65535, torch.uint16)
        return m, o, ops.resize_lanczos4(o, 61, 37)

    with torch.cuda.stream(s):
        eager = [t.clone() for t in run()]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            outs = run()
    torch.cuda.current_stream().wait_stream(s)
    img.copy_(torch.flip(img, [0]))
    eager2 = [t.clone() for t in run()]
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(eager[1], eager2[1])
    for a, b in zip(outs, eager2):
        assert torch.equal(a, b)


# ---------------------------------------------------------------- enhance()

def _close_to(got, want):
    """the fp32 bound: 8-bit results at most 1 LSB off, on at most 0.5 % of the values (rounding ties moved by the ~1e-5 network
    difference).  A 16-bit LSB (1.5e-5 of the range) is the size of that difference itself, so ties are ~250x more frequent there:
    16-bit results at most 2 LSB off (1 LSB, doubled for the Lanczos taps of outscale), on at most 5 % of the values."""
    d = np.abs(got.astype(np.int64) - want.astype(np.int64))
    lsb, frac = (2, 0.05) if want.dtype == np.uint16 else (1, 0.005)
    return d.max() <= lsb and (d > 0).mean() <= frac, (int(d.max()), float((d > 0).mean()))


def test_enhance_fp32_matches_the_reference(ref, weights):
    bad = {}
    for name in _cases(ref):
        up, outscale, alpha = _upsampler(ref, weights, name)
        img, want = ref[f"{name}/img"], ref[f"{name}/out"]
        got, mode = up.enhance(img, outscale=outscale, alpha_upsampler=alpha)
        assert isinstance(got, np.ndarray) and got.dtype == want.dtype and got.shape == want.shape, name
        assert mode == {2: "L", 3: "RGB", 4: "RGBA"}[img.ndim if img.ndim == 2 else img.shape[2]], name
        ok, stats = _close_to(got, want)
        if not ok:
            bad[name] = stats
    assert not bad, bad


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_enhance_16_bit_compute(ref, weights, dtype):
    for name in _cases(ref):
        kw = dict(half=True) if dtype == torch.float16 else dict(dtype=dtype)
        up, outscale, alpha = _upsampler(ref, weights, name, **kw)
        img, want = ref[f"{name}/img"], ref[f"{name}/out"]
        got, _ = up.enhance(img, outscale=outscale, alpha_upsampler=alpha)
        mr = 65535 if want.dtype == np.uint16 else 255
        d = np.abs(got.astype(np.float64) - want.astype(np.float64))
        assert got.dtype == want.dtype and d.max() <= 0.08 * mr and d.mean() <= 0.01 * mr, (name, d.max(), d.mean())


def test_enhance_tensor_inputs_come_back_on_their_device(ref, weights):
    name = "rgba8_net"
    up, outscale, alpha = _upsampler(ref, weights, name)
    img = ref[f"{name}/img"]
    want, _ = up.enhance(img)
    got_dev, mode = up.enhance(torch.from_numpy(img).to(DEV))
    got_cpu, _ = up.enhance(torch.from_numpy(img))
    assert got_dev.is_cuda and not got_cpu.is_cuda and mode == "RGBA"
    for got in (got_dev.cpu().numpy(), got_cpu.numpy()):  # three network runs: equal up to their run-to-run rounding
        assert got.dtype == want.dtype and got.shape == want.shape
        ok, stats = _close_to(got, want)
        assert ok, stats


@pytest.mark.parametrize("shape,pre_pad,tile", [((19, 27, 3), 10, 0), ((13, 30), 0, 0), ((21, 17, 4), 10, 0), ((37, 45, 3), 10, 16)])
def test_sizes_not_multiple_of_8_equal_the_composed_path(weights, shape, pre_pad, tile):
    """convert (torch on the host) -> TiledInference on the float planes -> convert back, against enhance(): the same values up to the
    run-to-run rounding of the network's fp32 atomics (the merge statistics), i.e. within the bound of the reference comparison"""
    rng = np.random.default_rng(sum(shape))
    img = rng.integers(0, 256, shape).astype(np.uint8)
    net = _net("realsr")
    up = RealESRGANer(4, weights["realsr"], model=net, tile=tile, tile_pad=8, pre_pad=pre_pad)
    got, _ = up.enhance(img)
    h, w = shape[:2]
    ph, pw = pad_plan(h, w, pre_pad, 4)
    planes = _planes_ref(img, 255, ph, pw, len(shape) == 3 and shape[2] == 4).to(DEV)
    y = TiledInference(up.runner.net, scale=4, multiple=8, tile_size=tile, tile_pad=8, dtype=torch.float32)(planes)
    want = ops.planes_to_image(y, 4 * h, 4 * w, 1 if len(shape) == 2 else shape[2], 255, torch.uint8).cpu().numpy()
    assert got.shape == want.shape == (4 * h, 4 * w) + shape[2:]
    ok, stats = _close_to(got, want)
    assert ok, stats


def kernel_census(fn):
    """(the kernels fn launches, as a Counter of their names in a torch.profiler trace, without copies and memsets; fn's result).
    The kernel records of a session's first milliseconds can be lost (a census once missed the first kernel of each session:
    image_to_planes of enhance(), conv_first of the net; sessions of a few short kernels lost all of them), so the session opens with
    a spin of about 0.1 s, fn runs twice, and only the kernels after a marker kernel between the two runs are counted; the result is
    the second run's."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda._sleep(200_000_000)  # the lead-in: spin_kernel, 2e8 cycles
        torch.cuda.synchronize()
        for run in range(2):
            out = fn()
            torch.cuda.synchronize()
            if run == 0:
                torch.cuda._sleep(1000)  # the marker: spin_kernel
                torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    marks = [i for i, e in enumerate(ev) if "spin_kernel" in e.name]  # the lead-in (if it was recorded), then the marker
    assert marks, [e.name for e in ev]
    return collections.Counter(e.name for e in ev[marks[-1] + 1:] if "emcpy" not in e.name and "emset" not in e.name), out


def kernel_names(census):
    """the bare function names in a census: "void vmb::scan_fwd_kernel<float, 2>(vmb::ScanFwdParams)" -> "scan_fwd_kernel" """
    bare = lambda n: n.replace("(anonymous namespace)::", "").split("<")[0].split("(")[0].split(" ")[-1].split("::")[-1]
    return collections.Counter(bare(n) for n in census.elements())


def test_launch_census(ref, weights):
    """between the input and the output only the library's image kernels and the network run: no torch pad / permute / cast / copy"""
    name = "rgb8"
    up, _, _ = _upsampler(ref, weights, name)
    x = torch.from_numpy(ref[f"{name}/img"]).to(DEV)
    ph, pw = pad_plan(x.shape[0], x.shape[1], up.pre_pad, 4)
    planes = ops.image_to_planes(x, 255, ph, pw)
    up.enhance(x)
    up.runner(planes)
    torch.cuda.synchronize()
    full, _ = kernel_census(lambda: up.enhance(x))
    net, _ = kernel_census(lambda: up.runner(planes))
    extra = full - net
    assert sorted(extra) == sorted(k for k in extra if "image_to_planes_kernel" in k or "planes_to_image_kernel" in k), extra
    assert sum(extra.values()) == 2 and not (net - full), (extra, net - full)
