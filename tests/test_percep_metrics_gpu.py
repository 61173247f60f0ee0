"""vmambair_b200.lpips and .dists on the GPU against the float64 torch restatements (oracle/lpips_ref.py, oracle/dists_ref.py) on the
same weights: seeded random VGG16 trunks with non-zero biases, random lin weights, random and the reference's alpha / beta.  Per
image |ours - fp64| <= 4 |torch fp32 restatement - fp64| + 1e-6.  Also identical inputs, the uint8 evaluation loop, determinism
without host synchronisation, CUDA-graph capture, the launch census, input validation, and parity with the lpips package where it is
installed.  TF32 is off unless a test says otherwise."""
import os

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as TF

from oracle import dists_ref, lpips_ref
from vmambair_b200 import _pmetric, ops
from vmambair_b200.dists import DISTS, calculate_dists
from vmambair_b200.lpips import LPIPS, calculate_lpips

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "dists_ref.npz"))
LPIPS_LAUNCHES = 1 + 8 + 4 * 2 + 1 + 1  # prep, ReLU stages, (layer + ReLU/pool) x 4, layer 5, final
DISTS_LAUNCHES = 1 + 8 + 5 + 1          # prep (with layer 0's statistics), ReLU stages, layers (with the L2 pool), final


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _set_trunk(module_of, seed):
    with torch.no_grad():
        for i, (w, b) in zip(_pmetric.CONVS, lpips_ref.seeded_vgg16_convs(seed)):
            module_of(i).weight.copy_(w)
            module_of(i).bias.copy_(b)


def _lpips(seed=0):
    torch.manual_seed(seed)
    m = LPIPS(pretrained=False, pnet_rand=True)
    _set_trunk(m.net.module, 100 + seed)
    with torch.no_grad():
        for lin in m.lins:
            lin.model[1].weight.copy_(torch.rand_like(lin.model[1].weight))
    return m.to(DEV)


def _dists(seed=0, real=False):
    torch.manual_seed(seed)
    m = DISTS(load_weights=False, vgg_weights=None)
    _set_trunk(m._module, 200 + seed)
    if real:
        with torch.no_grad():
            m.alpha.copy_(torch.from_numpy(GOLD["real_alpha"]))
            m.beta.copy_(torch.from_numpy(GOLD["real_beta"]))
    return m.to(DEV)


def _pair(shape, kind, lo=0.0, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    gt = lo + (1 - lo) * torch.rand(shape, device=DEV, generator=g)
    if kind == "noisy":
        return gt + 1e-2 * torch.randn(shape, device=DEV, generator=g), gt
    return lo + (1 - lo) * torch.rand(shape, device=DEV, generator=g), gt


def _within(ours, r64, r32, what):
    ours, r64, r32 = (t.detach().double().reshape(-1) for t in (ours, r64, r32))
    err, err32 = (ours - r64).abs(), (r32 - r64).abs()
    print(f"\n{what}: value {r64.abs().max().item():.3e}, err {err.max().item():.2e} (torch fp32 {err32.max().item():.2e})")
    assert bool((err <= 4 * err32 + 1e-6).all()), (err.tolist(), err32.tolist())


LP_SHAPES = [(1, 3, 16, 16), (3, 3, 37, 53), (1, 3, 64, 48), (2, 3, 256, 256)]


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("kind", ["unrelated", "noisy"])
@pytest.mark.parametrize("shape", LP_SHAPES)
def test_lpips_matches_fp64(shape, kind, normalize):
    m = _lpips()
    x, y = _pair(shape, kind, lo=0.0 if normalize else -1.0)
    sd = m.state_dict()
    with torch.no_grad():
        val, res = m(x, y, retPerLayer=True, normalize=normalize)
        v64, r64 = lpips_ref.lpips_from_state_dict({k: v.double() for k, v in sd.items()}, x.double(), y.double(), normalize)
        v32, r32 = lpips_ref.lpips_from_state_dict(sd, x, y, normalize)
    assert val.shape == (shape[0], 1, 1, 1) and val.dtype == torch.float32 and len(res) == 5
    assert torch.equal(val, m(x, y, normalize=normalize))
    _within(val, v64, v32, f"lpips {shape} {kind} normalize={normalize}")
    for k in range(5):
        _within(res[k], r64[k], r32[k], f"  layer {k}")


DI_SHAPES = [(1, 3, 1, 1), (1, 3, 3, 3), (3, 3, 37, 53), (1, 3, 64, 48), (2, 3, 256, 256)]


@pytest.mark.parametrize("real", [False, True])
@pytest.mark.parametrize("kind", ["unrelated", "noisy"])
@pytest.mark.parametrize("shape", DI_SHAPES)
def test_dists_matches_fp64(shape, kind, real):
    m = _dists(real=real)
    x, y = _pair(shape, kind)
    sd = m.state_dict()
    with torch.no_grad():
        s = m(x, y)
        s64 = dists_ref.dists_from_state_dict({k: v.double() for k, v in sd.items()}, x.double(), y.double())
        s32 = dists_ref.dists_from_state_dict(sd, x, y)
        mean = m(x, y, batch_average=True)
    assert s.shape == s64.shape and s.dtype == torch.float32 and mean.shape == ()
    _within(s, s64, s32, f"dists {shape} {kind} real={real}")
    _within(mean, s64.mean(), s32.mean(), "  batch_average")


def test_identical_inputs():
    x, _ = _pair((2, 3, 40, 56), "unrelated", lo=-1.0)
    with torch.no_grad():
        assert _lpips()(x, x.clone()).abs().max().item() <= 1e-7
        assert _dists()(x, x.clone()).abs().max().item() <= 1e-6


def _u8_pair(B, H, W, seed=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    gt = torch.randint(0, 256, (B, H, W, 3), device=DEV, generator=g, dtype=torch.uint8)
    noise = torch.randint(-12, 13, (B, H, W, 3), device=DEV, generator=g)
    return (gt.int() + noise).clamp(0, 255).to(torch.uint8), gt


def _script_lpips_tensor(img):
    """Metric/LPIPS.py's conversion of one (H, W, 3) uint8 BGR image: float32 / 255., BGR -> RGB, CHW, normalize(.5, .5)"""
    a = img.astype(np.float32) / 255.
    t = torch.from_numpy(np.ascontiguousarray(a[..., ::-1].transpose(2, 0, 1)))
    return TF.normalize(t, [0.5, 0.5, 0.5], [0.5, 0.5, 0.5], inplace=True)


def _script_dists_tensor(img):
    """Metric/dists.py's prepare_image of the RGB image: ToTensor, i.e. uint8 HWC -> float32 CHW / 255"""
    return TF.to_tensor(np.ascontiguousarray(img[..., ::-1]))


def test_evaluation_loop_matches_the_scripts_conversion():
    out, gt = _u8_pair(3, 37, 53)
    lp, di = _lpips(), _dists(real=True)
    o_np, g_np = out.cpu().numpy(), gt.cpu().numpy()
    with torch.no_grad():
        want_lp = lp(torch.stack([_script_lpips_tensor(a) for a in o_np]).to(DEV),
                     torch.stack([_script_lpips_tensor(a) for a in g_np]).to(DEV)).reshape(-1)
        want_di = di(torch.stack([_script_dists_tensor(a) for a in g_np]).to(DEV),
                     torch.stack([_script_dists_tensor(a) for a in o_np]).to(DEV)).reshape(-1)
    got_lp, got_di = calculate_lpips(out, gt, lp), calculate_dists(out, gt, di)
    assert got_lp.shape == (3,) and got_di.shape == (3,) and got_lp.dtype == got_di.dtype == torch.float32
    assert torch.equal(got_lp, want_lp) and torch.equal(got_di, want_di)
    v_lp, v_di = calculate_lpips(o_np[1], g_np[1], lp), calculate_dists(o_np[1], g_np[1], di)
    assert isinstance(v_lp, float) and isinstance(v_di, float)
    with torch.no_grad():
        assert v_lp == lp(_script_lpips_tensor(o_np[1])[None].to(DEV), _script_lpips_tensor(g_np[1])[None].to(DEV)).item()
        assert v_di == di(_script_dists_tensor(g_np[1])[None].to(DEV), _script_dists_tensor(o_np[1])[None].to(DEV)).item()


def _calls(lp, di, x, y, u8):
    with torch.no_grad():
        return [lp(x, y), di(x, y), calculate_lpips(*u8, lp), calculate_dists(*u8, di)]


def test_bitwise_reproducible_deterministic_and_without_host_sync():
    """two calls of each form under torch.use_deterministic_algorithms(True), the second with host synchronisation an error"""
    lp, di = _lpips(), _dists()
    x, y = _pair((2, 3, 64, 96), "noisy")
    u8 = _u8_pair(2, 40, 56)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = _calls(lp, di, x, y, u8)
        torch.cuda.set_sync_debug_mode("error")
        try:
            b = _calls(lp, di, x, y, u8)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    finally:
        torch.use_deterministic_algorithms(old)
    assert all(torch.equal(p, q) for p, q in zip(a, b))


def test_cuda_graph_replays_equal_to_eager():
    lp, di = _lpips(), _dists()
    x0, y0 = _pair((2, 3, 40, 72), "noisy")
    x, y = x0.clone(), y0.clone()
    with torch.no_grad():
        want = [lp(x0, y0), di(x0, y0)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):  # cuDNN's algorithm choice outside the capture
                lp(x, y), di(x, y)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            got = [lp(x, y), di(x, y)]
        x.copy_(torch.rand_like(x))
        graph.replay()
        x.copy_(x0)
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_launch_census():
    """per call: DESIGN §1.12's library launches, and one cuDNN convolution per VGG16 convolution"""
    lp, di = _lpips(), _dists()
    x, y = _pair((2, 3, 64, 64), "unrelated")
    for m, want in ((lp, LPIPS_LAUNCHES), (di, DISTS_LAUNCHES)):
        with torch.no_grad():
            m(x, y)
            n0 = ops.launch_count()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
                m(x, y)
        assert ops.launch_count() - n0 == want
        assert [e.name for e in prof.events()].count("aten::convolution") == 13


def test_input_validation():
    lp, di = _lpips(), _dists()
    x, y = _pair((2, 3, 32, 32), "unrelated")
    for m in (lp, di):
        with pytest.raises(ValueError):
            m(x.double(), y.double())
        with pytest.raises(ValueError):
            m(x, y[:, :, :31])
        with pytest.raises(ValueError):
            m(x[:, :2], y[:, :2])
        with pytest.raises(ValueError):
            m(x.cpu(), y.cpu())
    with pytest.raises(ValueError):
        lp(x[:, :, :15], y[:, :, :15])
    with pytest.raises(ValueError):
        calculate_lpips(*_u8_pair(1, 15, 32), lp)
    with pytest.raises(NotImplementedError):
        lp(x.requires_grad_(), y)


def test_parity_with_the_lpips_package():
    lpips_pkg = pytest.importorskip("lpips")
    torch.manual_seed(0)
    ref = lpips_pkg.LPIPS(net="vgg", pretrained=False, pnet_rand=True, verbose=False).to(DEV).eval()
    m = LPIPS(pretrained=False, pnet_rand=True).to(DEV)
    assert list(m.state_dict()) == list(ref.state_dict())
    with torch.no_grad():
        for lin in ref.lins:
            lin.model[-1].weight.copy_(torch.rand_like(lin.model[-1].weight))
    m.load_state_dict(ref.state_dict())
    sd = m.state_dict()
    for shape, kind in (((2, 3, 37, 53), "unrelated"), ((1, 3, 64, 48), "noisy")):
        x, y = _pair(shape, kind, lo=-1.0)
        with torch.no_grad():
            got, want32 = m(x, y), ref(x, y)
            v64, _ = lpips_ref.lpips_from_state_dict({k: v.double() for k, v in sd.items()}, x.double(), y.double())
        _within(got, v64, want32, f"lpips package {shape} {kind}")
