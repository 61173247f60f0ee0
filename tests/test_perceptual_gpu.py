"""vmambair_b200.perceptual on the GPU against the float64 torch restatement (oracle/perceptual_ref.py) on the same weights, with random
non-zero biases: the loss and the input gradient for every criterion, both input normalisations, several layer sets and shapes,
bf16 autocast and TF32; frozen parameters, determinism without host synchronisation, CUDA-graph capture, the launch census, and
the recipe's generator step on a small MambaRealSR11.  TF32 is off unless a test says otherwise."""
import pytest
import torch

from oracle import perceptual_ref
from vmambair_b200 import archs, gan, ops
from vmambair_b200.perceptual import PerceptualLoss

pytestmark = pytest.mark.gpu
DEV = "cuda"
RECIPE = {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1, "conv4_4": 1, "conv5_4": 1}
RELU_POOL = {"relu1_1": 0.5, "pool1": 1.0, "conv2_1": 0.3, "relu2_2": 1.0, "pool2": 0.7, "relu3_1": 1.0}
VGG16 = {"conv2_2": 0.5, "relu3_3": 1.0, "pool4": 1.0, "conv5_2": 0.2}


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _make(layers, vgg_type="vgg19", seed=0, **kw):
    torch.manual_seed(seed)
    loss = PerceptualLoss(layers, vgg_type=vgg_type, weights=None, **kw)
    with torch.no_grad():
        for m in loss.vgg.vgg_net:
            if isinstance(m, torch.nn.Conv2d):
                m.bias.normal_(0.0, 0.05)
    feats = perceptual_ref.features_from_state_dict(loss.state_dict(), vgg_type, layers)
    return loss.to(DEV), feats.to(DEV)


def _inputs(shape, seed=1, range_norm=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x, gt = torch.rand(shape, device=DEV, generator=g), torch.rand(shape, device=DEV, generator=g)
    return (2 * x - 1, 2 * gt - 1) if range_norm else (x, gt)


def _ref(feats, vgg_type, layers, x, gt, dtype, autocast=False, **kw):
    """(loss, dx) of the restatement in `dtype` (float64: the reference; float32: torch's own composition)"""
    xr = x.detach().to(dtype).requires_grad_()
    f = feats if dtype == torch.float32 else perceptual_ref.copy_to(feats, dtype)
    with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
        y = perceptual_ref.perceptual_loss(f, vgg_type, layers, xr, gt.to(dtype), **kw)
    y.backward()
    return y.detach().double(), xr.grad.double()


def _ours(loss, x, gt, autocast=False):
    xo = x.detach().clone().requires_grad_()
    with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
        y, style = loss(xo, gt)
    assert style is None and y.dtype == torch.float32 and y.shape == ()
    y.backward()
    return y.detach().double(), xo.grad.double()


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _compare(layers, vgg_type, shape, crit, use_input_norm, range_norm, pw=1.0, autocast=False, tf32=False):
    loss, feats = _make(layers, vgg_type, use_input_norm=use_input_norm, range_norm=range_norm, criterion=crit, perceptual_weight=pw)
    x, gt = _inputs(shape, range_norm=range_norm)
    kw = dict(use_input_norm=use_input_norm, range_norm=range_norm, perceptual_weight=pw, criterion=crit)
    y64, g64 = _ref(feats, vgg_type, layers, x, gt, torch.float64, **kw)
    torch.backends.cudnn.allow_tf32 = tf32
    y, g = _ours(loss, x, gt, autocast)
    y32, g32 = _ref(feats, vgg_type, layers, x, gt, torch.float32, autocast=autocast, **kw)
    el, eg = abs(y.item() - y64.item()) / abs(y64.item()), _rel(g, g64)
    el32, eg32 = abs(y32.item() - y64.item()) / abs(y64.item()), _rel(g32, g64)
    print(f"\n{vgg_type} {crit} {shape} norm={use_input_norm} range={range_norm} autocast={autocast} tf32={tf32}: "
          f"loss err {el:.2e} (torch {el32:.2e}), grad err {eg:.2e} (torch {eg32:.2e})")
    if autocast or tf32:
        assert el <= 2 * el32 and eg <= 2 * eg32
    else:
        assert el <= 1e-5, el
        assert eg <= max(1e-4, 2 * eg32), (eg, eg32)


CASES = [  # (layers, vgg_type, shape, criterion, use_input_norm, range_norm)
    (RECIPE, "vgg19", (2, 3, 256, 256), "l1", True, False),
    (RECIPE, "vgg19", (3, 3, 40, 72), "l1", True, False),
    (RECIPE, "vgg19", (2, 3, 37, 53), "l2", False, True),
    (RECIPE, "vgg19", (1, 3, 16, 16), "fro", True, True),
    (RECIPE, "vgg19", (3, 3, 40, 72), "fro", False, False),
    (RELU_POOL, "vgg19", (2, 3, 37, 53), "l1", False, True),
    (RELU_POOL, "vgg19", (3, 3, 40, 72), "l2", True, False),
    (RELU_POOL, "vgg19", (1, 3, 16, 16), "fro", True, False),
    (VGG16, "vgg16", (2, 3, 37, 53), "l1", True, True),
    (VGG16, "vgg16", (3, 3, 40, 72), "l2", False, False),
]


@pytest.mark.parametrize("layers,vgg_type,shape,crit,norm,rng", CASES)
def test_loss_and_gradient_fp32(layers, vgg_type, shape, crit, norm, rng):
    _compare(layers, vgg_type, shape, crit, norm, rng, pw=0.7)


def test_bf16_autocast():
    _compare(RECIPE, "vgg19", (2, 3, 40, 72), "l1", True, False, autocast=True)


def test_tf32_at_torch_defaults():
    _compare(RECIPE, "vgg19", (2, 3, 64, 64), "l1", True, False, tf32=True)


def test_fro_with_equal_inputs_is_zero_with_zero_gradient():
    loss, _ = _make(RECIPE, criterion="fro")
    x, _ = _inputs((2, 3, 40, 72))
    y, g = _ours(loss, x, x.clone())
    assert y.item() == 0.0 and torch.equal(g, torch.zeros_like(g))


def test_zero_perceptual_weight_returns_none():
    loss, _ = _make(RECIPE, perceptual_weight=0.0)
    x, gt = _inputs((1, 3, 16, 16))
    assert loss(x, gt) == (None, None)


def test_parameters_get_no_gradient():
    loss, _ = _make(RECIPE)
    x, gt = _inputs((2, 3, 40, 72))
    _ours(loss, x, gt)
    assert all(p.grad is None and not p.requires_grad for p in loss.parameters())


def test_bitwise_reproducible_without_host_sync():
    loss, _ = _make(RECIPE)
    x, gt = _inputs((2, 3, 64, 96))

    def run():
        torch.cuda.set_sync_debug_mode("error")
        try:
            return _ours(loss, x, gt)
        finally:
            torch.cuda.set_sync_debug_mode(0)

    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a, b = run(), run()
    finally:
        torch.use_deterministic_algorithms(old)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_cuda_graph_replays_equal_to_eager():
    """under the deterministic flag, so that cuDNN's data-gradient algorithm is deterministic too"""
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        loss, _ = _make(RECIPE)
        x0, gt0 = _inputs((2, 3, 40, 72))
        x = x0.clone().requires_grad_()
        gt = gt0.clone()
        want = _ours(loss, x0, gt0)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):  # warm up cuDNN's algorithm choice outside the capture
                x.grad = None
                loss(x, gt)[0].backward()
        torch.cuda.current_stream().wait_stream(s)
        x.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = loss(x, gt)[0]
            y.backward()
        with torch.no_grad():
            x.copy_(torch.rand_like(x))
            gt.copy_(torch.rand_like(gt))
        graph.replay()
        with torch.no_grad():
            x.copy_(x0)
            gt.copy_(gt0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y.detach().double(), want[0]) and torch.equal(x.grad.double(), want[1])
    finally:
        torch.use_deterministic_algorithms(old)


def test_launch_census():
    """per call: the normalisation, a stage per convolution and the loss forward; a stage per convolution and the normalisation's
    adjoint backward; one cuDNN convolution and one data-gradient convolution per VGG convolution"""
    loss, _ = _make(RECIPE)
    x, gt = _inputs((2, 3, 64, 64))
    n_conv = 16
    _ours(loss, x, gt)
    n0 = ops.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        _ours(loss, x, gt)
    names = [e.name for e in prof.events()]
    assert ops.launch_count() - n0 == (1 + n_conv + 1) + (n_conv + 1)
    assert names.count("aten::convolution") == n_conv
    assert names.count("aten::convolution_backward") == n_conv


def test_generator_step_with_mambarealsr11():
    """The recipe's generator step on a small MambaRealSR11: l_g_pix (L1) + l_g_percep + l_g_gan (UNetDiscriminatorSN frozen), with
    the drop-ins and with the restated perceptual loss in float64 and float32; the gradient at the generator's output is compared
    within the fp32 bounds."""
    torch.manual_seed(11)
    net_g = archs.MambaRealSR11(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    lq = torch.rand(2, 3, 16, 16, device=DEV)
    gt = torch.rand(2, 3, 64, 64, device=DEV)
    out = net_g(lq)
    net_d = gan.UNetDiscriminatorSN(3, num_feat=16).to(DEV)
    for p in net_d.parameters():
        p.requires_grad_(False)
    cri_gan = gan.GANLoss("vanilla", loss_weight=0.1)
    percep, feats = _make(RECIPE)
    grads = {}
    for impl in ("ours", "ref64", "ref32"):
        dt = torch.float64 if impl == "ref64" else torch.float32
        o = out.detach().to(dt).requires_grad_()
        l_pix = torch.nn.functional.l1_loss(o, gt.to(dt))
        if impl == "ours":
            l_percep = percep(o, gt)[0]
        else:
            f = perceptual_ref.copy_to(feats, dt)
            l_percep = perceptual_ref.perceptual_loss(f, "vgg19", RECIPE, o, gt.to(dt))
        net_d.eval()  # no u / v update: the three implementations see the same discriminator
        l_gan = cri_gan(net_d(o.float()), True, is_disc=False)
        (l_pix + l_percep + l_gan).backward()
        grads[impl] = o.grad.double()
    eg, eg32 = _rel(grads["ours"], grads["ref64"]), _rel(grads["ref32"], grads["ref64"])
    assert eg <= max(1e-4, 2 * eg32), (eg, eg32)
    torch.autograd.backward(out, grads["ours"].float())  # and into the generator
    assert all(torch.isfinite(p.grad).all() for p in net_g.parameters() if p.grad is not None)


@pytest.mark.parametrize("shape", [(2, 3, 15, 64), (2, 3, 64, 8)])
def test_too_small_raises(shape):
    loss, _ = _make(RECIPE)
    with pytest.raises(ValueError):
        loss(torch.rand(shape, device=DEV), torch.rand(shape, device=DEV))
