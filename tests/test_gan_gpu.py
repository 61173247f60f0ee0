"""vmambair_b200.gan on the GPU against the float64 torch restatement (oracle/gan_ref.py) on the same state: the recipe's three
train-mode calls per iteration, eval mode, the frozen-D and FlatAdam D steps, the junction kernels, the GAN loss, determinism without
host synchronisation, and one GAN iteration of a small MambaRealSR11 generator.  TF32 is off, for parity."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import gan_ref
from vmambair_b200 import archs, gan, ops
from vmambair_b200.optim import FlatAdam

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _pair(cin, nf, skip, seed=0):
    torch.manual_seed(seed)
    ours = gan.UNetDiscriminatorSN(cin, num_feat=nf, skip_connection=skip).to(DEV)
    ref = gan_ref.UNetDiscriminatorSNRef(cin, num_feat=nf, skip_connection=skip)
    ref.load_state_dict({k: v.cpu() for k, v in ours.state_dict().items()})
    return ours, ref.double().to(DEV)


def _our_loss():
    crit = gan.GANLoss("vanilla", real_label_val=1.0, fake_label_val=0.0, loss_weight=1.0)
    return lambda pred, real, is_disc, loss_weight=1.0: crit(pred, real, is_disc=is_disc)


def _rel(a, b):
    return (a.double() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _close(a, b, tol, what):
    err = _rel(a, b)
    assert err <= tol, f"{what}: max err {err:.3e} of max |ref| {b.abs().max().item():.3e} (bound {tol:.1e})"


def _compare_iteration(ours, ref, B, cin, H, W, tol, tol_uv, autocast=False):
    """The bound of each logits / gradient tensor is `tol` of its max |value|, or twice the error of torch's own composition in the
    same precision (the restatement in float32 on the same state, under the same autocast) where that is larger: at 256 x 256 the G
    step's input gradient is a mean over 65 536 logits with heavy cancellation, and torch's fp32 composition misses it by up to ~3 %
    of its max."""
    g = torch.Generator(device=DEV).manual_seed(1)
    fake = torch.randn(B, cin, H, W, device=DEV, generator=g)
    real = torch.rand(B, cin, H, W, device=DEV, generator=g)
    ref32 = copy.deepcopy(ref).float()
    with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
        got = gan_ref.recipe_iteration(ours, fake, real, loss=_our_loss())
    want = gan_ref.recipe_iteration(ref, fake.double(), real.double())
    with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
        base = gan_ref.recipe_iteration(ref32, fake, real)
    for i, (a, b, c) in enumerate(zip(got, want, base)):
        assert set(a) == set(b)
        for k in a:
            bound = tol_uv if k.endswith((".u", ".v")) else max(tol, 2 * _rel(c[k], b[k]))
            if bound > tol and not k.endswith((".u", ".v")):  # the widened bounds, reported
                print(f"\n{B}x{cin}x{H}x{W} autocast={autocast} call {i} {k}: err {_rel(a[k], b[k]):.2e}, bound {bound:.2e}")
            _close(a[k], b[k], bound, f"call {i} {k}")
    sa, sb = gan_ref.sn_state(ours), gan_ref.sn_state(ref)
    for name in gan_ref.SN_LAYERS:
        _close(sa[name][2], sb[name][2], tol_uv, f"sigma of {name}")


SHAPES = [  # (B, num_in_ch, H, W, num_feat, skip_connection)
    (1, 3, 256, 256, 64, True),
    (2, 3, 8, 8, 16, True),
    (2, 1, 8, 8, 16, False),
    (2, 3, 24, 40, 16, False),
    (3, 1, 24, 40, 8, True),
    (2, 3, 40, 72, 16, True),
    (2, 1, 40, 72, 16, False),
]


@pytest.mark.parametrize("B,cin,H,W,nf,skip", SHAPES)
def test_recipe_iteration_fp32(B, cin, H, W, nf, skip):
    ours, ref = _pair(cin, nf, skip)
    _compare_iteration(ours, ref, B, cin, H, W, tol=1e-4, tol_uv=1e-5)


@pytest.mark.parametrize("skip", [True, False])
def test_recipe_iteration_bf16_autocast(skip):
    ours, ref = _pair(3, 16, skip)
    _compare_iteration(ours, ref, 2, 3, 40, 72, tol=3e-2, tol_uv=1e-5, autocast=True)


def test_frozen_d_writes_no_parameter_gradient():
    ours, ref = _pair(3, 16, True)
    for p in ours.parameters():
        p.requires_grad_(False)
    x = torch.randn(2, 3, 24, 40, device=DEV, requires_grad=True)
    ours(x).square().mean().backward()
    assert all(p.grad is None for p in ours.parameters())
    xr = x.detach().double().requires_grad_()
    ref.train()
    ref(xr).square().mean().backward()
    _close(x.grad, xr.grad, 1e-4, "input gradient")


def test_eval_mode_keeps_u_and_v():
    ours, ref = _pair(3, 16, True)
    ours.eval()
    ref.eval()
    before = {k: v.clone() for k, v in ours.state_dict().items()}
    x = torch.randn(2, 3, 40, 72, device=DEV)
    n0 = ops.launch_count()
    with torch.no_grad():
        y = ours(x)
    launches = ops.launch_count() - n0
    for k, v in ours.state_dict().items():
        assert torch.equal(v, before[k]), k
    with torch.no_grad():
        _close(y, ref(x.double()), 1e-4, "eval logits")
    assert launches == 2 + 3 + 3 + 3  # spectral norm, 6 activations (x6 with its skip), 3 junctions


def test_d_step_accumulates_into_flat_adam_views():
    ours, ref = _pair(3, 16, True)
    opt = FlatAdam(ours.parameters(), lr=1e-4)
    g = torch.Generator(device=DEV).manual_seed(3)
    fake, real = torch.randn(2, 3, 24, 40, device=DEV, generator=g), torch.rand(2, 3, 24, 40, device=DEV, generator=g)
    crit = gan.GANLoss("vanilla")
    crit(ours(real), True, is_disc=True).backward()
    crit(ours(fake), False, is_disc=True).backward()
    for p in ref.parameters():
        p.grad = None
    gan_ref.gan_loss(ref(real.double()), True, is_disc=True).backward()
    gan_ref.gan_loss(ref(fake.double()), False, is_disc=True).backward()
    o = 0
    refp = dict(ref.named_parameters())
    names = {id(p): n for n, p in ours.named_parameters()}
    for p in opt.params:
        assert p.grad.data_ptr() == opt.flat_grad.data_ptr() + 4 * o, names[id(p)]
        _close(opt.flat_grad[o:o + p.numel()].view_as(p), refp[names[id(p)]].grad, 1e-4, names[id(p)])
        o += p.numel()
    opt.step()
    assert torch.isfinite(opt.flat_param).all()


@pytest.mark.parametrize("h,w", [(1, 1), (1, 5), (3, 7), (16, 16), (9, 32)])
@pytest.mark.parametrize("skip", [True, False])
def test_junction_forward_and_adjoint(h, w, skip):
    g = torch.Generator(device=DEV).manual_seed(h * 100 + w)
    pre = torch.randn(2, 5, h, w, device=DEV, generator=g)
    sk = torch.randn(2, 5, h, w, device=DEV, generator=g) if skip else None
    dout = torch.randn(2, 5, 2 * h, 2 * w, device=DEV, generator=g)
    pre64 = pre.double().requires_grad_()
    sk64 = sk.double().requires_grad_() if skip else None
    y64 = F.interpolate(F.leaky_relu(pre64, 0.2) + (sk64 if skip else 0), scale_factor=2, mode="bilinear", align_corners=False)
    y64.backward(dout.double())
    y = ops.gan_up(pre, sk)
    dpre, dskip = ops.gan_up_bwd(dout, pre, skip)
    eps = torch.finfo(torch.float32).eps
    assert (y.double() - y64).abs().max().item() <= 4 * eps * y64.abs().max().item()
    assert (dpre.double() - pre64.grad).abs().max().item() <= 8 * eps * pre64.grad.abs().max().item()
    if skip:
        assert (dskip.double() - sk64.grad).abs().max().item() <= 8 * eps * sk64.grad.abs().max().item()
    else:
        assert dskip is None


def test_activation_backward_adds_the_second_gradient():
    g = torch.Generator(device=DEV).manual_seed(5)
    pre, g1, g2 = (torch.randn(3, 4, 9, 11, device=DEV, generator=g) for _ in range(3))
    pre[0, 0, 0, 0] = 0.0
    y = ops.gan_act(pre.clone())
    assert torch.equal(y, F.leaky_relu(pre, 0.2))
    want = (g1.double() + g2.double()) * torch.where(pre > 0, 1.0, 0.2).double()
    got = ops.gan_act_bwd(g1.clone(), y, g2)
    assert (got.double() - want).abs().max().item() <= 2 * torch.finfo(torch.float32).eps * want.abs().max().item()


@pytest.mark.parametrize("real", [True, False])
@pytest.mark.parametrize("is_disc", [True, False])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gan_loss_value_and_gradient(real, is_disc, dtype):
    g = torch.Generator(device=DEV).manual_seed(int(real) * 2 + int(is_disc))
    x = (torch.randn(3, 1, 40, 24, device=DEV, generator=g) * 6).to(dtype)
    x.view(-1)[:4] = torch.tensor([80.0, -80.0, 0.0, 30.0], dtype=dtype)
    x.requires_grad_()
    crit = gan.GANLoss("vanilla", real_label_val=0.9, fake_label_val=0.1, loss_weight=0.7)
    y = crit(x, real, is_disc=is_disc)
    (2.5 * y).backward()
    x64 = x.detach().double().requires_grad_()
    y64 = gan_ref.gan_loss(x64, real, is_disc, real_label_val=0.9, fake_label_val=0.1, loss_weight=0.7)
    (2.5 * y64).backward()
    assert y.dtype == torch.float32 and y.shape == () and torch.isfinite(y)
    assert abs(y.item() - y64.item()) <= 1e-6 * abs(y64.item())
    assert x.grad.dtype == dtype and torch.isfinite(x.grad.float()).all()
    _close(x.grad, x64.grad, 1e-6 if dtype == torch.float32 else 1e-2, "loss gradient")


def test_bitwise_reproducible_without_host_sync():
    ours, _ = _pair(3, 16, True)
    state = {k: v.clone() for k, v in ours.state_dict().items()}
    g = torch.Generator(device=DEV).manual_seed(7)
    x0 = torch.randn(2, 3, 40, 72, device=DEV, generator=g)
    crit = gan.GANLoss("vanilla")

    def run():
        ours.load_state_dict(state)
        for p in ours.parameters():
            p.grad = None
        x = x0.clone().requires_grad_()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = ours(x)
            crit(y, True, is_disc=False).backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        return [y.detach(), x.grad] + [p.grad for p in ours.parameters()] + [b.clone() for b in ours.buffers()]

    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a, b = run(), run()
    finally:
        torch.use_deterministic_algorithms(old)
    assert len(a) == 2 + 12 + 16
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), i


@pytest.mark.parametrize("shape", [(2, 3, 36, 40), (2, 3, 40, 20), (2, 3, 7, 8)])
def test_sizes_not_multiple_of_8_raise(shape):
    ours, _ = _pair(3, 8, True)
    with pytest.raises(ValueError):
        ours(torch.zeros(shape, device=DEV))


def test_gan_iteration_with_mambarealsr11_generator():
    """One GAN iteration of a small MambaRealSR11 on the fused training path: the G step (G's output through the frozen D, l_g_gan
    into G) and the D step (real + fake passes), with the drop-ins and with the restated D and loss on the same state, the
    restatement in float64 (G's fp32 output cast up) and in float32.  G's fused backward adds with fp32 atomics, so its gradients
    differ run to run; as they are linear in the gradient reaching G's output, G's gradient error is taken from one backward of the
    difference of the two output gradients.  Bound: 2e-3 of each gradient's max |value|, or twice the fp32 restatement's error."""
    torch.manual_seed(11)
    net_g = archs.MambaRealSR11(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    lq = torch.rand(2, 3, 16, 16, device=DEV)
    gt = torch.rand(2, 3, 64, 64, device=DEV)
    out = net_g(lq)
    crit = gan.GANLoss("vanilla")
    dout, d_grads = {}, {}
    for impl in ("ours", "ref64", "ref32"):
        net_d, ref_d = _pair(3, 16, True, seed=12)
        if impl == "ours":
            loss, cast = (lambda pred, real, is_disc: crit(pred, real, is_disc=is_disc)), torch.float32
        else:
            net_d = ref_d if impl == "ref64" else ref_d.float()
            loss, cast = (lambda pred, real, is_disc: gan_ref.gan_loss(pred, real, is_disc)), next(net_d.parameters()).dtype
        for p in net_d.parameters():
            p.requires_grad_(False)
        o = out.detach().to(cast).requires_grad_()
        loss(net_d(o), True, False).backward()
        dout[impl] = o.grad.double()
        for p in net_d.parameters():
            p.requires_grad_(True)
        loss(net_d(gt.to(cast)), True, True).backward()
        loss(net_d(out.detach().to(cast)), False, True).backward()
        d_grads[impl] = {n: p.grad.double() for n, p in net_d.named_parameters()}
    params = [p for p in net_g.parameters() if p.requires_grad]
    names = [n for n, p in net_g.named_parameters() if p.requires_grad]
    jt = lambda d: torch.autograd.grad(net_g(lq), params, d.float(), allow_unused=True)  # a fresh graph per product
    g_ref, g_err, g_err32 = jt(dout["ref64"]), jt(dout["ours"] - dout["ref64"]), jt(dout["ref32"] - dout["ref64"])
    checked = 0
    for n, r, e, e32 in zip(names, g_ref, g_err, g_err32):
        if r is None:
            continue
        scale = max(r.abs().max().item(), 1e-30)
        err, err32 = e.abs().max().item() / scale, e32.abs().max().item() / scale
        assert err <= max(2e-3, 2 * err32), f"G {n}: err {err:.3e} (fp32 restatement {err32:.3e})"
        checked += 1
    assert checked > 0
    for n in d_grads["ours"]:
        _close(d_grads["ours"][n], d_grads["ref64"][n], max(2e-3, 2 * _rel(d_grads["ref32"][n], d_grads["ref64"][n])), f"D {n}")
