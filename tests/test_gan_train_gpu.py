"""GANTrainer and its kernels (csrc/gan_step.cu) on the GPU: the pixel loss / logit mean and the output-gradient junction against
float64 torch, the schedule kernel against LrRule, Adam with the learning rate read on the device against the host value, whole
iterations against the recipe's optimize_parameters composed from torch modules, CUDA-graph replays against eager steps, and a step
without host synchronisation."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import gan_ref, perceptual_ref
from vmambair_b200 import archs, gan, gan_train, ops
from vmambair_b200.degradations import USMSharp
from vmambair_b200.optim import FlatAdam
from vmambair_b200.perceptual import PerceptualLoss

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LAYERS = {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1.0, "conv4_4": 1.0, "conv5_4": 1.0}


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _opt(l1_usm=False, percep_usm=False, gan_usm=False, init_iters=0):
    """a RealSR recipe scaled down so that a few iterations cross the generator's decay and the discriminator's milestone"""
    return {"model_type": "MambaRealSRGAN", "l1_gt_usm": l1_usm, "percep_gt_usm": percep_usm, "gan_gt_usm": gan_usm,
            "train": {"ema_decay": 0.9,
                      "optim_g": {"type": "Adam", "lr": 2e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                      "optim_d": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                      "scheduler": {"type": "MultiStepLR", "milestones": [2], "gamma": 0.5},
                      "lr_sr": 2e-4, "gamma_sr": 0.5, "lr_decay_sr": 3, "warmup_iter": -1,
                      "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"},
                      "perceptual_opt": {"type": "PerceptualLoss", "layer_weights": LAYERS, "vgg_type": "vgg19"},
                      "gan_opt": {"type": "GANLoss", "gan_type": "vanilla", "real_label_val": 1.0, "fake_label_val": 0.0,
                                  "loss_weight": 0.1},
                      "net_d_iters": 1, "net_d_init_iters": init_iters}}


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("n", [1, 255, 257, 4099, 3 * 77 * 93, (1 << 20) + 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_mean_loss_against_float64(n, dtype):
    g = torch.Generator(device=DEV).manual_seed(n)
    x = torch.randn(n, device=DEV, generator=g).to(dtype)
    y = torch.rand(n, device=DEV, generator=g).to(dtype)
    l1 = ops.mean_loss(x, y, 0.7)
    ref = 0.7 * (x.double() - y.double()).abs().mean()
    assert abs(float(l1) - float(ref)) <= 1e-5 * abs(float(ref)) + 1e-7
    m = ops.mean_loss(x)
    ref_m = x.double().mean()
    assert abs(float(m) - float(ref_m)) <= 1e-5 * float(x.double().abs().mean()) + 1e-7
    for _ in range(3):  # one fixed order of summation: bitwise repeatable
        assert torch.equal(ops.mean_loss(x, y, 0.7), l1) and torch.equal(ops.mean_loss(x), m)


@pytest.mark.parametrize("n", [1, 257, 3 * 77 * 93])
@pytest.mark.parametrize("in_dt,out_dt", [(torch.float32, torch.float32), (torch.float32, torch.bfloat16),
                                          (torch.bfloat16, torch.bfloat16)])
@pytest.mark.parametrize("terms", ["both", "gan", "none"])
def test_out_grad_against_float64(n, in_dt, out_dt, terms):
    g = torch.Generator(device=DEV).manual_seed(7 * n)
    out = torch.rand(n, device=DEV, generator=g).to(in_dt)
    gt = torch.rand(n, device=DEV, generator=g).to(in_dt)
    gt[: n // 5] = out[: n // 5]  # sign(0) = 0
    gp = torch.randn(n, device=DEV, generator=g) * 1e-4 if terms == "both" else None
    gg = torch.randn(n, device=DEV, generator=g) * 1e-4 if terms != "none" else None
    d = ops.gan_out_grad(out, gt, gp, gg, 0.8, out_dt)
    assert d.dtype == out_dt and d.shape == out.shape
    ref = 0.8 * torch.sign(out.double() - gt.double()) / n
    for t in (gp, gg):
        if t is not None:
            ref = ref + t.double()
    tol = 1e-6 if out_dt == torch.float32 else 8e-3
    assert float((d.double() - ref).abs().max()) <= tol * float(ref.abs().max())
    # the autograd accumulation it replaces: the sum of the three terms' gradients at the output, in float64
    o = out.double().requires_grad_()
    total = 0.8 * F.l1_loss(o, gt.double())
    for t in (gp, gg):
        if t is not None:
            total = total + (o * t.double()).sum()
    total.backward()
    assert float((d.double() - o.grad).abs().max()) <= tol * float(o.grad.abs().max())


def test_mean_loss_and_out_grad_reject_strided_inputs():
    """the kernels index their inputs linearly: a view with other strides must be refused, not read as if it were dense"""
    big = torch.rand(2, 3, 40, 40, device=DEV)
    crop, dense = big[:, :, 4:36, 4:36], torch.rand(2, 3, 32, 32, device=DEV)
    with pytest.raises(ValueError):
        ops.mean_loss(dense, crop)
    with pytest.raises(ValueError):
        ops.mean_loss(crop)
    with pytest.raises(ValueError):
        ops.gan_out_grad(dense, crop, None, None, 1.0, torch.float32)
    with pytest.raises(ValueError):
        ops.gan_out_grad(dense, dense.clone(), None, torch.rand(2, 3, 32, 64, device=DEV)[..., ::2], 1.0, torch.float32)


def test_lr_schedule_kernel_against_lr_rule():
    rules = [gan_train.LrRule(1e-4, 0.5, 3), gan_train.LrRule(2e-4, milestones=(2, 5), milestone_gamma=0.1)]
    it = torch.zeros(1, dtype=torch.int64, device=DEV)
    lr = torch.zeros(2, dtype=torch.float32, device=DEV)
    for k in range(1, 12):
        ops.lr_schedule(it, lr, [r.c_rule() for r in rules])
        assert int(it) == k
        assert lr.tolist() == pytest.approx([r.at(k) for r in rules], rel=1e-7), k
    it.fill_(299999)
    ops.lr_schedule(it, lr, [gan_train.LrRule(1e-4, 0.5, 300000).c_rule()])
    assert float(lr[0]) == torch.tensor(5e-5, dtype=torch.float32).item()


def test_ema_update():
    g = torch.Generator(device=DEV).manual_seed(3)
    ema, p = torch.randn(100003, device=DEV, generator=g), torch.randn(100003, device=DEV, generator=g)
    ref = 0.999 * ema.double() + 0.001 * p.double()
    ops.ema_update(ema, p, 0.999)
    assert float((ema.double() - ref).abs().max()) <= 1e-6


def test_device_lr_adam_equals_host_lr_adam_bitwise():
    torch.manual_seed(0)
    w0 = torch.randn(1000, 37, device=DEV)
    opts = [FlatAdam([torch.nn.Parameter(w0.clone())], lr=3e-4, betas=(0.9, 0.99), weight_decay=0.01, decoupled=True, ema_decay=0.99)
            for _ in range(2)]
    lr = torch.tensor([3e-4], device=DEV)
    for step in range(3):
        g = torch.randn(1000 * 37, device=DEV)
        for o in opts:
            o.flat_grad.copy_(g)
        opts[0].step()
        opts[1].step(lr_device=lr)
        for k in ("flat_param", "exp_avg", "exp_avg_sq", "ema", "state"):
            assert torch.equal(getattr(opts[0], k), getattr(opts[1], k)), (step, k)


# ---------------------------------------------------------------------------------------------------------------- iterations
def _models(seed=0):
    torch.manual_seed(seed)
    net_g = archs.MambaRealSR11(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    net_d = gan.UNetDiscriminatorSN(3, num_feat=16).to(DEV).train()
    percep = PerceptualLoss(LAYERS, vgg_type="vgg19", weights=None).to(DEV)
    return net_g, net_d, percep


def _batches(k, b=2, lq=16, seed=5):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [(torch.rand(b, 3, lq, lq, device=DEV, generator=g), torch.rand(b, 3, 4 * lq, 4 * lq, device=DEV, generator=g))
            for _ in range(k)]


class _Reference:
    """MambaRealSRGAN's update_learning_rate + optimize_parameters + model_ema composed from torch modules: the generator's compose
    path, oracle/gan_ref's discriminator and loss, oracle/perceptual_ref, torch.optim.Adam, MultiStepLR and a manual EMA"""

    def __init__(self, net_g, net_d, percep, opt):
        self.o, t = opt, opt["train"]
        self.net_g = copy.deepcopy(net_g)
        self.ema = {k: v.detach().clone() for k, v in self.net_g.named_parameters()}
        self.net_d = gan_ref.UNetDiscriminatorSNRef(3, num_feat=16).to(DEV).train()
        self.net_d.load_state_dict(net_d.state_dict())
        self.feats = perceptual_ref.features_from_state_dict(percep.state_dict(), "vgg19", LAYERS).to(DEV)
        self.opt_g = torch.optim.Adam(self.net_g.parameters(), lr=t["optim_g"]["lr"], betas=t["optim_g"]["betas"])
        self.opt_d = torch.optim.Adam(self.net_d.parameters(), lr=t["optim_d"]["lr"], betas=t["optim_d"]["betas"])
        self.sched_d = torch.optim.lr_scheduler.MultiStepLR(self.opt_d, t["scheduler"]["milestones"], t["scheduler"]["gamma"])
        self.usm = USMSharp().to(DEV)

    def iteration(self, it, lq, gt):
        o, t = self.o, self.o["train"]
        if it > 1:
            self.sched_d.step()
        for pg in self.opt_g.param_groups:
            pg["lr"] = t["lr_sr"] * t["gamma_sr"] ** (it // t["lr_decay_sr"])
        gt_usm = self.usm(gt)
        l1_gt, percep_gt, gan_gt = (gt_usm if o[k] else gt for k in ("l1_gt_usm", "percep_gt_usm", "gan_gt_usm"))
        w_gan = t["gan_opt"]["loss_weight"]
        for p in self.net_d.parameters():
            p.requires_grad = False
        self.opt_g.zero_grad()
        output = self.net_g(lq)
        losses = {}
        if it % t["net_d_iters"] == 0 and it > t["net_d_init_iters"]:
            losses["l_g_pix"] = F.l1_loss(output, l1_gt)
            losses["l_g_percep"] = perceptual_ref.perceptual_loss(self.feats, "vgg19", LAYERS, output, percep_gt)
            losses["l_g_gan"] = gan_ref.gan_loss(self.net_d(output), True, is_disc=False, loss_weight=w_gan)
            (losses["l_g_pix"] + losses["l_g_percep"] + losses["l_g_gan"]).backward()
            self.opt_g.step()
        for p in self.net_d.parameters():
            p.requires_grad = True
        self.opt_d.zero_grad()
        real = self.net_d(gan_gt)
        losses["l_d_real"] = gan_ref.gan_loss(real, True, is_disc=True)
        losses["out_d_real"] = torch.mean(real.detach())
        losses["l_d_real"].backward()
        fake = self.net_d(output.detach().clone())
        losses["l_d_fake"] = gan_ref.gan_loss(fake, False, is_disc=True)
        losses["out_d_fake"] = torch.mean(fake.detach())
        losses["l_d_fake"].backward()
        self.opt_d.step()
        with torch.no_grad():
            d = t["ema_decay"]
            for k, p in self.net_g.named_parameters():
                self.ema[k].mul_(d).add_(p, alpha=1 - d)
        return {k: v.detach() for k, v in losses.items()}


@pytest.mark.parametrize("usm", [(True, False, True), (False, True, False)], ids=["l1+gan_usm", "percep_usm"])
def test_iterations_against_the_composed_reference(usm):
    """four iterations: the first skips the G step (net_d_init_iters 1), the generator's lr decays at iteration 3 and the
    discriminator's after its milestone 2; loss dict, both networks' parameters, the EMA and the spectral-norm u, v at 1e-4"""
    prev = archs._TRAIN_PATH
    archs.set_train_path("compose")
    try:
        opt = _opt(*usm, init_iters=1)
        net_g, net_d, percep = _models()
        ref = _Reference(net_g, net_d, percep, opt)
        tr = gan_train.GANTrainer(net_g, net_d, opt, 4, perceptual=percep)
        for it, (lq, gt) in enumerate(_batches(4), 1):
            ours = tr.step(lq, gt)
            want = ref.iteration(it, lq, gt)
            assert set(ours) == set(want), (it, set(ours) ^ set(want))
            for k in want:
                assert abs(float(ours[k]) - float(want[k])) <= 1e-4 * abs(float(want[k])) + 1e-7, (it, k, float(ours[k]), float(want[k]))
            assert float(tr.lr[0]) == pytest.approx(ref.opt_g.param_groups[0]["lr"], rel=1e-6)
            assert float(tr.lr[1]) == pytest.approx(ref.opt_d.param_groups[0]["lr"], rel=1e-6)
            # parameters as whole networks: zero-initialised biases hold a few Adam steps of about +-lr each, whose signs follow
            # gradients that are near zero there
            flat = lambda ts: torch.cat([t.detach().reshape(-1) for t in ts])
            assert _rel(tr.opt_g.flat_param, flat(ref.net_g.parameters())) <= 1e-4, it
            ema = tr.ema_state_dict()
            assert _rel(flat(ema[k] for k in ref.ema), flat(ref.ema.values())) <= 1e-4, it
            sd, sd_ref = net_d.state_dict(), ref.net_d.state_dict()
            params = [k for k in sd_ref if not k.endswith(("weight_u", "weight_v"))]
            assert _rel(flat(sd[k] for k in params), flat(sd_ref[k] for k in params)) <= 1e-4, it
            for k in sd_ref:
                if k.endswith(("weight_u", "weight_v")):
                    assert _rel(sd[k], sd_ref[k]) <= 1e-4, (it, k, _rel(sd[k], sd_ref[k]))
    finally:
        archs.set_train_path(prev)


def _conv_generator():
    """a small generator of cuDNN convolutions, bitwise reproducible (the fused OSS backward is not, DESIGN §6 item 5)"""
    torch.manual_seed(1)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 48, 3, 1, 1), torch.nn.LeakyReLU(0.2), torch.nn.Conv2d(48, 48, 3, 1, 1),
                               torch.nn.PixelShuffle(4)).to(DEV).train()


def test_graph_replays_equal_eager_steps_bitwise():
    prev = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        batches = _batches(10, seed=9)
        runs = {}
        for mode in ("eager", "graph"):
            net_g = _conv_generator()
            _, net_d, percep = _models()
            tr = gan_train.GANTrainer(net_g, net_d, _opt(gan_usm=True), 4, perceptual=percep)
            if mode == "graph":
                tr.capture(*batches[0])
                assert tr.iter == 0 and int(tr.iter_dev) == 0
            losses = [{k: v.clone() for k, v in tr.step(lq, gt).items()} for lq, gt in batches]
            runs[mode] = (losses, tr.opt_g.flat_param.clone(), tr.opt_g.ema.clone(), tr.opt_d.flat_param.clone(),
                          [b.clone() for n, b in net_d.named_buffers()], int(tr.iter_dev), tr.lr.clone())
        (le, *se), (lg, *sg) = runs["eager"], runs["graph"]
        for i, (a, b) in enumerate(zip(le, lg)):
            assert {k: float(v) for k, v in a.items()} == {k: float(v) for k, v in b.items()}, i
        for a, b in zip(se, sg):
            if isinstance(a, list):
                assert all(torch.equal(x, y) for x, y in zip(a, b))
            elif isinstance(a, torch.Tensor):
                assert torch.equal(a, b)
            else:
                assert a == b
    finally:
        torch.backends.cudnn.deterministic = prev


def test_step_without_host_synchronisation():
    net_g, net_d, percep = _models()
    tr = gan_train.GANTrainer(net_g, net_d, _opt(l1_usm=True), 4, perceptual=percep)
    (lq, gt), (lq2, gt2) = _batches(2, seed=3)
    tr.step(lq, gt)  # first call: lazy initialisation of cuDNN and the library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = tr.step(lq2, gt2)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert set(losses) == {"l_g_pix", "l_g_percep", "l_g_gan", "l_d_real", "out_d_real", "l_d_fake", "out_d_fake"}
    assert all(bool(torch.isfinite(v)) for v in losses.values())


def test_cropped_gt_trains_like_its_contiguous_copy():
    """RealESRNetDegradation hands over its GT as a crop of a larger batch (paired_random_crop) until its pair pool fills; with
    l1_gt_usm False that view is the pixel loss's target.  Eager and replayed steps on the crop equal eager steps on a contiguous
    copy bit for bit.  An eager step with the fused generator runs first, so its weight-gradient stream exists, unforked, while
    the conv generator's iteration is captured."""
    net_g, net_d0, percep0 = _models()
    gan_train.GANTrainer(net_g, net_d0, _opt(), 4, perceptual=percep0).step(*_batches(1)[0])
    prev = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        g = torch.Generator(device=DEV).manual_seed(21)
        big = [torch.rand(2, 3, 80, 72, device=DEV, generator=g) for _ in range(3)]
        crops = [b[:, :, 8:72, 4:68] for b in big]
        lqs = [torch.rand(2, 3, 16, 16, device=DEV, generator=g) for _ in range(3)]
        assert not crops[0].is_contiguous()
        runs = {}
        for mode in ("dense", "crop", "crop_graph"):
            _, net_d, percep = _models()
            tr = gan_train.GANTrainer(_conv_generator(), net_d, _opt(), 4, perceptual=percep)
            if mode == "crop_graph":
                tr.capture(lqs[0], crops[0])
            gts = [c.contiguous() for c in crops] if mode == "dense" else crops
            losses = [{k: float(v) for k, v in tr.step(lq, gt).items()} for lq, gt in zip(lqs, gts)]
            runs[mode] = (losses, tr.opt_g.flat_param.clone(), tr.opt_d.flat_param.clone())
        for mode in ("crop", "crop_graph"):
            assert runs[mode][0] == runs["dense"][0], mode
            assert torch.equal(runs[mode][1], runs["dense"][1]) and torch.equal(runs[mode][2], runs["dense"][2]), mode
    finally:
        torch.backends.cudnn.deterministic = prev
