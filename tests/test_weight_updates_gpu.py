"""Inference after every kind of weight update, against float64.

Validation runs no-grad inference on the network being trained, in the same process, between training steps.  The inference path keeps
converted copies of the weights -- the OSS blocks' kernel layout (fused._prepare), the U-Net convolutions' (unet._cached), the SR
tail's channels-last copy (MambaSISR6._tail_channels_last) and PerceptualLoss's bf16 VGG weights -- and rebuilds one when a parameter's
_version or data_ptr changes.  Each case builds a tiny network (one block per stage, dim 16), runs inference once (which fills those
caches: y_stale), applies one kind of weight update, runs inference again (y) and evaluates oss_ref.net_forward in float64 on the
network's current state_dict (y64).  Two assertions per case:

  correct   y within the bound of the suite's net-level inference checks: fp32 rtol 1e-3 / atol 1e-4 element-wise
            (tests/test_modules_gpu.py), bf16 the bound of tests/test_bench_parity_gpu.py against the oracle with bf16 storage;
  can fail  y_stale breaks that bound by at least 20 x, so that a cache which missed the update could not pass.

The updates use a learning rate of 1e-2 (the recipes' 2e-4 moves the output by about the tolerance).  The fp32 input, 2 x 24 x 40,
reaches the direction-aware scan at levels 1 and 2 (L % 8 == 0), the gathered path at level 3 (6 x 10) and the latent level (3 x 5),
the library's U-Net convolutions and, on the SR networks, the tail's channels-last path; the bf16 case at 128 x 128 reaches
merge_norm_gate's single-kernel path at level 1."""
import copy

import pytest
import torch

from oracle import cscan, oss_ref, perceptual_ref
from vmambair_b200 import archs, fused_train, gan, gan_train, restore_train
from vmambair_b200.optim import FlatAdam
from vmambair_b200.perceptual import PerceptualLoss

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LR = 1e-2
MARGIN = 20.0
NETS = {"sisr": archs.MambaSISR6, "realsr": archs.MambaRealSR11, "mamber32": archs.Mamber32}
MODEL = {"sisr": "MambaSISRModel", "realsr": "MambaRealSR"}


@pytest.fixture(autouse=True)
def _setup():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    cscan.use_host_threads()
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    fused_train.set_direct_grads(False)  # FlatAdam switches the direct .grad accumulation on; other test modules expect autograd's route


# ---------------------------------------------------------------------------------------------------------------- fixtures
def _net(kind, seed=0):
    torch.manual_seed(seed)
    return NETS[kind](dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()


def _sr_opt(kind, ema=0.999):
    """SISR stage 1 (MambaSISR15_x4.yml) / Real-ESRNet (mambaSR11_x4.yml), the keys the step reads, lr raised to LR"""
    return {"model_type": MODEL[kind], "scale": 4,
            "train": {"ema_decay": ema, "optim_g": {"type": "Adam", "lr": LR, "weight_decay": 0, "betas": [0.9, 0.99]},
                      "scheduler": {"type": "MultiStepLR", "milestones": [50000, 70000], "gamma": 0.5}, "warmup_iter": -1,
                      "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"}}}


def _derain_opt(lr=LR):
    """Deraining_mamber32.yml, the keys the step reads (AdamW, clip_grad_norm_(0.01), cosine restarts, mixup), lr raised; one batch
    as it comes (no progressive subset or crop)"""
    return {"model_type": "ImageCleanModel", "scale": 1, "datasets": {"train": {}},
            "train": {"warmup_iter": -1, "use_grad_clip": True,
                      "scheduler": {"type": "CosineAnnealingRestartCyclicLR", "periods": [48000, 96000], "restart_weights": [1, 1],
                                    "eta_mins": [0.000285, 0.000001]},
                      "mixing_augs": {"mixup": True, "mixup_beta": 1.2, "use_identity": False},
                      "optim_g": {"type": "AdamW", "lr": lr, "weight_decay": 1e-4, "betas": [0.9, 0.999]},
                      "pixel_opt": {"type": "L1Loss", "loss_weight": 1, "reduction": "mean"}}}


def _gan_opt():
    """mambaSR11GAN_x4.yml without the perceptual loss (no VGG file needed), the generator's lr (optim_g and lr_sr) raised to LR"""
    return {"model_type": "MambaRealSRGAN", "l1_gt_usm": True, "percep_gt_usm": True, "gan_gt_usm": False,
            "train": {"ema_decay": 0.999,
                      "optim_g": {"type": "Adam", "lr": LR, "weight_decay": 0, "betas": [0.9, 0.99]},
                      "optim_d": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                      "scheduler": {"type": "MultiStepLR", "milestones": [400000], "gamma": 0.5},
                      "lr_sr": LR, "gamma_sr": 0.5, "lr_decay_sr": 100000, "warmup_iter": -1,
                      "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"},
                      "gan_opt": {"type": "GANLoss", "gan_type": "vanilla", "real_label_val": 1.0, "fake_label_val": 0.0,
                                  "loss_weight": 0.1},
                      "net_d_iters": 1, "net_d_init_iters": 0}}


def _batch(kind, seed=3, size=16):
    """a training batch: 2 x 16^2 LQ with 4 x GT for the SR networks, 2 x 32^2 pairs for deraining"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    s, h = (4, size) if kind in MODEL else (1, 2 * size)
    return torch.rand(2, 3, h, h, device=DEV, generator=g), torch.rand(2, 3, s * h, s * h, device=DEV, generator=g)


def _restore_trainer(net, kind, lr=LR, **kw):
    return restore_train.RestorationTrainer(net, _sr_opt(kind) if kind in MODEL else _derain_opt(lr), **kw)


def _infer(net, x):
    """the recipes' validation: eval mode, no grad"""
    net.eval()
    try:
        with torch.no_grad():
            return net(x).clone()
    finally:
        net.train()


def _oracle(net, x, kind, store=None):
    """oss_ref.net_forward in float64 (torch ops on the GPU, the scan on the CPU) on the network's current weights; store: STORE_DTYPE"""
    sd = {k: v.detach().to(torch.float64).clone() for k, v in net.state_dict().items()}
    oss_ref.STORE_DTYPE = store
    try:
        with torch.no_grad():
            return oss_ref.net_forward(sd, x.to(torch.float64), kind)
    finally:
        oss_ref.STORE_DTYPE = None


# ---------------------------------------------------------------------------------------------------------------- updates
# each update: prepare(net, kind) runs before the first inference (a trainer or optimizer re-points the parameters into its flat
# buffer there, which changes their data_ptr) and returns apply(), the update itself, run between the two inferences
def _flat_adam(net, kind):
    opt = FlatAdam(net.parameters(), lr=LR, betas=(0.9, 0.99))

    def apply():
        g = torch.Generator(device=DEV).manual_seed(5)
        for p in opt.params:
            p.grad.copy_(torch.randn(p.shape, device=DEV, generator=g))
        opt.step()
    return apply


def _restore_eager(net, kind):
    tr = _restore_trainer(net, kind)
    return lambda: [tr.step(*_batch(kind, seed)) for seed in (3, 4)]


def _restore_replay(net, kind):
    tr = _restore_trainer(net, kind)
    lq, gt = _batch(kind)
    tr.capture(lq, gt)
    return lambda: [tr.step(lq, gt) for _ in range(2)]


def _gan(replay):
    def prepare(net, kind):
        torch.manual_seed(1)
        net_d = gan.UNetDiscriminatorSN(3, num_feat=16).to(DEV).train()
        tr = gan_train.GANTrainer(net, net_d, _gan_opt(), 4)
        lq, gt = _batch(kind)
        if replay:
            tr.capture(lq, gt)
        assert tr.g_step_at(tr.iter + 1)

        def apply():
            for _ in range(2):
                tr.step(lq, gt)
            assert (tr.graph is not None) == replay
        return apply
    return prepare


def _adamw(net, kind):
    opt = torch.optim.AdamW(net.parameters(), lr=LR)

    def apply():
        g = torch.Generator(device=DEV).manual_seed(5)
        for p in net.parameters():
            p.grad = torch.randn(p.shape, device=DEV, generator=g)
        opt.step()
    return apply


def _scale(name):
    """an in-place torch op on one parameter, under no_grad"""
    def prepare(net, kind):
        p = dict(net.named_parameters())[name]

        def apply():
            with torch.no_grad():
                p.mul_(3.0)
        return apply
    return prepare


def _new_storage(net, kind):
    def apply():
        g = torch.Generator(device=DEV).manual_seed(6)
        for p in net.parameters():
            p.data = p.detach() + 2 * LR * torch.randn(p.shape, device=DEV, generator=g)
    return apply


UPDATES = {"flat_adam": _flat_adam, "restore_eager": _restore_eager, "restore_replay": _restore_replay, "gan_eager": _gan(False),
           "gan_replay": _gan(True), "adamw": _adamw, "new_storage": _new_storage,
           "mul_block": _scale("encoder_level1.0.attn.out_conv.weight"), "mul_unet_conv": _scale("patch_embed.proj.weight"),
           "mul_tail_conv": _scale("tail.0.0.weight")}
CASES = [("flat_adam", "sisr"), ("flat_adam", "realsr"), ("flat_adam", "mamber32"),
         ("restore_eager", "sisr"), ("restore_eager", "mamber32"), ("restore_replay", "sisr"), ("restore_replay", "mamber32"),
         ("gan_eager", "realsr"), ("gan_replay", "realsr"),
         ("adamw", "mamber32"), ("new_storage", "realsr"),
         ("mul_block", "sisr"), ("mul_unet_conv", "sisr"), ("mul_tail_conv", "sisr")]


def _fp32_ratio(y, y64):
    """max over elements of |y - y64| / (atol + rtol |y64|): <= 1 is assert_close(rtol=1e-3, atol=1e-4)"""
    return float(((y.double() - y64).abs() / (1e-4 + 1e-3 * y64.abs())).max())


def _check_fp32(tag, y_stale, y, y64):
    r, r_stale = _fp32_ratio(y, y64), _fp32_ratio(y_stale, y64)
    print(f"\n{tag}: after the update {r:.3g} x the bound, the output before it {r_stale:.3g} x")
    assert r_stale >= MARGIN, f"{tag}: the update moved the output by only {r_stale:.3g} x the bound: this case cannot fail"
    torch.testing.assert_close(y.double(), y64, rtol=1e-3, atol=1e-4, msg=lambda m: f"{tag}: {m}")


@pytest.mark.parametrize("update,kind", CASES)
def test_inference_follows_the_update(update, kind):
    net = _net(kind)
    apply = UPDATES[update](net, kind)
    x = torch.rand(2, 3, 24, 40, device=DEV, generator=torch.Generator(device=DEV).manual_seed(11))
    y_stale = _infer(net, x)
    apply()
    y = _infer(net, x)
    _check_fp32(f"{update} {kind}", y_stale, y, _oracle(net, x, kind))


def test_inference_follows_the_ema_weights_loaded():
    """the recipes' net_g_ema: a second network that receives the trainer's EMA weights through load_state_dict"""
    net = _net("sisr")
    net_ema = copy.deepcopy(net)
    tr = restore_train.RestorationTrainer(net, _sr_opt("sisr", ema=0.5))
    x = torch.rand(2, 3, 24, 40, device=DEV, generator=torch.Generator(device=DEV).manual_seed(11))
    y_stale = _infer(net_ema, x)
    for seed in (3, 4):
        tr.step(*_batch("sisr", seed))
    net_ema.load_state_dict(tr.ema_state_dict(), strict=True)
    y = _infer(net_ema, x)
    _check_fp32("load_state_dict(ema_state_dict()) sisr", y_stale, y, _oracle(net_ema, x, "sisr"))


def test_bf16_inference_follows_graph_replays():
    """Deraining under bf16 autocast with the iteration captured and replayed; inference on bf16 input at 128 x 128, where level 1
    (C = 16) takes merge_norm_gate's single-kernel path.  Bound of tests/test_bench_parity_gpu.py: mean |err| <= 1.5 x and max |err|
    <= 3 x the bf16-storage oracle's (+ 1e-3 / 1e-2), and at most 0.05 / 0.5.  At 1e-2 a few steps throw this network's output
    far out of its range, and the bf16 bound with it; three steps at 2e-3 (ten times the recipes' rate) keep it in range"""
    net = _net("mamber32")
    tr = _restore_trainer(net, "mamber32", lr=2e-3, dtype=torch.bfloat16)
    lq, gt = _batch("mamber32")
    tr.capture(lq, gt)
    x = torch.rand(1, 3, 128, 128, device=DEV, generator=torch.Generator(device=DEV).manual_seed(12)).to(torch.bfloat16)
    y_stale = _infer(net, x)
    for _ in range(3):
        tr.step(lq, gt)
    y = _infer(net, x)
    ref, emu = _oracle(net, x, "mamber32"), _oracle(net, x, "mamber32", store=torch.bfloat16)
    e_emu = (emu - ref).abs()
    lim_mean, lim_max = 1.5 * float(e_emu.mean()) + 1e-3, 3.0 * float(e_emu.max()) + 1e-2
    err, err_stale = (y.double() - ref).abs(), (y_stale.double() - ref).abs()
    r = max(float(err.mean()) / lim_mean, float(err.max()) / lim_max)
    r_stale = max(float(err_stale.mean()) / lim_mean, float(err_stale.max()) / lim_max)
    print(f"\nbf16 replay mamber32: max {float(err.max()):.4f} mean {float(err.mean()):.5f} ({r:.3g} x the bound), before the update "
          f"max {float(err_stale.max()):.4f} mean {float(err_stale.mean()):.5f} ({r_stale:.3g} x); bf16-storage oracle max "
          f"{float(e_emu.max()):.4f} mean {float(e_emu.mean()):.5f}")
    assert r_stale >= MARGIN, f"the update moved the output by only {r_stale:.3g} x the bound: this case cannot fail"
    assert torch.isfinite(y).all()
    assert float(err.mean()) <= lim_mean and float(err.max()) <= lim_max
    assert float(err.mean()) <= 0.05 and float(err.max()) <= 0.5


# ---------------------------------------------------------------------------------------------------------------- PerceptualLoss
LAYERS = {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1.0, "conv4_4": 1.0, "conv5_4": 1.0}


def _percep_ours(loss, x, gt):
    xo = x.detach().clone().requires_grad_()
    with torch.autocast("cuda", torch.bfloat16):
        y = loss(xo, gt)[0]
    y.backward()
    return y.detach().double(), xo.grad.double()


def _percep_ref(feats, x, gt, dtype):
    f = feats if dtype == torch.float32 else perceptual_ref.copy_to(feats, dtype)
    xr = x.detach().to(dtype).requires_grad_()
    with torch.autocast("cuda", torch.bfloat16, enabled=dtype == torch.float32):
        y = perceptual_ref.perceptual_loss(f, "vgg19", LAYERS, xr, gt.to(dtype))
    y.backward()
    return y.detach().double(), xr.grad.double()


def test_perceptual_loss_follows_loaded_vgg_weights():
    """bf16 autocast keeps bf16 copies of the VGG weights; after load_state_dict of a second set, loss and input gradient follow
    oracle/perceptual_ref in float64 on the new weights within 2 x the error of torch's fp32 composition under the same autocast
    (tests/test_perceptual_gpu.py).  That composition's gradient is ~15-25 % of max|dx| off under bf16, and a second random set of
    the same scale moves dx by about 5 times that; the second set is the first with its convolution weights scaled by 0.6, which
    shrinks loss and gradient about ten- and sixtyfold, so that the first weights' results break both bounds by 20 x."""
    torch.manual_seed(0)
    loss = PerceptualLoss(LAYERS, vgg_type="vgg19", weights=None)
    with torch.no_grad():
        for m in loss.vgg.vgg_net:
            if isinstance(m, torch.nn.Conv2d):
                m.bias.normal_(0.0, 0.05)  # non-zero biases, as tests/test_perceptual_gpu.py
    loss = loss.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(1)
    x, gt = torch.rand(2, 3, 64, 64, device=DEV, generator=g), torch.rand(2, 3, 64, 64, device=DEV, generator=g)
    stale = _percep_ours(loss, x, gt)
    sd = {k: v * 0.6 if k.endswith(".weight") else v.clone() for k, v in loss.state_dict().items()}
    loss.load_state_dict(sd)
    y, dx = _percep_ours(loss, x, gt)
    feats = perceptual_ref.features_from_state_dict(sd, "vgg19", LAYERS).to(DEV)
    y64, g64 = _percep_ref(feats, x, gt, torch.float64)
    y32, g32 = _percep_ref(feats, x, gt, torch.float32)
    rel = lambda a, b: float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
    el, eg, el32, eg32 = rel(y, y64), rel(dx, g64), rel(y32, y64), rel(g32, g64)
    el_stale, eg_stale = rel(stale[0], y64), rel(stale[1], g64)
    print(f"\nloss err {el:.2e} (torch {el32:.2e}, before the load {el_stale:.2e}), grad err {eg:.2e} (torch {eg32:.2e}, before "
          f"the load {eg_stale:.2e})")
    assert el_stale >= MARGIN * 2 * el32 and eg_stale >= MARGIN * 2 * eg32, "the second weights do not move the loss: this case cannot fail"
    assert el <= 2 * el32 and eg <= 2 * eg32
