"""GANTrainer on the CPU: the learning-rate schedule the device kernel computes (restated by gan_train.LrRule.at) against the reference
formula and torch's MultiStepLR across decay boundaries, the option parsing of both GAN recipes' train sections, and the ABI mirrors of
the step's argument structs."""
import ctypes as C

import pytest
import torch

from vmambair_b200 import _lib, gan_train, ops

# the train sections (and the top-level keys the step reads) of RealSR/options/mambaSR11GAN_x4.yml and
# SRGAN/options/MambaSISR15GAN_x4.yml
_LOSSES = {
    "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"},
    "perceptual_opt": {"type": "PerceptualLoss", "layer_weights": {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1, "conv4_4": 1,
                                                                     "conv5_4": 1},
                       "vgg_type": "vgg19", "use_input_norm": True, "perceptual_weight": 1.0, "style_weight": 0, "range_norm": False,
                       "criterion": "l1"},
    "gan_opt": {"type": "GANLoss", "gan_type": "vanilla", "real_label_val": 1.0, "fake_label_val": 0.0, "loss_weight": 1.0},
    "net_d_iters": 1, "net_d_init_iters": 0,
}
REALSR = {"model_type": "MambaRealSRGAN", "scale": 4, "l1_gt_usm": False, "percep_gt_usm": False, "gan_gt_usm": False,
          "train": {"ema_decay": 0.999,
                    "optim_g": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                    "optim_d": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                    "scheduler": {"type": "MultiStepLR", "milestones": [400000], "gamma": 0.5},
                    "total_iter": 400000, "lr_sr": 1e-4, "gamma_sr": 0.5, "lr_decay_sr": 300000, "warmup_iter": -1, **_LOSSES}}
SISR = {"model_type": "MambaSISRGANModel", "scale": 4,
        "train": {"ema_decay": 0.999,
                  "optim_g": {"type": "Adam", "lr": 2e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                  "optim_d": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                  "scheduler": {"type": "MultiStepLR", "milestones": [150000], "gamma": 0.5},
                  "total_iter": 300000, "lr_sr": 2e-4, "gamma_sr": 0.5, "lr_decay_sr": 225000, "warmup_iter": -1, **_LOSSES}}


def _multistep(base, milestones, gamma, iters):
    """lr of torch's MultiStepLR as basicsr's update_learning_rate leaves it at iterations 1..iters (stepped from iteration 2 on)"""
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=base)
    sched = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=list(milestones), gamma=gamma)
    out = []
    for it in range(1, iters + 1):
        if it > 1:
            opt.step()
            sched.step()
        out.append(opt.param_groups[0]["lr"])
    return out


def test_generator_step_decay_matches_the_reference_formula():
    rule = gan_train.parse_options(REALSR).lr_g
    for it in (1, 2, 299999, 300000, 300001, 599999, 600000, 900000):
        ref = 1e-4 * 0.5 ** (it // 300000)  # MambaRealSRGAN_model.py:290
        assert rule.at(it) == pytest.approx(ref, rel=1e-15), it


@pytest.mark.parametrize("milestones,gamma", [([3], 0.5), ([2, 5, 6], 0.1), ([1, 4], 0.5)])
def test_multistep_matches_torch(milestones, gamma):
    rule = gan_train.LrRule(2e-4, milestones=tuple(milestones), milestone_gamma=gamma)
    want = _multistep(2e-4, milestones, gamma, 9)
    got = [rule.at(it) for it in range(1, 10)]
    assert got == pytest.approx(want, rel=1e-12)


def test_both_factors_together():
    rule = gan_train.LrRule(1.0, 0.5, 3, (4,), 0.1)
    assert [rule.at(it) for it in range(1, 8)] == pytest.approx([1, 1, 0.5, 0.5, 0.05, 0.025, 0.025])


def test_realsr_options():
    o = gan_train.parse_options(REALSR)
    assert o.model_type == "MambaRealSRGAN" and (o.l1_gt_usm, o.percep_gt_usm, o.gan_gt_usm) == (False, False, False)
    assert o.lr_g == gan_train.LrRule(1e-4, 0.5, 300000)
    assert o.lr_d == gan_train.LrRule(1e-4, milestones=(400000,), milestone_gamma=0.5)
    assert o.optim_g == {"lr": 1e-4, "betas": (0.9, 0.99), "eps": 1e-8, "weight_decay": 0.0} == o.optim_d
    assert o.ema_decay == 0.999 and o.pixel_weight == 1.0 and (o.net_d_iters, o.net_d_init_iters) == (1, 0)
    assert "type" not in o.perceptual_opt and o.perceptual_opt["vgg_type"] == "vgg19"
    assert o.gan_opt == {"gan_type": "vanilla", "real_label_val": 1.0, "fake_label_val": 0.0, "loss_weight": 1.0}
    on = dict(REALSR, l1_gt_usm=True, gan_gt_usm=True)
    o = gan_train.parse_options(on)
    assert (o.l1_gt_usm, o.percep_gt_usm, o.gan_gt_usm) == (True, False, True)


def test_sisr_options():
    o = gan_train.parse_options(SISR)
    assert o.model_type == "MambaSISRGANModel" and not (o.l1_gt_usm or o.percep_gt_usm or o.gan_gt_usm)
    assert o.lr_g == gan_train.LrRule(2e-4, milestones=(150000,), milestone_gamma=0.5)
    assert o.lr_d == gan_train.LrRule(1e-4, milestones=(150000,), milestone_gamma=0.5)
    assert o.lr_g.at(150000) == 2e-4 and o.lr_g.at(150001) == 1e-4


@pytest.mark.parametrize("change", [
    {"model_type": "SRGANModel"},
    {"train": dict(SISR["train"], optim_g={"type": "AdamW", "lr": 1e-4})},
    {"train": dict(SISR["train"], warmup_iter=100)},
    {"train": dict(SISR["train"], pixel_opt={"type": "MSELoss", "loss_weight": 1.0})},
    {"train": dict(SISR["train"], scheduler={"type": "CosineAnnealingRestartLR", "periods": [10]})},
])
def test_unimplemented_options_raise(change):
    with pytest.raises(NotImplementedError):
        gan_train.parse_options(dict(SISR, **change))


def test_abi_mirrors_of_the_step_structs():
    """field layout of the new mirrors (tests/test_abi_cpu.py checks them against the header) and the rule a schedule passes"""
    assert {f for f, _ in _lib.AdamArgs._fields_} >= {"lr", "lr_dev"}
    assert _lib.LrRule.milestones.size == 8 * _lib.LR_MAX_MILESTONES
    r = ops.lr_rule(1e-4, 0.5, 300000, (400000, 500000), 0.1)
    assert (r.base, r.step_gamma, r.step_size, r.n_milestones, list(r.milestones)[:3]) == \
        (1e-4, 0.5, 300000, 2, [400000, 500000, 0])
    a = _lib.LrScheduleArgs(iter=None, lr=None, rule=(_lib.LrRule * 2)(r), n_rules=1)
    assert a.rule[0].milestones[1] == 500000 and a.rule[1].n_milestones == 0
    assert C.sizeof(_lib.GanOutGradArgs) > 0 and C.sizeof(_lib.MeanLossArgs) > 0
    with pytest.raises(ValueError):
        ops.lr_rule(1.0, milestones=tuple(range(_lib.LR_MAX_MILESTONES + 1)))
