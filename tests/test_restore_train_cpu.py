"""RestorationTrainer on the CPU: option parsing of the seven first-stage recipes and its refusals, the cosine schedules the device
kernel computes (restated by gan_train.LrRule.at) against the reference scheduler classes' values in tests/golden/lr_schedules.npz
(tests/golden/make_golden_lr.py), the schedule's end on Deraining_mamber32, the progressive phase lookup and the order of the host's
draws against the reference loop restated in oracle/restore_ref.py, and the ABI mirrors of the new argument structs."""
import copy
import os
import random

import numpy as np
import pytest
import torch

from oracle import restore_ref
from vmambair_b200 import _lib, gan_train, ops, restore_train

# the keys the step reads from SRGAN/options/MambaSISR15_x4.yml, RealSR/options/mambaSR11_x4.yml and mambaSR11m_x4.yml
_SR_TRAIN = {"ema_decay": 0.999, "optim_g": {"type": "Adam", "lr": 2e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
             "warmup_iter": -1, "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"}}
SISR15 = {"model_type": "MambaSISRModel", "scale": 4, "datasets": {"train": {"gt_size": 256, "batch_size_per_gpu": 8}},
          "train": dict(_SR_TRAIN, scheduler={"type": "MultiStepLR", "milestones": [50000, 70000], "gamma": 0.5}, total_iter=100000)}
_REALSR_TRAIN = dict(_SR_TRAIN, scheduler={"type": "MultiStepLR", "milestones": [250000, 350000], "gamma": 0.5}, total_iter=500000,
                     mixing_augs={"mixup": False, "mixup_beta": 1.2, "use_identity": True})
SR11 = {"model_type": "MambaRealSR", "scale": 4, "gt_usm": False, "gt_size": 256,
        "datasets": {"train": {"gt_size": 256, "batch_size_per_gpu": 9}}, "train": _REALSR_TRAIN}
SR11M = dict(SR11, gt_size=32, datasets={"train": {"gt_size": 32, "batch_size_per_gpu": 1}})


def _derain(iters, total, periods, eta_mins, lr, wd):
    """Deraining/Deraining/Options/Deraining_mamber*.yml: the keys the step reads"""
    return {"model_type": "ImageCleanModel", "scale": 1,
            "datasets": {"train": {"batch_size_per_gpu": 8, "mini_batch_sizes": [8, 5, 3, 2, 1, 1], "iters": iters, "gt_size": 384,
                                   "gt_sizes": [128, 160, 192, 256, 320, 384]}},
            "train": {"total_iter": total, "warmup_iter": -1, "use_grad_clip": True,
                      "scheduler": {"type": "CosineAnnealingRestartCyclicLR", "periods": periods, "restart_weights": [1, 1],
                                    "eta_mins": eta_mins},
                      "mixing_augs": {"mixup": False, "mixup_beta": 1.2, "use_identity": True},
                      "optim_g": {"type": "AdamW", "lr": lr, "weight_decay": wd, "betas": [0.9, 0.999]},
                      "pixel_opt": {"type": "L1Loss", "loss_weight": 1, "reduction": "mean"}}}


DERAIN = {
    "mamber28": _derain([92000, 64000, 48000, 36000, 36000, 24000], 300000, [92000, 208000], [0.0003, 0.000001], 3e-4, 1e-4),
    "mamber32": _derain([36000, 24000, 24000, 24000, 24000, 24000], 156000, [48000, 96000], [0.000285, 0.000001], 1e-4, 5e-5),
    "mamber33": _derain([92000, 64000, 64000, 64000, 64000, 48000], 396000, [144000, 288000], [0.0003, 0.000001], 3e-4, 1e-4),
    "mamber34": _derain([92000, 64000, 64000, 64000, 64000, 48000], 396000, [144000, 288000], [0.0003, 0.000001], 3e-4, 1e-4),
}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_schedules.npz")


# ---------------------------------------------------------------------------------------------------------------- options
def test_sr_stage1_options():
    for opt, ms in ((SISR15, (50000, 70000)), (SR11, (250000, 350000)), (SR11M, (250000, 350000))):
        o = restore_train.parse_options(opt)
        assert o.model_type == opt["model_type"] and o.scale == 4 and not o.decoupled and o.max_grad_norm == 0.0
        assert o.optim == {"lr": 2e-4, "betas": (0.9, 0.99), "eps": 1e-8, "weight_decay": 0.0}
        assert o.lr == gan_train.LrRule(2e-4, milestones=ms, milestone_gamma=0.5)
        assert o.ema_decay == 0.999 and o.pixel_weight == 1.0
        assert not o.mixup and o.ends == ()  # mambaSR11 carries mixing_augs, its model ignores them; no progressive keys
        assert restore_train.phase_at(o, 1) == 0 and restore_train.phase_at(o, 10 ** 6) == 0


@pytest.mark.parametrize("name", sorted(DERAIN))
def test_deraining_options(name):
    opt = DERAIN[name]
    o = restore_train.parse_options(opt)
    t, d = opt["train"], opt["datasets"]["train"]
    assert o.model_type == "ImageCleanModel" and o.scale == 1 and o.decoupled and o.max_grad_norm == 0.01 and o.ema_decay == 0.0
    assert o.optim == {"lr": t["optim_g"]["lr"], "betas": (0.9, 0.999), "eps": 1e-8, "weight_decay": t["optim_g"]["weight_decay"]}
    s = t["scheduler"]
    assert o.lr == gan_train.LrRule(t["optim_g"]["lr"], periods=tuple(s["periods"]), restart_weights=(1.0, 1.0),
                                    eta_mins=tuple(s["eta_mins"]))
    assert not o.mixup and o.use_identity and o.mixup_beta == 1.2
    assert o.ends == tuple(np.cumsum(d["iters"])) and o.mini_batch_sizes == (8, 5, 3, 2, 1, 1)
    assert o.gt_sizes == (128, 160, 192, 256, 320, 384) and (o.batch_size, o.gt_size) == (8, 384)


def test_cosine_restart_lr_and_defaults():
    opt = copy.deepcopy(DERAIN["mamber28"])
    t = opt["train"]
    t["scheduler"] = {"type": "CosineAnnealingRestartLR", "periods": [10, 20], "restart_weights": [1, 0.5], "eta_min": 1e-7}
    t["optim_g"] = {"type": "AdamW", "lr": 1e-3}
    t["mixing_augs"] = {"mixup": True}
    del t["use_grad_clip"]
    o = restore_train.parse_options(opt)
    assert o.lr == gan_train.LrRule(1e-3, periods=(10, 20), restart_weights=(1.0, 0.5), eta_mins=(1e-7, 1e-7))
    assert o.optim["weight_decay"] == 1e-2 and o.max_grad_norm == 0.0  # torch.optim.AdamW's default decay; no clip key: no clip
    assert o.mixup and o.mixup_beta == 1.2 and not o.use_identity


def _with(opt, **train):
    opt = copy.deepcopy(opt)
    opt["train"].update(train)
    return opt


@pytest.mark.parametrize("opt", [
    dict(SISR15, model_type="SRModel"),
    dict(SISR15, model_type="MambaRealSRGAN"),
    _with(SISR15, optim_g={"type": "SGD", "lr": 1e-4}),
    _with(SISR15, warmup_iter=100),
    _with(SISR15, pixel_opt={"type": "MSELoss", "loss_weight": 1.0}),
    _with(SISR15, pixel_opt={"type": "L1Loss", "reduction": "sum"}),
    _with(SISR15, perceptual_opt={"type": "PerceptualLoss"}),
    _with(SISR15, scheduler={"type": "MultiStepRestartLR", "milestones": [10], "restarts": [20]}),
    _with(SISR15, scheduler={"type": "CosineAnnealingLR", "T_max": 10}),
], ids=["model", "gan_model", "sgd", "warmup", "mse", "l1_sum", "perceptual", "restarts", "torch_cosine"])
def test_unimplemented_options_raise(opt):
    with pytest.raises(NotImplementedError):
        restore_train.parse_options(opt)


@pytest.mark.parametrize("change", [
    {"scheduler": {"type": "CosineAnnealingRestartCyclicLR", "periods": [10, 20], "restart_weights": [1], "eta_mins": [0, 0]}},
    {"scheduler": {"type": "CosineAnnealingRestartCyclicLR", "periods": [1] * 9, "restart_weights": [1] * 9, "eta_mins": [0] * 9}},
])
def test_inconsistent_schedules_raise(change):
    with pytest.raises(ValueError):
        restore_train.parse_options(_with(DERAIN["mamber28"], **change))


def test_inconsistent_progressive_keys_raise():
    for change in ({"mini_batch_sizes": [8, 5]}, {"mini_batch_sizes": [80] * 6, "batch_size_per_gpu": 80}):
        opt = copy.deepcopy(DERAIN["mamber28"])
        opt["datasets"]["train"].update(change)
        with pytest.raises(ValueError):
            restore_train.parse_options(opt)


def test_gan_trainer_still_refuses_cosine_schedules():
    opt = {"model_type": "MambaSISRGANModel", "train": dict(_SR_TRAIN, optim_d=_SR_TRAIN["optim_g"],
                                                            scheduler=DERAIN["mamber28"]["train"]["scheduler"],
                                                            gan_opt={"type": "GANLoss", "gan_type": "vanilla"})}
    with pytest.raises(NotImplementedError):
        gan_train.parse_options(opt)


# ---------------------------------------------------------------------------------------------------------------- schedules
@pytest.mark.parametrize("name", ["mamber28", "mamber32", "mamber33", "mamber34", "restart"])
def test_cosine_schedules_match_the_reference_classes(name):
    g = np.load(GOLDEN)
    if name == "restart":
        rule = gan_train.LrRule(2e-4, periods=(10, 20, 30, 40), restart_weights=(1, 0.5, 0.5, 0.25), eta_mins=(1e-7,) * 4)
    else:
        rule = restore_train.parse_options(DERAIN[name]).lr
    its, want = g[f"{name}/it"], g[f"{name}/lr"]
    got = np.array([rule.at(int(it)) for it in its])
    assert len(its) >= 100
    np.testing.assert_array_equal(got, want)


def test_mamber32_schedule_ends_before_its_run():
    """156 000 iterations, periods summing to 144 000: the reference dies at iteration 144 002 (get_position_from_periods -> None)"""
    rule = restore_train.parse_options(DERAIN["mamber32"]).lr
    assert rule.at(144001) == pytest.approx(1e-6, rel=1e-12)
    with pytest.raises(ValueError, match="48000, 96000"):
        rule.at(144002)


def test_lr_rule_struct_carries_the_periods():
    r = restore_train.parse_options(DERAIN["mamber33"]).lr.c_rule()
    assert (r.n_periods, list(r.periods)[:3], list(r.eta_mins)[:2], r.n_milestones) == (2, [144000, 288000, 0], [0.0003, 1e-6], 0)
    assert r.base == 3e-4 and list(r.restart_weights)[:2] == [1.0, 1.0]
    plain = ops.lr_rule(1e-4, 0.5, 3, (4,), 0.1)  # n_periods 0: the step-decay / milestone rule, unchanged
    assert plain.n_periods == 0 and plain.n_milestones == 1
    with pytest.raises(ValueError):
        ops.lr_rule(1e-4, milestones=(3,), periods=(10,), restart_weights=(1,), eta_mins=(0,))
    with pytest.raises(ValueError):
        ops.lr_rule(1e-4, periods=(10, 0), restart_weights=(1, 1), eta_mins=(0, 0))


# ---------------------------------------------------------------------------------------------------------------- phases, draws
@pytest.mark.parametrize("name", ["mamber28", "mamber32"])
def test_phase_lookup_at_the_boundaries(name):
    opt = DERAIN[name]
    o = restore_train.parse_options(opt)
    its = [1, 2] + [e + d for e in o.ends for d in (-1, 0, 1)] + [opt["train"]["total_iter"], 10 ** 6]
    for it in its:
        assert restore_train.phase_at(o, it) == restore_ref.phase(opt, it), it


def _apply(p, lq, gt, scale):
    """the plan as torch indexing and the mix expression"""
    if p.idx is not None:
        lq, gt = lq[p.idx], gt[p.idx]
    if p.size is not None:
        lq = lq[:, :, p.row0:p.row0 + p.size, p.col0:p.col0 + p.size]
        gt = gt[:, :, scale * p.row0:scale * (p.row0 + p.size), scale * p.col0:scale * (p.col0 + p.size)]
    if p.lam is not None:
        r = torch.tensor(p.perm)
        lq, gt = p.lam * lq + (1 - p.lam) * lq[r], p.lam * gt + (1 - p.lam) * gt[r]
    return lq, gt


def _small(mixup, identity, scale=1):
    """a Deraining recipe shrunk to images of 24 px: six phases of 3 iterations"""
    opt = copy.deepcopy(DERAIN["mamber28"])
    opt["scale"] = scale
    opt["datasets"]["train"].update(iters=[3] * 6, gt_size=24, gt_sizes=[8, 10, 12, 16, 20, 24])
    opt["train"]["mixing_augs"] = {"mixup": mixup, "mixup_beta": 1.2, "use_identity": identity}
    return opt


@pytest.mark.parametrize("mixup,identity,scale", [(False, True, 1), (True, True, 1), (True, False, 1), (True, True, 2)])
def test_draws_follow_the_reference_loop(mixup, identity, scale):
    """from the same seeds, the plan applied with torch equals the reference loop's batch at every iteration of all six phases,
    and both leave Python's and torch's random streams in the same state"""
    opt = _small(mixup, identity, scale)
    o = restore_train.parse_options(opt)
    g = torch.Generator().manual_seed(4)
    lq = torch.rand(8, 3, 24, 24, generator=g)
    gt = torch.rand(8, 3, 24 * scale, 24 * scale, generator=g)
    mix = restore_ref.Mixup(1.2, identity) if mixup else None
    mixed = 0
    for it in range(1, 21):
        random.seed(100 + it)
        torch.manual_seed(200 + it)
        want_lq, want_gt, j = restore_ref.prepare(opt, it, lq, gt, mix)
        after = random.random(), float(torch.rand(()))
        random.seed(100 + it)
        torch.manual_seed(200 + it)
        p = restore_train.plan_batch(o, it, 8)
        assert (random.random(), float(torch.rand(()))) == after, it
        assert p.phase == j, it
        got_lq, got_gt = _apply(p, lq, gt, scale)
        assert torch.equal(got_lq, want_lq) and torch.equal(got_gt, want_gt), it
        mixed += p.lam is not None
    assert (mixed > 0) == mixup and (mixed < 20 or not identity)


def test_abi_mirrors_of_the_new_structs():
    a = _lib.BatchCropMixArgs(n_tensors=2, batch=3, lam=0.25, one_minus_lam=0.75, mix=1)
    assert len(a.idx) == len(a.perm) == _lib.CROP_MIX_MAX_IMAGES == 64 and len(a.t) == 2
    assert _lib.LrRule.periods.size == 8 * _lib.LR_MAX_PERIODS
    assert "vmb_batch_crop_mix" in _lib.SYMBOLS
