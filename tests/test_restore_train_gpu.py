"""RestorationTrainer and its kernels on the GPU: the cosine schedule kernel against LrRule at every iteration of the four Deraining
schedules, the input-preparation kernel (ops.batch_crop_mix) bitwise against the torch expression, whole iterations of the three
first-stage recipes against the reference composed from torch modules, CUDA-graph replays against eager steps across a phase change,
a step without host synchronisation, the deraining network's gradients against the float64 module oracle, and the recipe's full
Mamber32 at its first and last phase."""
import copy
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cscan, oss_ref, restore_ref
from tests import test_train_net_gpu as net_yardstick
from tests.test_restore_train_cpu import DERAIN
from vmambair_b200 import archs, gan_train, ops, restore_train
from vmambair_b200.degradations import RealESRNetDegradation

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------- schedule
def _device_lrs(rules, n, chunk=1000):
    """lr of up to two rules at iterations 1..n from the schedule kernel: a graph of `chunk` launches, each followed by a copy of
    the lr into its row, replayed n / chunk times"""
    it = torch.zeros(1, dtype=torch.int64, device=DEV)
    lr = torch.zeros(2, dtype=torch.float32, device=DEV)
    rows = torch.empty(chunk, 2, dtype=torch.float32, device=DEV)
    c_rules = [r.c_rule() for r in rules]
    ops.lr_schedule(it, lr, c_rules)  # warm-up launch, then back to iteration 0
    it.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for k in range(chunk):
            ops.lr_schedule(it, lr, c_rules)
            rows[k].copy_(lr)
    out = []
    for _ in range((n + chunk - 1) // chunk):
        graph.replay()
        out.append(rows.clone())
    return torch.cat(out)[:n, :len(rules)].cpu().numpy()


def test_cosine_schedule_kernel_at_every_iteration():
    rules = {k: restore_train.parse_options(o).lr for k, o in DERAIN.items()}
    ends = {k: sum(r.periods) + 1 for k, r in rules.items()}  # the last iteration with an lr
    for pair in (("mamber28", "mamber32"), ("mamber33", "mamber34")):
        n = max(ends[k] for k in pair) + 3
        got = _device_lrs([rules[k] for k in pair], n)
        for col, k in enumerate(pair):
            want = np.array([rules[k].at(it) for it in range(1, ends[k] + 1)], dtype=np.float32)
            bad = np.flatnonzero(got[:ends[k], col] != want)
            assert bad.size == 0, (k, bad[:5] + 1, got[bad[:5], col], want[bad[:5]])
            assert np.isnan(got[ends[k]:, col]).all(), k  # past the periods: no lr


def test_step_and_milestone_rules_unchanged():
    rules = [gan_train.LrRule(1e-4, 0.5, 3), gan_train.LrRule(2e-4, milestones=(2, 5), milestone_gamma=0.1)]
    got = _device_lrs(rules, 20, chunk=10)
    want = np.array([[r.at(it) for r in rules] for it in range(1, 21)], dtype=np.float32)
    np.testing.assert_array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------- preparation
def _torch_prep(lq, gt, idx, row0, col0, size, scale, lam, perm):
    lq, gt = lq[idx], gt[idx]
    if size is not None:
        lq = lq[:, :, row0:row0 + size, col0:col0 + size]
        gt = gt[:, :, scale * row0:scale * (row0 + size), scale * col0:scale * (col0 + size)]
    if lam is not None:
        r = torch.tensor(perm, device=DEV)
        lq, gt = lam * lq + (1 - lam) * lq[r, :], lam * gt + (1 - lam) * gt[r, :]
    return lq, gt


def _sources(b, h, scale, layout, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if layout == "dense":
        return torch.rand(b, 3, h, h, device=DEV, generator=g), torch.rand(b, 3, scale * h, scale * h, device=DEV, generator=g)
    if layout == "cropped":  # RealESRNetDegradation's gt: a window of a larger batch
        big = torch.rand(b, 3, h + 5, h + 9, device=DEV, generator=g)
        bigt = torch.rand(b, 3, scale * h + 7, scale * h + 3, device=DEV, generator=g)
        return big[:, :, 2:2 + h, 7:7 + h], bigt[:, :, 5:5 + scale * h, 1:1 + scale * h]
    # channels-last storage, and the batch itself strided
    lq = torch.rand(2 * b, 3, h, h, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)[::2]
    gt = torch.rand(2 * b, 3, scale * h, scale * h, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)[::2]
    return lq, gt


@pytest.mark.parametrize("layout", ["dense", "cropped", "channels_last"])
@pytest.mark.parametrize("scale", [1, 4])
@pytest.mark.parametrize("b,k", [(1, 1), (5, 3), (8, 8)])
def test_batch_crop_mix_is_the_torch_expression(layout, scale, b, k):
    lq, gt = _sources(b, 23, scale, layout, seed=b * 10 + k + scale)
    rng = random.Random(b * k + scale)
    torch.manual_seed(b + k)
    beta = torch.distributions.Beta(torch.tensor([1.2]), torch.tensor([1.2]))
    for size, row0, col0 in ((None, 0, 0), (11, 3, 7), (17, 5, 1)):
        idx = rng.sample(range(b), k=k)
        for lam, perm in ((None, None), (beta.rsample((1, 1)).item(), torch.randperm(k).tolist())):
            got = ops.batch_crop_mix(lq, gt, idx, row0, col0, size, scale, lam, perm)
            want = _torch_prep(lq, gt, idx, row0, col0, size, scale, lam, perm)
            for g_, w_ in zip(got, want):
                assert g_.is_contiguous() and g_.shape == w_.shape
                assert torch.equal(g_, w_), (size, lam, float((g_ - w_).abs().max()))
    # repeated images and a pure gather into given buffers
    out = tuple(torch.full(t.shape, float("nan"), device=DEV) for t in _torch_prep(lq, gt, [0] * k, 1, 2, 9, scale, None, None))
    ops.batch_crop_mix(lq, gt, [0] * k, 1, 2, 9, scale, out=out)
    assert all(torch.equal(o, w) for o, w in zip(out, _torch_prep(lq, gt, [0] * k, 1, 2, 9, scale, None, None)))


def test_batch_crop_mix_rejects_bad_arguments():
    lq, gt = _sources(4, 16, 2, "dense", 0)
    bad = [
        dict(idx=[4]),                          # image out of range
        dict(idx=list(range(4)) * 17),          # 68 images > 64
        dict(row0=9, size=8),                   # window leaves lq
        dict(perm=[0, 0], lam=0.5, idx=[1, 2]),  # not a permutation
        dict(scale=5),                          # gt window leaves gt
    ]
    for b in bad:
        kw = dict(idx=[0, 1], row0=0, col0=0, size=8, scale=2, lam=None, perm=None)
        kw.update(b)
        with pytest.raises(ValueError):
            ops.batch_crop_mix(lq, gt, **kw)
    with pytest.raises(ValueError):
        ops.batch_crop_mix(lq.half(), gt.half(), [0], 0, 0, 8, 2)
    with pytest.raises(ValueError):
        ops.batch_crop_mix(lq, gt, [0], 0, 0, 8, 2, out=(torch.empty(1, 3, 8, 8, device=DEV), torch.empty(1, 3, 8, 8, device=DEV)))


# ---------------------------------------------------------------------------------------------------------------- iterations
def _derain_small(mixup=True, clip=True, identity=True):
    """Deraining_mamber28 shrunk: batches of 4 at 24 px, phases (4 x 8, 3 x 16, 2 x 24) of 2, 2 and 3 iterations, cosine periods
    of 3 and 4 iterations: seven iterations cross two phase changes and a restart"""
    opt = copy.deepcopy(DERAIN["mamber28"])
    opt["datasets"]["train"].update(batch_size_per_gpu=4, mini_batch_sizes=[4, 3, 2], iters=[2, 2, 3], gt_size=24, gt_sizes=[8, 16, 24])
    t = opt["train"]
    t.update(total_iter=7, use_grad_clip=clip, mixing_augs={"mixup": mixup, "mixup_beta": 1.2, "use_identity": identity})
    t["scheduler"].update(periods=[3, 4], eta_mins=[1e-4, 1e-6])
    t["optim_g"].update(lr=2e-4)
    return opt


def _sr_small(model, ema=0.9):
    t = {"ema_decay": ema, "optim_g": {"type": "Adam", "lr": 2e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
         "scheduler": {"type": "MultiStepLR", "milestones": [2], "gamma": 0.5}, "warmup_iter": -1,
         "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"}}
    return {"model_type": model, "scale": 4, "train": t}


class _Reference:
    """the reference loop composed from torch modules: update_learning_rate (the restated schedule), the batch preparation of
    oracle/restore_ref, the network's compose path, F.l1_loss, backward, clip_grad_norm_(0.01), torch.optim.Adam / AdamW, EMA"""

    def __init__(self, net, opt):
        self.opt, self.o = opt, restore_train.parse_options(opt)
        self.net = copy.deepcopy(net)
        self.ema = {k: v.detach().clone() for k, v in self.net.named_parameters()}
        og = self.o.optim
        cls = torch.optim.AdamW if self.o.decoupled else torch.optim.Adam
        self.optim = cls(self.net.parameters(), lr=og["lr"], betas=og["betas"], eps=og["eps"], weight_decay=og["weight_decay"])
        self.mix = restore_ref.Mixup(self.o.mixup_beta, self.o.use_identity) if self.o.mixup else None

    def iteration(self, it, lq, gt):
        for pg in self.optim.param_groups:
            pg["lr"] = self.o.lr.at(it)
        lq, gt, _ = restore_ref.prepare(self.opt, it, lq, gt, self.mix)
        self.optim.zero_grad()
        l_pix = self.o.pixel_weight * F.l1_loss(self.net(lq), gt)
        l_pix.backward()
        if self.o.max_grad_norm:
            torch.nn.utils.clip_grad_norm_(self.net.parameters(), 0.01)
        self.optim.step()
        if self.o.ema_decay > 0:
            with torch.no_grad():
                for k, p in self.net.named_parameters():
                    self.ema[k].mul_(self.o.ema_decay).add_(p, alpha=1 - self.o.ema_decay)
        return {"l_pix": l_pix.detach()}


def _flat(ts):
    return torch.cat([t.detach().reshape(-1) for t in ts])


def _run_against_reference(net, opt, batches):
    prev = archs._TRAIN_PATH
    archs.set_train_path("compose")
    try:
        ref = _Reference(net, opt)
        tr = restore_train.RestorationTrainer(net, opt)
        random.seed(11)
        torch.manual_seed(12)
        for it, (lq, gt) in enumerate(batches, 1):
            state = random.getstate(), torch.get_rng_state()
            ours = tr.step(lq, gt)
            after = random.getstate(), torch.get_rng_state()
            random.setstate(state[0])
            torch.set_rng_state(state[1])
            want = ref.iteration(it, lq, gt)
            assert random.getstate() == after[0] and torch.equal(torch.get_rng_state(), after[1]), it
            assert abs(float(ours["l_pix"]) - float(want["l_pix"])) <= 1e-4 * abs(float(want["l_pix"])) + 1e-7, \
                (it, float(ours["l_pix"]), float(want["l_pix"]))
            assert float(tr.lr[0]) == np.float32(ref.optim.param_groups[0]["lr"]), it
            assert _rel(tr.opt_g.flat_param, _flat(ref.net.parameters())) <= 1e-4, it
            if ref.o.ema_decay > 0:
                ema = tr.ema_state_dict()
                assert _rel(_flat(ema[k] for k in ref.ema), _flat(ref.ema.values())) <= 1e-4, it
        return tr
    finally:
        archs.set_train_path(prev)


def test_deraining_iterations_against_the_composed_reference():
    torch.manual_seed(0)
    net = archs.Mamber32(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    opt = _derain_small()
    g = torch.Generator(device=DEV).manual_seed(3)
    batches = [(torch.rand(4, 3, 24, 24, device=DEV, generator=g), torch.rand(4, 3, 24, 24, device=DEV, generator=g)) for _ in range(7)]
    tr = _run_against_reference(net, opt, batches)
    o = tr.o
    assert [restore_train.phase_at(o, it) for it in range(1, 8)] == [0, 0, 1, 1, 2, 2, 2]
    assert o.lr.at(4) == pytest.approx(1e-4) and o.lr.at(5) > 1e-4 * 1.5  # a restart between iterations 4 and 5


def test_sisr_iterations_against_the_composed_reference():
    torch.manual_seed(1)
    net = archs.MambaSISR6(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    g = torch.Generator(device=DEV).manual_seed(4)
    batches = [(torch.rand(2, 3, 16, 16, device=DEV, generator=g), torch.rand(2, 3, 64, 64, device=DEV, generator=g)) for _ in range(4)]
    tr = _run_against_reference(net, _sr_small("MambaSISRModel"), batches)
    assert tr.o.lr.at(2) == 2e-4 and tr.o.lr.at(3) == 1e-4


def test_realesrnet_iterations_against_the_composed_reference():
    torch.manual_seed(2)
    net = archs.MambaRealSR11(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    deg_opt = dict(gt_usm=False, resize_prob=[0.2, 0.7, 0.1], resize_range=[0.15, 1.5], gaussian_noise_prob=0.5, noise_range=[1, 30],
                   poisson_scale_range=[0.05, 3], gray_noise_prob=0.4, jpeg_range=[30, 95], second_blur_prob=0.8,
                   resize_prob2=[0.3, 0.4, 0.3], resize_range2=[0.3, 1.2], gaussian_noise_prob2=0.5, noise_range2=[1, 25],
                   poisson_scale_range2=[0.05, 2.5], gray_noise_prob2=0.4, jpeg_range2=[30, 95], gt_size=64, queue_size=180)
    deg = RealESRNetDegradation(deg_opt, 4)
    g = torch.Generator(device=DEV).manual_seed(5)
    batches = []
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    for _ in range(3):
        gt = torch.rand(2, 3, 96, 96, device=DEV, generator=g)
        ks = [torch.rand(2, 21, 21, device=DEV, generator=g) + 0.05 for _ in range(3)]
        lq, gt_c = deg(gt, *[k / k.sum((1, 2), keepdim=True) for k in ks])
        batches.append((lq.clone(), gt_c))  # gt_c: a cropped view of the batch, as the degradation hands it over
    assert tuple(batches[0][1].shape) == (2, 3, 64, 64) and tuple(batches[0][0].shape) == (2, 3, 16, 16)
    _run_against_reference(net, _sr_small("MambaRealSR"), batches)


# ---------------------------------------------------------------------------------------------------------------- replay
def _conv_net():
    """a small network of cuDNN convolutions, bitwise reproducible (the fused OSS backward is not, DESIGN §6 item 5)"""
    torch.manual_seed(1)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 32, 3, 1, 1), torch.nn.LeakyReLU(0.2), torch.nn.Conv2d(32, 3, 3, 1, 1)).to(DEV).train()


def test_graph_replays_equal_eager_steps_across_a_phase_change():
    """seven iterations with subset, crop and mixup over three phases; the graph run captures each phase as it starts.  The clip's
    norm is summed with atomics, so it is off here to make the comparison bitwise."""
    prev = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    try:
        opt = _derain_small(clip=False)
        g = torch.Generator(device=DEV).manual_seed(9)
        batches = [(torch.rand(4, 3, 24, 24, device=DEV, generator=g), torch.rand(4, 3, 24, 24, device=DEV, generator=g)) for _ in range(7)]
        runs = {}
        for mode in ("eager", "graph"):
            tr = restore_train.RestorationTrainer(_conv_net(), opt)
            random.seed(5)
            torch.manual_seed(6)
            losses, captured = [], None
            for lq, gt in batches:
                if mode == "graph" and tr.phase_at(tr.iter + 1) != captured:
                    before = ([t.clone() for t in tr._state()], tr.iter, random.getstate(), torch.get_rng_state())
                    tr.capture(lq, gt)
                    captured = tr.phase_at(tr.iter + 1)
                    assert all(torch.equal(a, b) for a, b in zip(before[0], tr._state())) and tr.iter == before[1]
                    assert random.getstate() == before[2] and torch.equal(torch.get_rng_state(), before[3])
                losses.append(float(tr.step(lq, gt)["l_pix"]))
            runs[mode] = (losses, tr.opt_g.flat_param.clone(), tr.opt_g.exp_avg.clone(), int(tr.iter_dev), float(tr.lr[0]))
        (le, *se), (lg, *sg) = runs["eager"], runs["graph"]
        assert le == lg
        for a, b in zip(se, sg):
            assert torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b
    finally:
        torch.backends.cudnn.deterministic = prev


def test_step_without_host_synchronisation():
    torch.manual_seed(0)
    net = archs.Mamber32(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    tr = restore_train.RestorationTrainer(net, _derain_small(identity=False), start_iter=2)  # phase 1: subset 3 of 4, crop 16 of 24
    g = torch.Generator(device=DEV).manual_seed(1)
    lq, gt = torch.rand(4, 3, 24, 24, device=DEV, generator=g), torch.rand(4, 3, 24, 24, device=DEV, generator=g)
    tr.step(lq, gt)  # first call: lazy initialisation of cuDNN and the library
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = tr.step(lq, gt)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert set(losses) == {"l_pix"} and bool(torch.isfinite(losses["l_pix"]))


def test_schedule_end_raises_before_launching():
    torch.manual_seed(0)
    net = archs.Mamber32(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).to(DEV).train()
    tr = restore_train.RestorationTrainer(net, DERAIN["mamber32"], start_iter=144001)
    lq = torch.rand(8, 3, 384, 384, device=DEV)
    p0 = tr.opt_g.flat_param.clone()
    with pytest.raises(ValueError, match="48000, 96000"):
        tr.step(lq, lq)
    torch.cuda.synchronize()
    assert tr.iter == 144001 and int(tr.iter_dev) == 144001 and torch.equal(tr.opt_g.flat_param, p0)


# ---------------------------------------------------------------------------------------------------------------- the deraining net
def test_deraining_step_gradients_match_float64_oracle():
    """one step of a small Mamber32 on the fused training path (fp32): its output and every parameter gradient (read back from
    AdamW's first moment, (1 - beta1) g after the first step) against float64 autograd of oss_ref.net_forward(kind='mamber32'), fed
    the step's own L1 gradient; the yardsticks of tests/test_train_net_gpu.py"""
    cscan.use_host_threads()
    archs.set_train_path("fused")
    torch.manual_seed(3)
    net = archs.Mamber32(dim=16, num_blocks=[1, 1, 1, 1], num_refinement_blocks=1).train()
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():  # away from init, where the LayerNorm biases are 0 and the weights 1 and hide dropped terms
        for p in net.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g))
    net = net.to(DEV)
    lq = torch.rand(2, 3, 32, 32, generator=g).to(DEV)
    gt = torch.rand(2, 3, 32, 32, generator=g).to(DEV)
    ref_net = copy.deepcopy(net)
    opt = _derain_small(mixup=False, clip=False)
    opt["datasets"]["train"] = {}  # one batch as it comes: no subset, no crop
    opt["train"]["optim_g"].update(weight_decay=0.0)
    tr = restore_train.RestorationTrainer(net, opt)
    outs = []
    hook = net.register_forward_hook(lambda m, i, o: outs.append(o.detach().clone()))
    try:
        tr.step(lq, gt)
    finally:
        hook.remove()
    torch.cuda.synchronize()
    beta1 = tr.o.optim["betas"][0]
    got, o = {"out": outs[0]}, 0
    for n, p in ref_net.named_parameters():
        got[n] = (tr.opt_g.exp_avg[o:o + p.numel()] / (1 - beta1)).view_as(p)
        o += p.numel()
    dout = torch.sign(outs[0].double() - gt.double()) / gt.numel()

    def oracle(dtype):
        sd = net_yardstick._leaves(ref_net, dtype)

        def run():
            out = oss_ref.net_forward(sd, lq.to(dtype), "mamber32")
            out.backward(dout.to(dtype))
            return out.detach()

        out = net_yardstick._with_store(None, run)
        return {"out": out, **{k: p.grad for k, p in sd.items()}}

    ref64, ref32 = oracle(torch.float64), oracle(torch.float32)
    bad = net_yardstick._check("mamber32 step fp32", got, ref64, ref32, False, k32=4)
    assert not bad, "\n".join(bad)


# ---------------------------------------------------------------------------------------------------------------- full size
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("start,shape", [(0, (8, 128)), (132000, (1, 384))], ids=["first_phase", "last_phase"])
def test_full_mamber32_phases_capture_and_replay(start, shape, dtype):
    torch.manual_seed(0)
    net = archs.Mamber32(dim=48, num_blocks=[3, 5, 7, 9], num_refinement_blocks=2, ffn_expansion_factor=2.66, bias=False).to(DEV).train()
    tr = restore_train.RestorationTrainer(net, DERAIN["mamber32"], dtype=dtype, start_iter=start)
    g = torch.Generator(device=DEV).manual_seed(2)
    lq, gt = torch.rand(8, 3, 384, 384, device=DEV, generator=g), torch.rand(8, 3, 384, 384, device=DEV, generator=g)
    tr.capture(lq, gt)
    assert tuple(tr._lq.shape) == (shape[0], 3, shape[1], shape[1])
    losses = [tr.step(lq, gt)["l_pix"].clone() for _ in range(3)]
    torch.cuda.synchronize()
    assert all(bool(torch.isfinite(v)) for v in losses) and bool(torch.isfinite(tr.opt_g.flat_param).all())
    assert tr.iter == start + 3 and int(tr.iter_dev) == start + 3
