"""The GAN recipes' training iteration as one step on this library: `GANTrainer`.

It reproduces `optimize_parameters` of MambaRealSRGAN (RealSR/VmambaIR/models/MambaRealSRGAN_model.py:289-364, recipe
RealSR/options/mambaSR11GAN_x4.yml) and of MambaSISRGANModel (SRGAN/VmambaIR/models/MambaSISRGAN_model.py, recipe
SRGAN/options/MambaSISR15GAN_x4.yml) in the reference's order, from the recipe's option keys:

  schedule  one thread on the device advances the iteration counter and writes both learning rates (ops.lr_schedule): the
            generator's lr_sr * gamma_sr ** (iter // lr_decay_sr) for MambaRealSRGAN, else its MultiStepLR; the discriminator's
            MultiStepLR.  Both optim.FlatAdam steps read them on the device.
  G step    (when iter % net_d_iters == 0 and iter > net_d_init_iters) D frozen but in train mode, so its spectral norm's u, v advance
            on this call as on the other two; L1 (ops.mean_loss), PerceptualLoss and GANLoss on the output against l1_gt /
            percep_gt / gan_gt (gt or its USM sharpening, *_gt_usm).  The perceptual and GAN data gradients are taken separately and
            one kernel (ops.gan_out_grad) joins them with the L1 gradient into the generator's output gradient, in its dtype; then
            the generator's backward and its Adam + EMA step.
  D step    GANLoss on D(gan_gt) and D(output.detach()), each backpropagated into D's flat gradient, their logit means
            (ops.mean_loss) for the loss dict, D's Adam step.  An iteration without a G step still updates the EMA (basicsr's
            model_ema runs every iteration).

Nothing reads the host: `step` returns the loss dict as device tensors, and `capture` records the whole iteration -- forward, losses,
both backwards (with the generator's weight-gradient stream joined inside), both optimizer kernels -- as one CUDA graph, which it
trusts only after a replay matched the eager step.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

from . import _lib, ops
from .degradations import USMSharp
from .gan import GANLoss
from .optim import FlatAdam
from .perceptual import PerceptualLoss

_MODELS = ("MambaRealSRGAN", "MambaSISRGANModel")


@dataclass
class LrRule:
    """lr at iteration it = base * step_gamma ** (it // step_size) * milestone_gamma ** #{m in milestones : m <= it - 1}; the first
    factor is MambaRealSRGAN's generator decay (step_size 0: none), the second basicsr's MultiStepLR, stepped it - 1 times when
    iteration it runs (update_learning_rate steps from the second iteration on).  With `periods`, the rule is instead basicsr's
    CosineAnnealingRestartCyclicLR (Deraining/basicsr/models/lr_scheduler.py:115-235) at last_epoch it - 1, one restart weight
    and eta_min per period (equal eta_mins: CosineAnnealingRestartLR).  `at` is what the schedule kernel computes."""
    base: float
    step_gamma: float = 1.0
    step_size: int = 0
    milestones: tuple = ()
    milestone_gamma: float = 1.0
    periods: tuple = ()
    restart_weights: tuple = ()
    eta_mins: tuple = ()

    def at(self, it: int) -> float:
        if self.periods:
            return self._cosine(it - 1)
        lr = float(self.base)
        if self.step_size > 0:
            lr *= math.pow(self.step_gamma, it // self.step_size)
        passed = sum(m <= it - 1 for m in self.milestones)
        if passed:
            lr *= math.pow(self.milestone_gamma, passed)
        return lr

    def _cosine(self, e):
        start = 0
        for period, weight, eta_min in zip(self.periods, self.restart_weights, self.eta_mins):
            if e <= start + period:  # get_position_from_periods: the first cumulative period >= e
                return eta_min + weight * 0.5 * (self.base - eta_min) * (1 + math.cos(math.pi * ((e - start) / period)))
            start += period
        raise ValueError(f"iteration {e + 1}: the cosine schedule's periods {list(self.periods)} end at iteration {start + 1}, and "
                         "the reference scheduler has no learning rate after them")

    def c_rule(self):
        return ops.lr_rule(self.base, self.step_gamma, self.step_size, self.milestones, self.milestone_gamma, self.periods,
                           self.restart_weights, self.eta_mins)


@dataclass
class GANOptions:
    model_type: str
    l1_gt_usm: bool
    percep_gt_usm: bool
    gan_gt_usm: bool
    ema_decay: float
    optim_g: dict
    optim_d: dict
    lr_g: LrRule
    lr_d: LrRule
    pixel_weight: float                 # 0: no pixel loss (no pixel_opt)
    perceptual_opt: dict | None         # PerceptualLoss kwargs, None: no perceptual loss
    gan_opt: dict = field(default_factory=dict)
    net_d_iters: int = 1
    net_d_init_iters: int = 0


def _adam(o, who):
    if o.get("type") != "Adam":
        raise NotImplementedError(f"{who}: type {o.get('type')!r}; only Adam is implemented")
    return {"lr": float(o["lr"]), "betas": tuple(float(b) for b in o.get("betas", (0.9, 0.999))), "eps": float(o.get("eps", 1e-8)),
            "weight_decay": float(o.get("weight_decay", 0.0))}


def _milestones(train):
    s = train.get("scheduler")
    if s is None:
        return (), 1.0
    if s.get("type") not in ("MultiStepLR", "MultiStepRestartLR") or s.get("restarts", [0]) != [0]:
        raise NotImplementedError(f"scheduler {s.get('type')!r} with restarts {s.get('restarts')}: only MultiStepLR is implemented")
    ms = tuple(int(m) for m in s.get("milestones", ()))
    if len(ms) > _lib.LR_MAX_MILESTONES:
        raise ValueError(f"scheduler: {len(ms)} milestones, at most {_lib.LR_MAX_MILESTONES}")
    return ms, float(s.get("gamma", 0.1))


def parse_options(opt) -> GANOptions:
    """the recipe's options (the parsed YAML: model_type, *_gt_usm, train) -> GANOptions.  Raises NotImplementedError for what the
    step does not implement (optimizers other than Adam, warm-up, losses other than the recipes')."""
    model = opt.get("model_type")
    if model not in _MODELS:
        raise NotImplementedError(f"model_type {model!r}: GANTrainer reproduces {', '.join(_MODELS)}")
    train = opt["train"]
    if train.get("warmup_iter", -1) > 0:
        raise NotImplementedError("warmup_iter > 0 is not implemented")
    og, od = _adam(train["optim_g"], "optim_g"), _adam(train["optim_d"], "optim_d")
    ms, gamma = _milestones(train)
    if model == "MambaRealSRGAN":  # optimize_parameters overwrites the generator's lr every iteration
        lr_g = LrRule(float(train["lr_sr"]), float(train["gamma_sr"]), int(train["lr_decay_sr"]))
    else:
        lr_g = LrRule(og["lr"], milestones=ms, milestone_gamma=gamma)
    lr_d = LrRule(od["lr"], milestones=ms, milestone_gamma=gamma)
    pix = train.get("pixel_opt")
    if pix is not None and (pix.get("type") != "L1Loss" or pix.get("reduction", "mean") != "mean"):
        raise NotImplementedError(f"pixel_opt {pix}: only L1Loss with reduction 'mean' is implemented")
    percep = train.get("perceptual_opt")
    if percep is not None:
        if percep.get("type") != "PerceptualLoss":
            raise NotImplementedError(f"perceptual_opt type {percep.get('type')!r}")
        percep = {k: v for k, v in percep.items() if k != "type"}
    gan_opt = train.get("gan_opt")
    if gan_opt is None or gan_opt.get("type") != "GANLoss":
        raise NotImplementedError("gan_opt must be a GANLoss")
    usm = model == "MambaRealSRGAN"  # MambaSISRGANModel compares with gt throughout
    return GANOptions(model_type=model, l1_gt_usm=usm and opt.get("l1_gt_usm", True) is not False,
                      percep_gt_usm=usm and opt.get("percep_gt_usm", True) is not False,
                      gan_gt_usm=usm and opt.get("gan_gt_usm", True) is not False, ema_decay=float(train.get("ema_decay", 0.0)),
                      optim_g=og, optim_d=od, lr_g=lr_g, lr_d=lr_d,
                      pixel_weight=float(pix.get("loss_weight", 1.0)) if pix is not None else 0.0, perceptual_opt=percep,
                      gan_opt={k: v for k, v in gan_opt.items() if k != "type"}, net_d_iters=int(train.get("net_d_iters", 1)),
                      net_d_init_iters=int(train.get("net_d_init_iters", 0)))


class GANTrainer:
    """One iteration of the GAN recipes' second stage on this library.

    Args:
        net_g: the generator (e.g. archs.MambaRealSR11), fp32 CUDA parameters, in train mode.
        net_d: gan.UNetDiscriminatorSN, fp32 CUDA parameters.
        opt: the recipe's options (model_type, l1_gt_usm / percep_gt_usm / gan_gt_usm, train); see parse_options.
        scale: the SR scale (gt is scale x lq).
        perceptual: a PerceptualLoss to use instead of building one from train.perceptual_opt (whose VGG weights are looked up as
            PerceptualLoss(weights='auto') does).
        dtype: torch.float32, or torch.bfloat16 to run generator, discriminator and VGG under bf16 autocast.
        start_iter: the iteration before the first step (a resumed run's current_iter).

    The parameters move into optim.FlatAdam's flat buffers (one optimizer per network; the generator's carries the EMA, see
    ema_state_dict).  step(lq, gt) runs one iteration; its loss dict holds l_g_pix, l_g_percep, l_g_gan (iterations with a G step),
    l_d_real, out_d_real, l_d_fake, out_d_fake as 0-dim fp32 device tensors.  After capture(), step copies the batch into the
    graph's inputs and replays it; the returned tensors are then the graph's, overwritten by the next replay."""

    def __init__(self, net_g, net_d, opt, scale, perceptual=None, dtype=torch.float32, start_iter=0):
        if dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"GANTrainer runs in float32 or bfloat16, not {dtype}")
        self.o = o = parse_options(opt)
        self.net_g, self.net_d, self.scale, self.dtype = net_g, net_d, int(scale), dtype
        dev = next(net_g.parameters()).device
        self.opt_g = FlatAdam(net_g.parameters(), lr=o.optim_g["lr"], betas=o.optim_g["betas"], eps=o.optim_g["eps"],
                              weight_decay=o.optim_g["weight_decay"], ema_decay=o.ema_decay)
        self.opt_d = FlatAdam(net_d.parameters(), lr=o.optim_d["lr"], betas=o.optim_d["betas"], eps=o.optim_d["eps"],
                              weight_decay=o.optim_d["weight_decay"])
        self.cri_gan = GANLoss(**o.gan_opt)
        if perceptual is None and o.perceptual_opt is not None:
            perceptual = PerceptualLoss(**o.perceptual_opt).to(dev)
        self.cri_perceptual = perceptual
        self.usm = USMSharp().to(dev) if (o.l1_gt_usm or o.percep_gt_usm or o.gan_gt_usm) else None
        self.iter = int(start_iter)                                               # host copy: decides the G gate
        self.iter_dev = torch.full((1,), int(start_iter), dtype=torch.int64, device=dev)
        self.lr = torch.zeros(2, dtype=torch.float32, device=dev)                 # [generator, discriminator]
        self._one = torch.ones((), dtype=torch.float32, device=dev)
        self._rules = [o.lr_g.c_rule(), o.lr_d.c_rule()]
        self.graph = None

    def g_step_at(self, it):
        """does iteration `it` update the generator (optimize_parameters' net_d_iters / net_d_init_iters gate)?"""
        return it % self.o.net_d_iters == 0 and it > self.o.net_d_init_iters

    def _autocast(self):
        return torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.dtype == torch.bfloat16)

    def _set_d_grad(self, on):
        for p in self.net_d.parameters():
            p.requires_grad_(on)

    def _iteration(self, lq, gt, g_on):
        o, losses = self.o, {}
        ops.lr_schedule(self.iter_dev, self.lr, self._rules)
        gt_usm = self.usm(gt) if self.usm is not None else None
        l1_gt, percep_gt, gan_gt = (gt_usm if f else gt for f in (o.l1_gt_usm, o.percep_gt_usm, o.gan_gt_usm))
        # ---- generator
        self._set_d_grad(False)
        with self._autocast():
            out = self.net_g(lq)
        fake = out.detach().float().contiguous()
        if g_on:
            x = fake.detach().requires_grad_()
            g_percep = g_gan = None
            if o.pixel_weight:
                losses["l_g_pix"] = ops.mean_loss(fake, l1_gt, o.pixel_weight)
            with self._autocast():
                l_percep = self.cri_perceptual(x, percep_gt)[0] if self.cri_perceptual is not None else None
                l_g_gan = self.cri_gan(self.net_d(x), True, is_disc=False)
            if l_percep is not None:
                losses["l_g_percep"] = l_percep.detach()
                g_percep, = torch.autograd.grad(l_percep, x, self._one)
            losses["l_g_gan"] = l_g_gan.detach()
            g_gan, = torch.autograd.grad(l_g_gan, x, self._one)
            g_percep = g_percep.contiguous() if g_percep is not None else None  # autograd does not promise a layout
            out.backward(ops.gan_out_grad(fake, l1_gt, g_percep, g_gan.contiguous(), o.pixel_weight, out.dtype))
            self.opt_g.step(lr_device=self.lr[0:1])
        # ---- discriminator
        self._set_d_grad(True)
        for name, inp, real in (("real", gan_gt, True), ("fake", fake, False)):
            with self._autocast():
                pred = self.net_d(inp)
                l_d = self.cri_gan(pred, real, is_disc=True)
            losses[f"l_d_{name}"] = l_d.detach()
            losses[f"out_d_{name}"] = ops.mean_loss(pred.detach().contiguous())
            l_d.backward()
        self.opt_d.step(lr_device=self.lr[1:2])
        if not g_on and o.ema_decay > 0:
            ops.ema_update(self.opt_g.ema, self.opt_g.flat_param, o.ema_decay)
        return losses

    def _check(self, lq, gt):
        if lq.dim() != 4 or gt.dim() != 4 or lq.shape[:2] != gt.shape[:2] or \
                (gt.shape[2], gt.shape[3]) != (self.scale * lq.shape[2], self.scale * lq.shape[3]):
            raise ValueError(f"GANTrainer: gt {tuple(gt.shape)} must be {self.scale} x lq {tuple(lq.shape)}")

    def step(self, lq, gt):
        """one iteration on the batch (lq, gt), any strides (e.g. RealESRNetDegradation's cropped gt) -> loss dict of 0-dim fp32
        device tensors"""
        self._check(lq, gt)
        lq, gt = lq.contiguous(), gt.contiguous()
        self.iter += 1
        g_on = self.g_step_at(self.iter)
        if self.graph is not None and g_on and lq.shape == self._lq.shape and gt.shape == self._gt.shape:
            self._lq.copy_(lq, non_blocking=True)
            self._gt.copy_(gt, non_blocking=True)
            self.graph.replay()
            for o in (self.opt_g, self.opt_d):  # the replayed Adam kernels run no Python: announce their writes to the inference caches
                o.mark_written()
            return self._losses
        return self._iteration(lq, gt, g_on)

    # ---- CUDA graph
    def _state(self):
        bufs = [getattr(self.opt_g, k) for k in ("flat_param", "exp_avg", "exp_avg_sq", "ema", "state") if getattr(self.opt_g, k) is not None]
        bufs += [getattr(self.opt_d, k) for k in ("flat_param", "exp_avg", "exp_avg_sq", "state")]
        bufs += [b for n, b in self.net_d.named_buffers() if n.endswith(("weight_u", "weight_v"))]
        return bufs + [self.iter_dev, self.lr]

    def _snapshot(self):
        return [t.clone() for t in self._state()], self.iter

    def _restore(self, snap):
        with torch.no_grad():
            for t, s in zip(self._state(), snap[0]):
                t.copy_(s)
        for o in (self.opt_g, self.opt_d):
            o.mark_written()
        self.iter = snap[1]

    def capture(self, lq, gt):
        """record one iteration with a G step on batches of lq's and gt's shapes as one CUDA graph; step() replays it for iterations
        with a G step on those shapes.  It takes a batch rather than only its shape because the graph is checked on it: the replay
        must match an eager step on the same state (loss dict within 1e-3, each network's gradient within 2e-2 in relative norm) or
        RuntimeError is raised.  The trainer's state is left as it was."""
        self._check(lq, gt)
        dev = lq.device
        self._lq, self._gt = (t.clone(memory_format=torch.contiguous_format) for t in (lq, gt))
        snap = self._snapshot()
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):  # warm-up outside the capture: cuDNN plans, library launch state
            self._iteration(self._lq, self._gt, True)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self._restore(snap)
        for o in (self.opt_g, self.opt_d):
            o.check_views()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._losses = self._iteration(self._lq, self._gt, True)
        # the replayed iteration must reproduce the eager one before it is trusted.  The gradients are compared through Adam's first
        # moment, which is linear in them (the parameter update of an early Adam step is about lr * sign(grad), so it flips wherever
        # a gradient is near zero and the fused backward's atomics reorder a sum)
        opts = {"G": self.opt_g, "D": self.opt_d}
        m0 = {k: o.exp_avg.clone() for k, o in opts.items()}
        eager = {k: v.clone() for k, v in self._iteration(self._lq, self._gt, True).items()}
        m_e = {k: o.exp_avg.clone() for k, o in opts.items()}
        self._restore(snap)
        graph.replay()
        torch.cuda.synchronize(dev)
        bad = [f"{k}: {float(self._losses[k])} vs {float(v)}" for k, v in eager.items()
               if abs(float(self._losses[k]) - float(v)) > 1e-3 * abs(float(v)) + 1e-6]
        for k, o in opts.items():
            rel = float((o.exp_avg - m_e[k]).norm() / (m_e[k] - m0[k]).norm().clamp_min(1e-30))
            if rel > 2e-2:
                bad.append(f"{k} gradient differs by {rel:.3g} in relative norm")
        self._restore(snap)
        if bad:
            raise RuntimeError("GANTrainer: the CUDA graph's replay differs from the eager iteration: " + "; ".join(bad))
        self.graph = graph

    def ema_state_dict(self):
        """the generator's EMA weights under its parameter names (the reference's net_g_ema / `params_ema`)"""
        return self.opt_g.ema_state_dict(self.net_g)


__all__ = ["GANTrainer", "GANOptions", "LrRule", "parse_options"]
