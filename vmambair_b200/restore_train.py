"""The pixel-loss recipes' training iteration as one step on this library: `RestorationTrainer`.

It reproduces the first training stage of the three tasks, from the recipe's option keys:

  ImageCleanModel  Deraining (Deraining/Deraining/Options/Deraining_mamber*.yml), driven by Restormer's loop
                   (Deraining/basicsr/train.py:213-270): the progressive patch / batch schedule, mixup
                   (Deraining/basicsr/models/image_restoration_model.py:22-49, 136-173), L1, clip_grad_norm_(0.01) and AdamW,
                   CosineAnnealingRestartCyclicLR (Deraining/basicsr/models/lr_scheduler.py:115-235)
  MambaSISRModel   SISR stage 1 (SRGAN/options/MambaSISR15_x4.yml; SRGAN/VmambaIR/models/MambaSISR_model.py:120-147): L1, Adam,
                   MultiStepLR, EMA 0.999
  MambaRealSR      Real-ESRNet (RealSR/options/mambaSR11_x4.yml; RealSR/VmambaIR/models/MambaRealSR_model.py:147-160, 305-333): the
                   same, on the pairs vmambair_b200.degradations.RealESRNetDegradation synthesises

One step, in the reference's order:

  host      advance the iteration counter; look up the progressive phase (the first j with it <= the cumulative iters[j], else the
            last); random.sample the phase's mini-batch, draw the crop origin (x0 offsets rows) with random.random(), and, for mixup,
            random.randint, Beta(b, b).rsample on torch's default CPU generator and torch.randperm.  No draw reads the device.
  prepare   one kernel (ops.batch_crop_mix) gathers, crops (gt at x scale) and mixes lq and gt into the iteration's inputs.
  iterate   the schedule kernel (ops.lr_schedule: the iteration's lr on the device), forward (bf16 autocast on request), the L1 loss
            (ops.mean_loss), its gradient at the output (ops.gan_out_grad with only the pixel term), backward, and one
            optim.FlatAdam step (Adam or AdamW, the clip, the EMA) reading the device lr.

The iterate part is captured per phase as one CUDA graph (capture); a step of that phase then only prepares the graph's inputs and
replays it.  Nothing in a step reads the host.
"""
from __future__ import annotations

import random
from dataclasses import dataclass

import torch

from . import _lib, ops
from .gan_train import LrRule, _adam, _milestones
from .optim import FlatAdam

_MODELS = ("ImageCleanModel", "MambaSISRModel", "MambaRealSR")
_COSINE = ("CosineAnnealingRestartLR", "CosineAnnealingRestartCyclicLR")
_CLIP = 0.01  # image_restoration_model.py:167: clip_grad_norm_(net_g.parameters(), 0.01)


@dataclass
class RestoreOptions:
    model_type: str
    optim: dict                      # lr, betas, eps, weight_decay
    decoupled: bool                  # AdamW
    max_grad_norm: float             # 0: no clip
    lr: LrRule
    ema_decay: float
    pixel_weight: float
    scale: int
    mixup: bool = False
    mixup_beta: float = 1.2
    use_identity: bool = False
    batch_size: int = 0              # datasets.train.batch_size_per_gpu (progressive recipes only)
    gt_size: int = 0                 # datasets.train.gt_size, the largest patch
    ends: tuple = ()                 # cumulative iters: phase j runs the iterations up to ends[j]; () no progressive schedule
    mini_batch_sizes: tuple = ()
    gt_sizes: tuple = ()


@dataclass
class BatchPlan:
    """the host's draws for one iteration: the phase, the images of the batch (None: all, in order), the crop window in lq pixels
    (size None: no crop), and the mixup (lam None: none; perm indexes the subset)"""
    phase: int
    idx: list | None = None
    row0: int = 0
    col0: int = 0
    size: int | None = None
    lam: float | None = None
    perm: list | None = None


def _lr_rule(train, base):
    s = train.get("scheduler") or {}
    if s.get("type") not in _COSINE:
        ms, gamma = _milestones(train)
        return LrRule(base, milestones=ms, milestone_gamma=gamma)
    periods = tuple(int(p) for p in s["periods"])
    weights = tuple(float(w) for w in s.get("restart_weights", (1,)))
    if s["type"] == "CosineAnnealingRestartLR":
        etas = (float(s.get("eta_min", 0)),) * len(periods)
    else:
        etas = tuple(float(e) for e in s.get("eta_mins", (0,)))
    if not len(periods) == len(weights) == len(etas) or len(periods) > _lib.LR_MAX_PERIODS:
        raise ValueError(f"scheduler: periods {list(periods)}, restart_weights {list(weights)} and eta_mins {list(etas)} must have "
                         f"one length, at most {_lib.LR_MAX_PERIODS}")
    return LrRule(base, periods=periods, restart_weights=weights, eta_mins=etas)


def parse_options(opt) -> RestoreOptions:
    """the recipe's options (the parsed YAML: model_type, scale, datasets.train, train) -> RestoreOptions.  Raises
    NotImplementedError for what the step does not implement (optimizers other than Adam / AdamW, schedulers other than MultiStepLR
    without restarts and the two cosine ones, warm-up, losses other than L1 with mean reduction), ValueError for inconsistent keys."""
    model = opt.get("model_type")
    if model not in _MODELS:
        raise NotImplementedError(f"model_type {model!r}: RestorationTrainer reproduces {', '.join(_MODELS)}")
    train = opt["train"]
    if train.get("warmup_iter", -1) > 0:
        raise NotImplementedError("warmup_iter > 0 is not implemented")
    if train.get("perceptual_opt") is not None:
        raise NotImplementedError("perceptual_opt: the first stage takes the pixel loss only")
    og = train["optim_g"]
    kind = og.get("type")
    if kind not in ("Adam", "AdamW"):
        raise NotImplementedError(f"optim_g: type {kind!r}; only Adam and AdamW are implemented")
    # torch.optim.AdamW's weight_decay defaults to 1e-2, Adam's to 0
    optim = _adam(dict(og, type="Adam", weight_decay=og.get("weight_decay", 1e-2 if kind == "AdamW" else 0.0)), "optim_g")
    pix = train.get("pixel_opt")
    if pix is None or pix.get("type") != "L1Loss" or pix.get("reduction", "mean") != "mean":
        raise NotImplementedError(f"pixel_opt {pix}: only L1Loss with reduction 'mean' is implemented")
    clean = model == "ImageCleanModel"  # the SR models ignore use_grad_clip and mixing_augs
    mix = (train.get("mixing_augs") or {}) if clean else {}
    o = RestoreOptions(model_type=model, optim=optim, decoupled=kind == "AdamW",
                       max_grad_norm=_CLIP if clean and train.get("use_grad_clip", False) else 0.0,
                       lr=_lr_rule(train, optim["lr"]), ema_decay=float(train.get("ema_decay", 0.0)),
                       pixel_weight=float(pix.get("loss_weight", 1.0)), scale=int(opt.get("scale", 1)),
                       mixup=bool(mix.get("mixup", False)), mixup_beta=float(mix.get("mixup_beta", 1.2)),
                       use_identity=bool(mix.get("use_identity", False)))
    d = (opt.get("datasets") or {}).get("train") or {}
    if d.get("iters") is not None:
        iters, mbs, gts = (tuple(int(v) for v in d[k]) for k in ("iters", "mini_batch_sizes", "gt_sizes"))
        if not len(iters) == len(mbs) == len(gts) >= 1:
            raise ValueError(f"datasets.train: iters {list(iters)}, mini_batch_sizes {list(mbs)} and gt_sizes {list(gts)} differ in length")
        o.batch_size, o.gt_size = int(d["batch_size_per_gpu"]), int(d["gt_size"])
        if min(mbs) < 1 or max(min(mb, o.batch_size) for mb in mbs) > _lib.CROP_MIX_MAX_IMAGES:
            raise ValueError(f"datasets.train: batches {list(mbs)} of {o.batch_size}: at most {_lib.CROP_MIX_MAX_IMAGES} images per step")
        o.ends = tuple(sum(iters[:j + 1]) for j in range(len(iters)))
        o.mini_batch_sizes, o.gt_sizes = mbs, gts
    return o


def phase_at(o: RestoreOptions, it: int) -> int:
    """the progressive phase iteration `it` runs in (train.py: the first j with it <= ends[j], else the last; 0 without phases)"""
    for j, end in enumerate(o.ends):
        if it <= end:
            return j
    return max(len(o.ends) - 1, 0)


def plan_batch(o: RestoreOptions, it: int, batch: int) -> BatchPlan:
    """the host's draws for iteration `it` on a batch of `batch` images, in the reference's order (train.py:245-262, then
    Mixing_Augment.__call__ / mixup): Python's random for the subset, the crop origin and the identity choice; torch's default CPU
    generator for lam and the permutation"""
    p = BatchPlan(phase_at(o, it))
    k = batch
    if o.ends:
        mb, mg = o.mini_batch_sizes[p.phase], o.gt_sizes[p.phase]
        if mb < o.batch_size:
            p.idx = random.sample(range(0, o.batch_size), k=mb)
            k = mb
        if mg < o.gt_size:
            p.row0 = int((o.gt_size - mg) * random.random())
            p.col0 = int((o.gt_size - mg) * random.random())
            p.size = mg
    if o.mixup:
        # one augment (mixup); with use_identity, randint(0, 1) == 1 picks the identity
        if random.randint(0, 1 if o.use_identity else 0) < 1:
            beta = torch.distributions.Beta(torch.tensor([o.mixup_beta]), torch.tensor([o.mixup_beta]))
            p.lam = beta.rsample((1, 1)).item()
            p.perm = torch.randperm(k).tolist()
    return p


class RestorationTrainer:
    """One iteration of the pixel-loss recipes' first stage on this library.

    Args:
        net_g: the network (archs.Mamber32 for Deraining, archs.MambaSISR6, archs.MambaRealSR11), fp32 CUDA parameters, train mode.
        opt: the recipe's options (model_type, scale, datasets.train, train); see parse_options.
        dtype: torch.float32, or torch.bfloat16 to run the network under bf16 autocast.
        start_iter: the iteration before the first step (a resumed run's current_iter): phase and schedule follow from it.

    The parameters move into optim.FlatAdam's flat buffers.  step(lq, gt) takes the loader's batch (float32 CUDA tensors, any
    strides, gt = scale x lq) and returns {'l_pix': 0-dim fp32 device tensor}.  After capture(), steps of the captured phase replay
    its CUDA graph; the returned tensor is then the graph's, overwritten by the next replay."""

    def __init__(self, net_g, opt, dtype=torch.float32, start_iter=0):
        if dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"RestorationTrainer runs in float32 or bfloat16, not {dtype}")
        self.o = o = parse_options(opt)
        self.net_g, self.dtype = net_g, dtype
        dev = next(net_g.parameters()).device
        self.opt_g = FlatAdam(net_g.parameters(), lr=o.optim["lr"], betas=o.optim["betas"], eps=o.optim["eps"],
                              weight_decay=o.optim["weight_decay"], decoupled=o.decoupled, ema_decay=o.ema_decay,
                              max_grad_norm=o.max_grad_norm)
        self.iter = int(start_iter)                                               # host copy: decides phase and draws
        self.iter_dev = torch.full((1,), int(start_iter), dtype=torch.int64, device=dev)
        self.lr = torch.zeros(1, dtype=torch.float32, device=dev)
        self._rules = [o.lr.c_rule()]
        self.graph = self._graph_key = None

    def phase_at(self, it):
        """the progressive phase of iteration `it`: a loop recaptures when the next iteration's phase differs from the captured one"""
        return phase_at(self.o, it)

    def _autocast(self):
        return torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.dtype == torch.bfloat16)

    def _iteration(self, lq, gt):
        w = self.o.pixel_weight
        ops.lr_schedule(self.iter_dev, self.lr, self._rules)
        with self._autocast():
            out = self.net_g(lq)
        fake = out.detach().float().contiguous()
        l_pix = ops.mean_loss(fake, gt, w)
        out.backward(ops.gan_out_grad(fake, gt, None, None, w, out.dtype))
        self.opt_g.step(lr_device=self.lr)
        return {"l_pix": l_pix}

    def _check(self, lq, gt):
        s = self.o.scale
        if lq.dim() != 4 or gt.dim() != 4 or lq.shape[0] != gt.shape[0] or (gt.shape[2], gt.shape[3]) != (s * lq.shape[2], s * lq.shape[3]):
            raise ValueError(f"RestorationTrainer: gt {tuple(gt.shape)} must be {s} x lq {tuple(lq.shape)}")
        if self.o.ends and lq.shape[0] != self.o.batch_size:
            raise ValueError(f"RestorationTrainer: batch of {lq.shape[0]} images, the recipe's batch_size_per_gpu is {self.o.batch_size}")

    def _key(self, phase, k, size, lq, gt):
        return phase, k, size, lq.shape[1], gt.shape[1], tuple(lq.shape[2:])

    def step(self, lq, gt):
        """one iteration on the loader's batch (lq, gt) -> {'l_pix': 0-dim fp32 device tensor}.  Raises ValueError, before anything
        runs, at an iteration past the cosine schedule's periods (the reference scheduler has no lr there)."""
        it = self.iter + 1
        self.o.lr.at(it)
        self._check(lq, gt)
        p = plan_batch(self.o, it, lq.shape[0])
        self.iter = it
        idx = p.idx if p.idx is not None else range(lq.shape[0])
        replay = self.graph is not None and self._graph_key == self._key(p.phase, len(idx), p.size, lq, gt)
        inp = ops.batch_crop_mix(lq, gt, idx, p.row0, p.col0, p.size, self.o.scale, p.lam, p.perm,
                                 out=(self._lq, self._gt) if replay else None)
        if replay:
            self.graph.replay()
            self.opt_g.mark_written()  # the replayed Adam kernel runs no Python: announce its write to the inference caches
            return self._losses
        return self._iteration(*inp)

    # ---- CUDA graph
    def _state(self):
        o = self.opt_g
        return [t for t in (o.flat_param, o.exp_avg, o.exp_avg_sq, o.ema, o.state, self.iter_dev, self.lr) if t is not None]

    def _restore(self, snap):
        with torch.no_grad():
            for t, s in zip(self._state(), snap):
                t.copy_(s)
        self.opt_g.mark_written()

    def capture(self, lq, gt):
        """record the iteration of the next step's phase, on batches of that phase's shapes, as one CUDA graph (releasing the graph
        of an earlier phase); later steps of the phase replay it.  The graph's inputs are prepared from (lq, gt) with the first
        images and the crop at the origin, so that no host random stream is drawn from.  The replay must match an eager iteration
        on the same state (loss within 1e-3, the gradient within 2e-2 in relative norm, through Adam's first moment) or
        RuntimeError is raised.  The trainer's state is left as it was."""
        self._check(lq, gt)
        self.graph = self._graph_key = self._lq = self._gt = self._losses = None
        o, dev = self.o, lq.device
        phase = self.phase_at(self.iter + 1)
        k = o.mini_batch_sizes[phase] if o.ends and o.mini_batch_sizes[phase] < o.batch_size else lq.shape[0]
        size = o.gt_sizes[phase] if o.ends and o.gt_sizes[phase] < o.gt_size else None
        self._lq, self._gt = ops.batch_crop_mix(lq, gt, range(k), 0, 0, size, o.scale)
        snap = [t.clone() for t in self._state()]
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):  # warm-up outside the capture: cuDNN plans, library launch state
            self._iteration(self._lq, self._gt)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self._restore(snap)
        self.opt_g.check_views()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            losses = self._iteration(self._lq, self._gt)
        m0 = self.opt_g.exp_avg.clone()
        eager = float(self._iteration(self._lq, self._gt)["l_pix"])
        m_e = self.opt_g.exp_avg.clone()
        self._restore(snap)
        graph.replay()
        torch.cuda.synchronize(dev)
        bad = []
        if abs(float(losses["l_pix"]) - eager) > 1e-3 * abs(eager) + 1e-6:
            bad.append(f"l_pix: {float(losses['l_pix'])} vs {eager}")
        rel = float((self.opt_g.exp_avg - m_e).norm() / (m_e - m0).norm().clamp_min(1e-30))
        if rel > 2e-2:
            bad.append(f"gradient differs by {rel:.3g} in relative norm")
        self._restore(snap)
        if bad:
            raise RuntimeError("RestorationTrainer: the CUDA graph's replay differs from the eager iteration: " + "; ".join(bad))
        self.graph, self._losses = graph, losses
        self._graph_key = self._key(phase, k, size, lq, gt)

    def ema_state_dict(self):
        """the EMA weights under the network's parameter names (the reference's net_g_ema / `params_ema`); recipes with ema_decay"""
        if self.opt_g.ema is None:
            raise ValueError("RestorationTrainer: the recipe keeps no EMA (ema_decay 0)")
        return self.opt_g.ema_state_dict(self.net_g)


__all__ = ["RestorationTrainer", "RestoreOptions", "BatchPlan", "parse_options", "phase_at", "plan_batch"]
