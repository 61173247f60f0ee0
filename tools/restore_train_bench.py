"""Time of one first-stage training iteration (vmambair_b200.restore_train.RestorationTrainer) against what a user writes today, in
fp32 and under bf16 autocast, at the recipes' shapes:

  Deraining  Deraining_mamber33.yml's six progressive phases (8 x 128^2, 5 x 160^2, 3 x 192^2, 2 x 256^2, 1 x 320^2, 1 x 384^2,
             cropped from batches of 8 x 384^2) on the recipe's full Mamber32 (dim 48, [3, 5, 7, 9] + 2, ffn 2.66, bias False):
             AdamW, clip_grad_norm_(0.01), CosineAnnealingRestartCyclicLR;
  SISR15     MambaSISR15_x4.yml's stage 1 (MambaSISR6 dim 48, [15, 1, 1, 1] + 15, 8 x 3 x 64^2 LQ): Adam, MultiStepLR, EMA 0.999.

  trainer    the trainer's step: the host draws, the preparation kernel and the phase's CUDA graph replayed;
  torch      the same network modules, eager, with the same batch preparation in torch (indexing, slicing, the mixup expression
             when on), F.l1_loss, torch.optim.AdamW / Adam, clip_grad_norm_, the lr set by a torch LambdaLR / MultiStepLR on the
             host, and a torch EMA where the recipe keeps one.

The two alternate in rounds of --steps iterations after --warmup; reported are the median ms per iteration and images/s over
--rounds rounds, the card and its power limit from the same run, and which OSS blocks of the deraining net leave the fused training
path (fused.unsupported_reason), as one JSON line per workload and a summary line.

    python tools/restore_train_bench.py [--steps 5] [--warmup 2] [--rounds 3] [--out results.json]
"""
import argparse
import copy
import json
import os
import random
import statistics
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import archs, fused, restore_train  # noqa: E402

DERAIN = {"model_type": "ImageCleanModel", "scale": 1,
          "datasets": {"train": {"batch_size_per_gpu": 8, "mini_batch_sizes": [8, 5, 3, 2, 1, 1], "gt_size": 384,
                                 "iters": [92000, 64000, 64000, 64000, 64000, 48000], "gt_sizes": [128, 160, 192, 256, 320, 384]}},
          "train": {"total_iter": 396000, "warmup_iter": -1, "use_grad_clip": True,
                    "scheduler": {"type": "CosineAnnealingRestartCyclicLR", "periods": [144000, 288000], "restart_weights": [1, 1],
                                  "eta_mins": [0.0003, 0.000001]},
                    "mixing_augs": {"mixup": False, "mixup_beta": 1.2, "use_identity": True},
                    "optim_g": {"type": "AdamW", "lr": 3e-4, "weight_decay": 1e-4, "betas": [0.9, 0.999]},
                    "pixel_opt": {"type": "L1Loss", "loss_weight": 1, "reduction": "mean"}}}
SISR = {"model_type": "MambaSISRModel", "scale": 4,
        "train": {"ema_decay": 0.999, "optim_g": {"type": "Adam", "lr": 2e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                  "scheduler": {"type": "MultiStepLR", "milestones": [50000, 70000], "gamma": 0.5}, "total_iter": 100000,
                  "warmup_iter": -1, "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"}}}


def derain_net():
    return archs.Mamber32(dim=48, num_blocks=[3, 5, 7, 9], num_refinement_blocks=2, ffn_expansion_factor=2.66, bias=False)


def sisr_net():
    return archs.MambaSISR6(dim=48, num_blocks=[15, 1, 1, 1], num_refinement_blocks=15)


class Torch:
    """the iteration a user writes today around the same modules"""

    def __init__(self, net, opt, dtype):
        self.net, self.opt, self.dtype = net, opt, dtype
        self.o = o = restore_train.parse_options(opt)
        cls = torch.optim.AdamW if o.decoupled else torch.optim.Adam
        self.optim = cls(net.parameters(), lr=o.optim["lr"], betas=o.optim["betas"], eps=o.optim["eps"],
                         weight_decay=o.optim["weight_decay"])
        if o.lr.periods:
            self.sched = torch.optim.lr_scheduler.LambdaLR(self.optim, lambda e: o.lr.at(e + 1) / o.lr.base)
        else:
            self.sched = torch.optim.lr_scheduler.MultiStepLR(self.optim, list(o.lr.milestones), o.lr.milestone_gamma)
        self.ema = [p.detach().clone() for p in net.parameters()] if o.ema_decay > 0 else None
        self.iter = 0

    def step(self, lq, gt):
        o = self.o
        self.iter += 1
        if self.iter > 1:
            self.sched.step()
        p = restore_train.plan_batch(o, self.iter, lq.shape[0])
        if p.idx is not None:
            lq, gt = lq[p.idx], gt[p.idx]
        if p.size is not None:
            s = o.scale
            lq = lq[:, :, p.row0:p.row0 + p.size, p.col0:p.col0 + p.size]
            gt = gt[:, :, s * p.row0:s * (p.row0 + p.size), s * p.col0:s * (p.col0 + p.size)]
        self.optim.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.dtype == torch.bfloat16):
            out = self.net(lq)
        loss = F.l1_loss(out.float(), gt)
        loss.backward()
        if o.max_grad_norm:
            torch.nn.utils.clip_grad_norm_(self.net.parameters(), o.max_grad_norm)
        self.optim.step()
        if self.ema is not None:
            with torch.no_grad():
                torch._foreach_lerp_(self.ema, [p.detach() for p in self.net.parameters()], 1 - o.ema_decay)
        return {"l_pix": loss.detach()}


def left_fused(net, lq):
    """the OSS blocks of `net` whose training call leaves the fused kernels on `lq`'s shape, with the reason"""
    out, seen = {}, {}
    names = {m: n for n, m in net.named_modules()}
    hooks = [m.register_forward_pre_hook(lambda m, a: seen.setdefault(m, a[0].detach()))
             for m in net.modules() if isinstance(m, archs.MamberBlock)]
    try:
        net(lq)  # the training call, forward only
    finally:
        for h in hooks:
            h.remove()
    for m, x in seen.items():
        r = fused.unsupported_reason(m, x)
        if r is not None:
            out[names[m]] = r
    return out


def workload(name, make_net, opt, phase_iter, lq_shape, gt_shape, images, dtype, args, dev):
    torch.manual_seed(0)
    random.seed(0)
    net = make_net().to(dev).train()
    net_t = copy.deepcopy(net)
    g = torch.Generator(device=dev).manual_seed(1)
    lq, gt = torch.rand(*lq_shape, device=dev, generator=g), torch.rand(*gt_shape, device=dev, generator=g)
    tr = restore_train.RestorationTrainer(net, opt, dtype=dtype, start_iter=phase_iter)
    ref = Torch(net_t, opt, dtype)
    ref.iter = phase_iter
    tr.capture(lq, gt)
    paths = {"trainer": lambda: tr.step(lq, gt), "torch": lambda: ref.step(lq, gt)}
    for fn in paths.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in paths}
    for _ in range(args.rounds):
        for k, fn in paths.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
            times[k].append(1e3 * (time.perf_counter() - t0) / args.steps)
    ms = {k: statistics.median(v) for k, v in times.items()}
    rec = {"workload": name, "dtype": "bf16" if dtype == torch.bfloat16 else "fp32", "images": images,
           **{f"{k}_ms": round(v, 2) for k, v in ms.items()}, **{f"{k}_img_s": round(1e3 * images / v, 1) for k, v in ms.items()},
           "speedup": round(ms["torch"] / ms["trainer"], 3), "rounds_ms": {k: [round(x, 2) for x in v] for k, v in times.items()}}
    del tr, ref, net, net_t
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "restore_train_bench needs a GPU"
    dev = torch.device("cuda", 0)
    gpu, pl = gpu_info()
    o = restore_train.parse_options(DERAIN)
    starts = [0] + list(o.ends[:-1])
    work = [(f"derain phase {j} {o.mini_batch_sizes[j]}x{o.gt_sizes[j]}^2", derain_net, DERAIN, starts[j],
             (8, 3, 384, 384), (8, 3, 384, 384), min(o.mini_batch_sizes[j], 8)) for j in range(6)]
    work.append(("sisr15 stage 1 8x64^2", sisr_net, SISR, 0, (8, 3, 64, 64), (8, 3, 256, 256), 8))
    net = derain_net().to(dev).train()
    leaving = {f"{s}^2": left_fused(net, torch.rand(b, 3, s, s, device=dev)) for b, s in ((8, 128), (1, 384))}
    del net
    recs = []
    for dtype in (torch.float32, torch.bfloat16):
        for w in work:
            rec = workload(*w, dtype, args, dev)
            rec.update(gpu=gpu, power_limit=pl)
            print(json.dumps(rec), flush=True)
            recs.append(rec)
    summary = {"gpu": gpu, "power_limit": pl, "steps": args.steps, "rounds": args.rounds, "left_fused_path": leaving}
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"records": recs, **summary}, f, indent=1)


if __name__ == "__main__":
    main()
