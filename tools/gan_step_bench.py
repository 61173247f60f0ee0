"""Time of one GAN training iteration at the RealSR recipe's shape (RealSR/options/mambaSR11GAN_x4.yml: batch 9, GT 256 = 4 x LQ 64,
MambaRealSR11 dim 48 [6, 2, 2, 1] + 6, UNetDiscriminatorSN num_feat 64, VGG19 perceptual loss on the recipe's five layers, all under
bf16 autocast) on three paths, alternated step by step in one process:

  graph     vmambair_b200.gan_train.GANTrainer, the iteration replayed from its CUDA graph;
  eager     the same trainer stepped eagerly;
  composed  the same iteration as the reference writes it (MambaRealSRGAN_model.py:289-364): the same generator (this library's
            drop-in), oracle/gan_ref's discriminator and loss, oracle/perceptual_ref's VGG loss, torch L1, autograd's accumulation of
            the three output gradients, torch.optim.Adam for both networks with the lr set on the host (the generator's step decay,
            MultiStepLR for the discriminator), and a torch EMA.

All three start from the same state.  Reported: the median ms per iteration and its range over --steps (CUDA events after a device
synchronise), this library's launches per iteration (counted on an eager step), the card and its power limit, as one JSON line.
The VGG weights are torchvision's random initialisation (timing does not depend on them).

    python tools/gan_step_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import collections
import copy
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gan_ref, perceptual_ref  # noqa: E402
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import archs, gan, gan_train, ops  # noqa: E402
from vmambair_b200.perceptual import PerceptualLoss  # noqa: E402

B, LQ, NF = 9, 64, 64
LAYERS = {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1.0, "conv4_4": 1.0, "conv5_4": 1.0}
OPT = {"model_type": "MambaRealSRGAN", "l1_gt_usm": False, "percep_gt_usm": False, "gan_gt_usm": False,
       "train": {"ema_decay": 0.999,
                 "optim_g": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                 "optim_d": {"type": "Adam", "lr": 1e-4, "weight_decay": 0, "betas": [0.9, 0.99]},
                 "scheduler": {"type": "MultiStepLR", "milestones": [400000], "gamma": 0.5},
                 "lr_sr": 1e-4, "gamma_sr": 0.5, "lr_decay_sr": 300000, "warmup_iter": -1,
                 "pixel_opt": {"type": "L1Loss", "loss_weight": 1.0, "reduction": "mean"},
                 "perceptual_opt": {"type": "PerceptualLoss", "layer_weights": LAYERS, "vgg_type": "vgg19"},
                 "gan_opt": {"type": "GANLoss", "gan_type": "vanilla", "real_label_val": 1.0, "fake_label_val": 0.0,
                             "loss_weight": 1.0},
                 "net_d_iters": 1, "net_d_init_iters": 0}}


def composed(net_g, net_d_state, percep_state, dev):
    """the reference's iteration on torch modules around the same generator"""
    t = OPT["train"]
    net_d = gan_ref.UNetDiscriminatorSNRef(3, num_feat=NF).to(dev).train()
    net_d.load_state_dict(net_d_state)
    feats = perceptual_ref.features_from_state_dict(percep_state, "vgg19", LAYERS).to(dev)
    opt_g = torch.optim.Adam(net_g.parameters(), lr=t["optim_g"]["lr"], betas=t["optim_g"]["betas"])
    opt_d = torch.optim.Adam(net_d.parameters(), lr=t["optim_d"]["lr"], betas=t["optim_d"]["betas"])
    sched_d = torch.optim.lr_scheduler.MultiStepLR(opt_d, t["scheduler"]["milestones"], t["scheduler"]["gamma"])
    decay = t["ema_decay"]
    g_params = list(net_g.parameters())
    ema = [p.detach().clone() for p in g_params]
    it = [0]

    def step(lq, gt):
        it[0] += 1
        if it[0] > 1:  # basicsr's update_learning_rate
            sched_d.step()
        for pg in opt_g.param_groups:
            pg["lr"] = t["lr_sr"] * t["gamma_sr"] ** (it[0] // t["lr_decay_sr"])
        for p in net_d.parameters():
            p.requires_grad = False
        opt_g.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = net_g(lq).float()
            l_pix = F.l1_loss(out, gt)
            l_percep = perceptual_ref.perceptual_loss(feats, "vgg19", LAYERS, out, gt)
            l_gan = gan_ref.gan_loss(net_d(out), True, is_disc=False)
        (l_pix + l_percep + l_gan).backward()
        opt_g.step()
        losses = {"l_g_pix": l_pix.detach(), "l_g_percep": l_percep.detach(), "l_g_gan": l_gan.detach()}
        for p in net_d.parameters():
            p.requires_grad = True
        opt_d.zero_grad()
        for name, inp, real in (("real", gt, True), ("fake", out.detach().clone(), False)):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                pred = net_d(inp)
                l_d = gan_ref.gan_loss(pred, real, is_disc=True)
            losses[f"l_d_{name}"] = l_d.detach()
            losses[f"out_d_{name}"] = torch.mean(pred.detach())
            l_d.backward()
        opt_d.step()
        with torch.no_grad():
            torch._foreach_mul_(ema, decay)
            torch._foreach_add_(ema, g_params, alpha=1 - decay)
        return losses
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gan_step_bench measures on a GPU")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    g0 = archs.MambaRealSR11(inp_channels=3, out_channels=3, dim=48, num_blocks=[6, 2, 2, 1], num_refinement_blocks=6,
                             heads=[1, 2, 4, 8], ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias").to(dev).train()
    d0 = gan.UNetDiscriminatorSN(3, num_feat=NF, skip_connection=True).to(dev).train()
    percep = PerceptualLoss(LAYERS, vgg_type="vgg19", weights=None).to(dev)
    d_state, p_state = {k: v.clone() for k, v in d0.state_dict().items()}, percep.state_dict()
    gen = torch.Generator(device=dev).manual_seed(1)
    lq = torch.rand(B, 3, LQ, LQ, device=dev, generator=gen)
    gt = torch.rand(B, 3, 4 * LQ, 4 * LQ, device=dev, generator=gen)

    paths = {"composed": composed(copy.deepcopy(g0), d_state, p_state, dev)}
    trainers = {}
    for name in ("graph", "eager"):
        d = copy.deepcopy(d0)
        trainers[name] = gan_train.GANTrainer(copy.deepcopy(g0), d, OPT, 4, perceptual=percep, dtype=torch.bfloat16)
    trainers["graph"].capture(lq, gt)
    paths["graph"] = trainers["graph"].step
    paths["eager"] = trainers["eager"].step
    for _ in range(args.warmup):
        for fn in paths.values():
            fn(lq, gt)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    trainers["eager"].step(lq, gt)
    launches = ops.launch_count() - n0
    times = collections.defaultdict(list)
    for _ in range(args.steps):
        for name, fn in paths.items():
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn(lq, gt)
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
    losses = {k: float(v) for k, v in trainers["graph"].step(lq, gt).items()}
    if not all(v == v and abs(v) < 1e6 for v in losses.values()):
        raise SystemExit(f"gan_step_bench: a loss is not finite: {losses}")
    gpu, pl = gpu_info()
    print(json.dumps({"workload": f"GAN iteration (MambaRealSRGAN.optimize_parameters) b={B} LQ {LQ}x{LQ} GT {4 * LQ}x{4 * LQ}, "
                                  f"MambaRealSR11 + UNetDiscriminatorSN({NF}) + VGG19 perceptual, bf16 autocast",
                      "gpu": gpu, "power_limit": pl, "steps": args.steps,
                      "ms_per_step": {k: {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
                                      for k, v in times.items()},
                      "library_launches_per_step": launches, "losses_last": losses}))


if __name__ == "__main__":
    main()
