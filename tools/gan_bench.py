"""Time of the discriminator's work in one Real-ESRGAN GAN iteration at the recipe's shape (batch 9, 3 x 256 x 256, float32, TF32 at
torch's defaults), with vmambair_b200.gan's drop-ins and with the torch restatement oracle/gan_ref.py (nn.Conv2d + spectral_norm +
F.interpolate, the reference module's composition), alternated in one process.  One step is what MambaRealSRGAN_model.py:289-359 does
with net_d and cri_gan:
  G pass: D frozen, l_g_gan = GANLoss(D(fake), True) backpropagated into `fake` only;
  D step: GANLoss(D(gt), True, is_disc) and GANLoss(D(fake.detach()), False, is_disc) backpropagated into D's parameters, then D's
          Adam step on optim.FlatAdam (the same optimizer kernel on both sides).
Both sides start from the same state.  Reported: the median ms per step and its spread over `--steps` (CUDA events after a device
synchronise), launches of this library per step, CUDA kernels per step, and from a separate torch.profiler run the kernel time
inside aten convolutions (cuDNN) against everything else; the card name and power limit.

    python tools/gan_bench.py [--steps 30] [--warmup 5]
"""
import argparse
import collections
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gan_ref  # noqa: E402
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import gan, ops  # noqa: E402
from vmambair_b200.optim import FlatAdam  # noqa: E402

B, H, NF = 9, 256, 64


def make_side(cls, loss_fn, state, fake, gt):
    net = cls(3, num_feat=NF, skip_connection=True).cuda()
    net.load_state_dict(state)
    net.train()
    opt = FlatAdam(net.parameters(), lr=1e-4, betas=(0.9, 0.99))

    def step():
        for p in net.parameters():
            p.requires_grad_(False)
        f = fake.detach().requires_grad_()
        loss_fn(net(f), True, False).backward()
        for p in net.parameters():
            p.requires_grad_(True)
        loss_fn(net(gt), True, True).backward()
        loss_fn(net(fake.detach()), False, True).backward()
        opt.step()
    return step


def conv_split(prof):
    """(kernel ms inside aten convolution ops, kernel ms elsewhere, kernels) of a profile"""
    conv = other = 0.0
    n = 0
    for ev in prof.events():
        if not ev.kernels:
            continue
        p, in_conv = ev, False
        while p is not None:
            if "convolution" in p.name:
                in_conv = True
                break
            p = p.cpu_parent
        t = sum(k.duration for k in ev.kernels) / 1e3
        n += len(ev.kernels)
        if in_conv:
            conv += t
        else:
            other += t
    return conv, other, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gan_bench measures on a GPU"
    torch.manual_seed(0)
    state = {k: v.clone() for k, v in gan.UNetDiscriminatorSN(3, num_feat=NF).state_dict().items()}
    g = torch.Generator(device="cuda").manual_seed(1)
    fake = torch.randn(B, 3, H, H, device="cuda", generator=g)
    gt = torch.rand(B, 3, H, H, device="cuda", generator=g)
    crit = gan.GANLoss("vanilla", real_label_val=1.0, fake_label_val=0.0, loss_weight=1.0)
    sides = {
        "library": make_side(gan.UNetDiscriminatorSN, lambda x, real, d: crit(x, real, is_disc=d), state, fake, gt),
        "restatement": make_side(gan_ref.UNetDiscriminatorSNRef, lambda x, real, d: gan_ref.gan_loss(x, real, d), state, fake, gt),
    }
    for _ in range(args.warmup):
        for fn in sides.values():
            fn()
    torch.cuda.synchronize()
    times = collections.defaultdict(list)
    launches = {}
    for _ in range(args.steps):
        for name, fn in sides.items():
            torch.cuda.synchronize()
            n0 = ops.launch_count()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
            launches[name] = ops.launch_count() - n0
    split = {}
    for name, fn in sides.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                fn()
            torch.cuda.synchronize()
        conv, other, n = conv_split(prof)
        k = args.profile_steps
        split[name] = {"conv_kernel_ms_per_step": conv / k, "other_kernel_ms_per_step": other / k, "kernels_per_step": n / k}
    gpu, pl = gpu_info()
    print(json.dumps({"workload": f"UNetDiscriminatorSN GAN step b={B} 3x{H}x{H} num_feat={NF} fp32 (TF32 convs: "
                                  f"{torch.backends.cudnn.allow_tf32})",
                      "gpu": gpu, "power_limit": pl, "steps": args.steps,
                      "ms_per_step": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
                      "library_launches_per_step": launches, "profile": split}, indent=1))


if __name__ == "__main__":
    main()
