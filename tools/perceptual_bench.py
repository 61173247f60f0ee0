"""Time of the GAN recipes' perceptual loss in one generator step (forward + backward into the generator output) at the recipe's shape,
with vmambair_b200.perceptual.PerceptualLoss and with torch's composition (oracle/perceptual_ref.py: torchvision's VGG19 `features` +
basicsr's loss restated) on the same weights, alternated in one process.  fp32 inputs, convolutions at torch's default TF32 setting.
Layers: conv1_2 0.1, conv2_2 0.1, conv3_4 1, conv4_4 1, conv5_4 1, criterion l1, use_input_norm.

Reported per batch size: median and min-max ms per step over `--steps` alternated rounds (CUDA events after a device synchronise),
library launches per step, and from a separate torch.profiler run the kernel time inside aten convolutions against everything else
and the kernels per step; the loss and gradient differences between the two sides; the bytes the drop-in keeps for the backward,
computed from the shapes; the conv chain alone (16 forward convolutions over 2B images + 16 data gradients over B) in NCHW and in
channels_last; the card name and power limit.

    python tools/perceptual_bench.py [--steps 20] [--warmup 3] [--batches 9 8]
"""
import argparse
import collections
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import perceptual_ref  # noqa: E402
from tools.gan_bench import conv_split  # noqa: E402
from tools.scan_oflex_bench import gpu_info  # noqa: E402
from vmambair_b200 import ops  # noqa: E402
from vmambair_b200.perceptual import PerceptualLoss  # noqa: E402

RECIPE = {"conv1_2": 0.1, "conv2_2": 0.1, "conv3_4": 1, "conv4_4": 1, "conv5_4": 1}
H = 256


def saved_bytes(loss, B, Hh, W):
    """bytes the drop-in keeps for the backward (codes and l1 signs), and what fp32 activations of the output half would take"""
    ours = full = 0
    for m, relu, pool, sites in loss.vgg.stages():
        c = m.out_channels
        cells = B * c * ((Hh + 1) // 2) * ((W + 1) // 2)
        ours += cells * (int(relu) + sum(1 for s in sites[:2] if s in loss.layer_weights))
        full += 4 * B * c * Hh * W
        if pool:
            Hh, W = Hh // 2, W // 2
    return ours, full


def conv_chain(loss, B, channels_last):
    """the 16 convolutions alone, on preallocated inputs and output gradients in one memory format: forward over 2B images, data
    gradient over B"""
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    layers, h, w = [], H, H
    for m, relu, pool, _ in loss.vgg.stages():
        mk = lambda *shape: torch.randn(shape, device="cuda").contiguous(memory_format=fmt)
        layers.append((m.weight.contiguous(memory_format=fmt), m.bias, mk(2 * B, m.in_channels, h, w), mk(B, m.out_channels, h, w)))
        if pool:
            h, w = h // 2, w // 2

    def step():
        for wt, b, xin, gout in layers:
            torch.ops.aten.convolution(xin, wt, b, [1, 1], [1, 1], [1, 1], False, [0, 0], 1)
            empty = gout.new_empty(1).expand((B,) + tuple(xin.shape[1:]))
            torch.ops.aten.convolution_backward(gout, empty, wt, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])
    return step


def time_round(fns, steps, warmup):
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    times, launches = collections.defaultdict(list), {}
    for _ in range(steps):
        for name, fn in fns.items():
            torch.cuda.synchronize()
            n0 = ops.launch_count()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
            launches[name] = ops.launch_count() - n0
    return ({k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}, launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--batches", type=int, nargs="+", default=[9, 8])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perceptual_bench measures on a GPU"
    torch.backends.cudnn.allow_tf32 = True
    torch.manual_seed(0)
    loss = PerceptualLoss(RECIPE, weights=None)
    with torch.no_grad():
        for m, *_ in loss.vgg.stages():
            m.bias.normal_(0.0, 0.05)
    feats = perceptual_ref.features_from_state_dict(loss.state_dict(), "vgg19", RECIPE).cuda()
    loss = loss.cuda()
    out = {"workload": f"PerceptualLoss VGG19 {RECIPE} l1, forward + backward into x, 3x{H}x{H} fp32, TF32 convs"}
    for B in args.batches:
        g = torch.Generator(device="cuda").manual_seed(B)
        x0, gt = torch.rand(B, 3, H, H, device="cuda", generator=g), torch.rand(B, 3, H, H, device="cuda", generator=g)
        res = {}

        def ours():
            x = x0.clone().requires_grad_()
            y = loss(x, gt)[0]
            y.backward()
            res["ours"] = (y.detach(), x.grad)

        def torch_comp():
            x = x0.clone().requires_grad_()
            y = perceptual_ref.perceptual_loss(feats, "vgg19", RECIPE, x, gt)
            y.backward()
            res["torch"] = (y.detach(), x.grad)

        sides = {"library": ours, "torch_composition": torch_comp}
        ms, launches = time_round(sides, args.steps, args.warmup)
        split = {}
        for name, fn in sides.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.profile_steps):
                    fn()
                torch.cuda.synchronize()
            conv, other, n = conv_split(prof)
            k = args.profile_steps
            split[name] = {"conv_kernel_ms_per_step": conv / k, "other_kernel_ms_per_step": other / k, "kernels_per_step": n / k}
        chains = {"nchw": conv_chain(loss, B, False), "channels_last": conv_chain(loss, B, True)}
        chain_ms, _ = time_round(chains, args.steps, args.warmup)
        # differences, and the float64 reference at this shape
        x64 = x0.double().requires_grad_()
        y64 = perceptual_ref.perceptual_loss(perceptual_ref.copy_to(feats, torch.float64), "vgg19", RECIPE, x64, gt.double())
        y64.backward()
        rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()
        ours_b, full_b = saved_bytes(loss, B, H, H)
        out[f"batch_{B}"] = {
            "ms_per_step": ms, "library_launches_per_step": launches, "profile": split, "conv_chain_ms": chain_ms,
            "loss": {"library": res["ours"][0].item(), "torch": res["torch"][0].item(), "float64": y64.item()},
            "grad_rel_err_vs_float64": {"library": rel(res["ours"][1], x64.grad), "torch": rel(res["torch"][1], x64.grad)},
            "saved_bytes_library": ours_b, "fp32_activation_bytes_x_half": full_b}
    gpu, pl = gpu_info()
    out.update(gpu=gpu, power_limit=pl, steps=args.steps)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
