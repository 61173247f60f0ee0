"""Per-site timing of the U-Net's non-OSS stages: vmb_conv3x3 (+ folded shuffle / concatenation slice / add) vs the torch ops
the reference runs (nn.Conv2d on cuDNN + pixel_(un)shuffle + cat / interpolate + add).  B = 8, bf16, light SR net geometry.
  python tools/conv_bench.py [--batch 8] [--hw 64]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from vmambair_b200 import ops


def timeit(fn, n=10, reps=20):
    """device time per call inside a CUDA graph of `reps` back-to-back calls (no host launch latency in the number; warm L2)"""
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(3):
            fn()
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for _ in range(reps):
                fn()
        ts = []
        for _ in range(n):
            s, e = torch.cuda.Event(True), torch.cuda.Event(True)
            s.record(st)
            g.replay()
            e.record(st)
            st.synchronize()
            ts.append(s.elapsed_time(e) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--hw", type=int, default=64)
    a = ap.parse_args()
    B, S, dt = a.batch, a.hw, torch.bfloat16
    sites = [("patch_embed", 3, 48, S, ops.CONV_PLAIN), ("down1_2", 48, 24, S, ops.CONV_UNSHUFFLE2),
             ("down2_3", 96, 48, S // 2, ops.CONV_UNSHUFFLE2), ("down3_4", 192, 96, S // 4, ops.CONV_UNSHUFFLE2),
             ("up4_3", 384, 768, S // 8, ops.CONV_SHUFFLE2), ("up3_2", 192, 384, S // 4, ops.CONV_SHUFFLE2),
             ("up2_1", 96, 192, S // 2, ops.CONV_SHUFFLE2)]
    for name, cin, cout, hw, mode in sites:
        x = torch.randn(B, cin, hw, hw, device="cuda", dtype=dt)
        w = (torch.randn(cout, cin, 3, 3, device="cuda") / (3 * cin ** 0.5)).to(dt)
        wp = ops.pack_conv3x3_weight(w, dt)
        post = {ops.CONV_PLAIN: lambda y: y, ops.CONV_UNSHUFFLE2: lambda y: F.pixel_unshuffle(y, 2),
                ops.CONV_SHUFFLE2: lambda y: F.pixel_shuffle(y, 2)}[mode]
        t_ref = timeit(lambda: post(F.conv2d(x, w, None, padding=1)))
        t_our = timeit(lambda: ops.conv3x3(x, wp, None, cout, mode))
        gflop = 2 * 9 * cin * cout * hw * hw * B / 1e9
        print(json.dumps({"site": name, "cin": cin, "cout": cout, "hw": hw, "gflop": round(gflop, 3), "torch_us": round(t_ref, 1),
                          "vmb_us": round(t_our, 1)}))
    # SR tail: last conv (NHWC in) + nearest-upsampled image + NHWC -> NCHW
    x = torch.randn(B, 96, 4 * S, 4 * S, device="cuda", dtype=dt).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(3, 96, 3, 3, device="cuda") / 30).to(dt)
    wcl = w.contiguous(memory_format=torch.channels_last)
    b = torch.randn(3, device="cuda")
    img = torch.rand(B, 3, S, S, device="cuda", dtype=dt)
    wp = ops.pack_conv3x3_weight(w, dt)
    t_ref = timeit(lambda: F.conv2d(x, wcl, b.to(dt), padding=1).contiguous() + F.interpolate(img, scale_factor=4, mode="nearest"))
    t_our = timeit(lambda: ops.conv3x3(x, wp, b, 3, ops.CONV_ADD_NEAREST, add=img, add_scale=4, nhwc=True))
    print(json.dumps({"site": "conv_last + interpolate + add", "cin": 96, "cout": 3, "hw": 4 * S, "torch_us": round(t_ref, 1),
                      "vmb_us": round(t_our, 1)}))
    # skip concatenation + reduce_chan (level 3): torch.cat + 1x1 conv vs pixlin over the in-place buffer
    for name, c, hw in (("cat+reduce_chan_level3", 192, S // 4), ("cat+reduce_chan_level2", 96, S // 2)):
        u, e = torch.randn(B, c, hw, hw, device="cuda", dtype=dt), torch.randn(B, c, hw, hw, device="cuda", dtype=dt)
        w1 = (torch.randn(c, 2 * c, 1, 1, device="cuda") / (2 * c) ** 0.5).to(dt)
        cat = torch.cat([u, e], 1)
        wq = ops.pad_weight(w1.view(c, 2 * c))
        t_ref = timeit(lambda: F.conv2d(torch.cat([u, e], 1), w1))
        t_our = timeit(lambda: ops.pixlin(cat.view(B, 2 * c, hw * hw), wq))
        print(json.dumps({"site": name, "torch_us": round(t_ref, 1), "vmb_us": round(t_our, 1)}))


if __name__ == "__main__":
    main()
