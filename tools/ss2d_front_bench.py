"""Where the time of the SS2D core's front goes: the three launches behind the in_conv (dwconv3x3_t, then pixlin on x with
w_big02 and on its (W,H) copy with w_big13) at the light SR net's block geometries, B = 8 unless SF_B is set.

Each launch is replayed alone from a CUDA graph, timed with CUDA events, the L2 flushed (a 256 MB write) before it; the chain is
also timed as one graph of its three launches (with the library's programmatic dependent launch, as in the bench step); medians
of SF_REPS (default 30) rounds.  Algorithmic bytes per launch are its operands read once and its output written
once; GB/s is against the H100 SXM data sheet's 3.35 TB/s (a reference line, not a measurement).  `fused_floor_us` prices the
bytes a single fused launch would still move (x read; xc, xt, d02, d13 written; weights read) at the best rate any of the three
launches reaches.

The second table times pixlin alone at the x_proj shape (64 x 64, K = C) while varying the output rows M and the reduction K
separately: if the time follows M (the output tiles a CTA writes) and not K (the input it reads and multiplies), the GEMM is
bound by its output stores, and a fused prologue that saves input reads cannot shorten it.  One JSON line per row."""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from vmambair_b200 import ops  # noqa: E402

HBM = 3350.0
GEOMS = [(48, 64, 64), (96, 64, 64), (96, 32, 32), (192, 16, 16), (384, 8, 8)]  # (C, H, W) of the light SR net's blocks
N = 16
ES = 2  # bf16


def timed(fn, flush, reps):
    """median device time of fn's launches, replayed from a CUDA graph (no host launch gaps inside the window)"""
    ev = lambda: torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        flush.zero_()
        s, e = ev(), ev()
        s.record()
        graph.replay()
        e.record()
        torch.cuda.synchronize()
        t.append(s.elapsed_time(e) * 1e3)
    return statistics.median(t)


def main():
    dev = torch.device("cuda", 0)
    B = int(os.environ.get("SF_B", 8))
    reps = int(os.environ.get("SF_REPS", 30))
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = None
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": pl, "batch": B}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    g = torch.Generator().manual_seed(0)
    dt = torch.bfloat16
    for C, H, W in GEOMS:
        L, M2 = H * W, 2 * (C + 2 * N)
        xz = torch.randn(B, 2 * C, L, generator=g).to(dev, dt)
        dw = (torch.randn(C, 9, generator=g) / 3).to(dev)
        dw_b = (torch.randn(C, generator=g) * 0.1).to(dev)
        w02 = ops.pad_weight((torch.randn(M2, C, generator=g) / C ** 0.5).to(dev, dt))
        w13 = ops.pad_weight((torch.randn(M2, C, generator=g) / C ** 0.5).to(dev, dt))
        x = xz[:, :C]  # the channel slice the block passes
        xc, xt = ops.dwconv3x3_t(x, dw, dw_b, C, H, W)
        act, d, w = ES * B * C * L, ES * B * M2 * L, ES * M2 * C
        stages = [("dwconv3x3_t", lambda: ops.dwconv3x3_t(x, dw, dw_b, C, H, W), 3 * act),
                  ("pixlin02", lambda: ops.pixlin(xc, w02), act + d + w),
                  ("pixlin13", lambda: ops.pixlin(xt, w13), act + d + w)]

        def chain():
            a, b = ops.dwconv3x3_t(x, dw, dw_b, C, H, W)
            ops.pixlin(a, w02)
            ops.pixlin(b, w13)

        row = dict(C=C, H=H, W=W, B=B)
        best = 0.0
        for name, fn, nb in stages:
            us = timed(fn, flush, reps)
            row[name] = dict(us=round(us, 2), MB=round(nb / 1e6, 2), GBs=round(nb / us / 1e3, 1),
                             frac_of_3350=round(nb / us / 1e3 / HBM, 3))
            best = max(best, nb / us / 1e3)
        row["stage_sum_us"] = round(sum(row[n]["us"] for n, _, _ in stages), 2)
        row["chain_us"] = round(timed(chain, flush, reps), 2)
        fused_bytes = 3 * act + 2 * d + 2 * w
        row["fused_MB"] = round(fused_bytes / 1e6, 2)
        row["fused_floor_us"] = round(fused_bytes / best / 1e3, 2)
        print(json.dumps(row), flush=True)

    # pixlin at the full-resolution x_proj shape: time against output rows M (K = 96) and against K (M = 256)
    P = 64 * 64
    for K, M in [(96, 64), (96, 128), (96, 256), (96, 512), (48, 256), (192, 256), (384, 256)]:
        xk = torch.randn(B, K, P, generator=g).to(dev, dt)
        wk = ops.pad_weight((torch.randn(M, K, generator=g) / K ** 0.5).to(dev, dt))
        us = timed(lambda: ops.pixlin(xk, wk), flush, reps)
        rd, wr = ES * B * K * P + ES * M * K, ES * B * M * P
        print(json.dumps(dict(sweep="pixlin", K=K, M=M, P=P, B=B, us=round(us, 2), read_MB=round(rd / 1e6, 2),
                              write_MB=round(wr / 1e6, 2), GBs=round((rd + wr) / us / 1e3, 1),
                              write_GBs=round(wr / us / 1e3, 1))), flush=True)


if __name__ == "__main__":
    main()
