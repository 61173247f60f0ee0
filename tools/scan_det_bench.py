"""Cost of the deterministic mode: the atomic and the deterministic scan backward (and cross_selective_scan forward + backward, whose
backward also runs the weight-gradient GEMM) alternated in one process, CUDA events after warm-up, best of --rounds.  Shapes: the flat
scan backward at (B, D, L) = (8, 384, 4096), (1, 384, 4096) and (4, 192, 65536), bf16, N = 16, 4 groups; cross_selective_scan at
B = 4, C = 96, 64x64, bf16.  Prints one JSON line per shape with ms per call (every round and the best), the workspace bytes of each
mode, the card name and its power limit.

    python tools/scan_det_bench.py [--iters 20] [--warmup 3] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # torch's cuBLAS under use_deterministic_algorithms (weight unfold)
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vmambair_b200 import cross_scan, ops  # noqa: E402

SCAN_SHAPES = [(8, 384, 4096), (1, 384, 4096), (4, 192, 65536)]
N, G = 16, 4


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                            timeout=20).stdout.strip().splitlines()[0]
    except Exception as e:  # the record still names the card
        pl = f"unknown ({e})"
    return name, pl


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def workspace_bytes(fn):
    """the workspace sizes ops requests while fn runs"""
    seen, orig = [], ops._workspace

    def spy(nbytes, given, dev, who):
        seen.append(int(nbytes))
        return orig(nbytes, given, dev, who)
    ops._workspace = spy
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        ops._workspace = orig
    return seen


def alternate(variants, a):
    times = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, f in variants.items():
            times[k].append(timed(f, a.iters, a.warmup))
    rec = {}
    for k, v in times.items():
        rec[f"{k}_ms"] = [round(t, 4) for t in v]
        rec[f"{k}_ms_min"] = round(min(v), 4)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scan_det_bench: needs a CUDA device")
    name, pl = gpu_info()
    g = torch.Generator(device="cuda").manual_seed(0)
    dt = torch.bfloat16
    for b, D, L in SCAN_SHAPES:
        u = torch.randn(b, D, L, device="cuda", generator=g).to(dt)
        delta = (0.1 * torch.randn(b, D, L, device="cuda", generator=g) - 4.0).to(dt)
        A = -torch.arange(1, N + 1, dtype=torch.float32, device="cuda").repeat(D, 1)
        Bm = torch.randn(b, G, N, L, device="cuda", generator=g).to(dt)
        Cm = torch.randn(b, G, N, L, device="cuda", generator=g).to(dt)
        Dv = torch.randn(D, device="cuda", generator=g)
        bias = torch.rand(D, device="cuda", generator=g)
        _, ck = ops.selective_scan_fwd(u, delta, A, Bm, Cm, Dv, bias, True, need_ckpt=True)
        dout = torch.randn(b, D, L, device="cuda", generator=g).to(dt)
        variants = {k: (lambda det=det: ops.selective_scan_bwd(u, delta, A, Bm, Cm, Dv, bias, dout, ck, True, deterministic=det))
                    for k, det in (("atomic", False), ("det", True))}
        rec = {"op": "selective_scan_bwd", "B": b, "D": D, "L": L, "N": N, "G": G, "dtype": "bf16", "gpu": name, "power_limit": pl,
               "atomic_workspace_bytes": workspace_bytes(variants["atomic"])[0],
               "det_workspace_bytes": workspace_bytes(variants["det"])[0]}
        rec.update(alternate(variants, a))
        print(json.dumps(rec), flush=True)
        del u, delta, Bm, Cm, ck, dout, variants
        torch.cuda.empty_cache()

    B, C, H, W, R = 4, 96, 64, 64, 6
    x = torch.randn(B, C, H, W, device="cuda", generator=g).to(dt).requires_grad_()
    prm = [0.2 * torch.randn(4, R + 2 * N, C, device="cuda", generator=g), 0.1 * torch.randn(4, R + 2 * N, device="cuda", generator=g),
           0.3 * torch.randn(4, C, R, device="cuda", generator=g), 0.1 * torch.rand(4, C, device="cuda", generator=g) - 4.0,
           torch.log(torch.arange(1, N + 1, dtype=torch.float32, device="cuda")).repeat(4 * C, 1), torch.ones(4 * C, device="cuda")]
    prm = [p.requires_grad_() for p in prm]
    assert cross_scan.grouped_supported(C, H * W, N, dt)

    def step(det):
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            y = cross_scan.cross_selective_scan(x, *prm, out_norm=torch.nn.Identity())
            y.backward(torch.ones_like(y))
        finally:
            torch.use_deterministic_algorithms(prev)
    variants = {"atomic": lambda: step(False), "det": lambda: step(True)}
    rec = {"op": "cross_selective_scan fwd+bwd", "B": B, "C": C, "H": H, "W": W, "N": N, "dtype": "bf16", "gpu": name, "power_limit": pl,
           "atomic_workspace_bytes": workspace_bytes(variants["atomic"]), "det_workspace_bytes": workspace_bytes(variants["det"])}
    rec.update(alternate(variants, a))
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
