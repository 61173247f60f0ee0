"""Micro-benchmark of the selective-scan operator at the north-star shape (SURVEY.md 8d)."""
import argparse
import json
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vmambair_b200 import ops


def bench(fn, iters=20, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(True), torch.cuda.Event(True)
        torch.cuda._sleep(400_000)  # let the host run ahead so launch latency is not timed
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--C", type=int, nargs="+", default=[96])
    ap.add_argument("--L", type=int, nargs="+", default=[4096])
    ap.add_argument("--dtypes", nargs="+", default=["bf16", "fp32"])
    ap.add_argument("--bwd", action="store_true")
    ap.add_argument("--ref", action="store_true", help="also time the reference CUDA kernel rebuilt for sm_90a (oracle/_ref)")
    a = ap.parse_args()
    dev = "cuda"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    peak = 6486.5
    for dn in a.dtypes:
        dt = {"bf16": torch.bfloat16, "fp32": torch.float32, "fp16": torch.float16}[dn]
        s = 2 if dt != torch.float32 else 4
        for C in a.C:
            for L in a.L:
                for B in a.B:
                    K, N = 4, 16
                    D = K * C
                    torch.manual_seed(0)
                    u = torch.randn(B, D, L, device=dev).to(dt)
                    delta = (0.5 * torch.rand(B, D, L, device=dev)).to(dt)
                    A = -0.5 * torch.rand(D, N, device=dev)
                    Bm = torch.randn(B, K, N, L, device=dev).to(dt)
                    Cm = torch.randn(B, K, N, L, device=dev).to(dt)
                    Dv = torch.randn(D, device=dev)
                    bias = 0.5 * torch.rand(D, device=dev)
                    ms = bench(lambda: ops.selective_scan_fwd(u, delta, A, Bm, Cm, Dv, bias, True, True), flush=flush)
                    byts = B * (s * (3 * D * L + 2 * K * N * L) + 4 * (D * N + 2 * D))
                    rec = dict(op="scan_fwd", dtype=dn, B=B, C=C, L=L, ms=round(ms, 4), us_per_img=round(ms * 1e3 / B, 3),
                               GBps=round(byts / ms / 1e6, 1), frac_measured_peak=round(byts / ms / 1e6 / peak, 4),
                               Gupd_per_s=round(B * D * L * N / ms / 1e6, 1))
                    if a.bwd:
                        dout = torch.randn_like(u)
                        out, ck = ops.selective_scan_fwd(u, delta, A, Bm, Cm, Dv, bias, True, True)
                        msb = bench(lambda: ops.selective_scan_bwd(u, delta, A, Bm, Cm, Dv, bias, dout, ck, True), flush=flush)
                        bb = B * (s * (5 * D * L + 4 * K * N * L))
                        rec.update(bwd_ms=round(msb, 4), bwd_us_per_img=round(msb * 1e3 / B, 3), bwd_GBps=round(bb / msb / 1e6, 1))
                    if a.ref:
                        import importlib.util
                        so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "selective_scan_cuda_core.so")
                        spec = importlib.util.spec_from_file_location("selective_scan_cuda_core", so)
                        refm = importlib.util.module_from_spec(spec); spec.loader.exec_module(refm)
                        msr = bench(lambda: refm.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1), flush=flush)
                        rec.update(ref_ms=round(msr, 4), ref_us_per_img=round(msr * 1e3 / B, 3), speedup_vs_ref=round(msr / ms, 2))
                        if a.bwd:
                            o_r, x_r = refm.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1)
                            msrb = bench(lambda: refm.bwd(u, delta, A, Bm, Cm, Dv, bias, dout, x_r, True, 1), flush=flush)
                            rec.update(ref_bwd_ms=round(msrb, 4), bwd_speedup_vs_ref=round(msrb / msb, 2))
                    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
