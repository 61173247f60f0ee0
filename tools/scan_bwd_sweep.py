"""state-split sweep of the TMA selective-scan backward (VMB_SCAN_SS_BWD) at the north-star shape, next to the reference kernel."""
import json, os, sys, importlib.util
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vmambair_b200 import ops
from tools.scan_bench import bench

dev = "cuda"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "selective_scan_cuda_core.so")
refm = None
if os.path.exists(so):
    spec = importlib.util.spec_from_file_location("selective_scan_cuda_core", so)
    refm = importlib.util.module_from_spec(spec); spec.loader.exec_module(refm)
for dt in (torch.bfloat16,):
    for B in (1, 4, 8):
        D, K, N, L = 384, 4, 16, 4096
        torch.manual_seed(0)
        u = torch.randn(B, D, L, device=dev).to(dt); delta = (0.5 * torch.rand(B, D, L, device=dev)).to(dt)
        A = -0.5 * torch.rand(D, N, device=dev); Bm = torch.randn(B, K, N, L, device=dev).to(dt); Cm = torch.randn(B, K, N, L, device=dev).to(dt)
        Dv = torch.randn(D, device=dev); bias = 0.5 * torch.rand(D, device=dev); dout = torch.randn_like(u)
        out, ck = ops.selective_scan_fwd(u, delta, A, Bm, Cm, Dv, bias, True, True)
        rec = dict(B=B)
        if refm is not None:
            o_r, x_r = refm.fwd(u, delta, A, Bm, Cm, Dv, bias, True, 1)
            rec["ref_us_per_img"] = round(bench(lambda: refm.bwd(u, delta, A, Bm, Cm, Dv, bias, dout, x_r, True, 1), flush=flush) * 1e3 / B, 1)
        for ss in (0, 1, 2, 4):
            if ss:
                os.environ["VMB_SCAN_SS_BWD"] = str(ss)
            else:
                os.environ.pop("VMB_SCAN_SS_BWD", None)
            ms = bench(lambda: ops.selective_scan_bwd(u, delta, A, Bm, Cm, Dv, bias, dout, ck, True), flush=flush)
            rec[f"ss{ss}" if ss else "auto"] = round(ms * 1e3 / B, 1)
        print(json.dumps(rec), flush=True)
