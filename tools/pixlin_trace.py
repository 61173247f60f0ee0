"""Timeline of one persistent wgmma pixlin launch (VMB_TC_TRACE=1): per-CTA %globaltimer stamps."""
import sys, os, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["VMB_PIXLIN_TC"] = "2"
import torch
from vmambair_b200 import ops, _lib
dev, dt, B, P = "cuda", torch.bfloat16, 8, 4096
for name, (K, M, kind) in {"w_big96": (96, 256, "plain"), "pin96": (96, 510, "ln"), "pout96": (255, 96, "res")}.items():
    x = torch.randn(B, K, P, device=dev).to(dt); res = torch.randn(B, M, P, device=dev).to(dt)
    w = ops.pad_weight((torch.randn(M, K, device=dev) / K ** 0.5).to(dt)); bias = torch.randn(M, device=dev)
    lw, lb = torch.rand(K, device=dev) + 0.5, torch.randn(K, device=dev) * 0.1
    def call():
        if kind == "ln": ops.pixlin(x, w, bias, ln=(1, lw, lb))
        elif kind == "plain": ops.pixlin(x, w)
        else: ops.pixlin(x, w, bias, residual=res)
    os.environ["VMB_TC_TRACE"] = "0"
    for _ in range(3): call()
    torch.cuda.synchronize()
    os.environ["VMB_TC_TRACE"] = "1"
    call(); torch.cuda.synchronize()
    buf = (ctypes.c_longlong * (160 * 64))()
    assert _lib.lib().vmb_debug_tc_trace(buf, 160 * 64) == 0
    ctas = min(160, torch.cuda.get_device_properties(0).multi_processor_count)  # one CTA per SM, <= 160 traced
    t = [[buf[c * 64 + i] for i in range(64)] for c in range(ctas)]
    t0 = min(r[0] for r in t)
    print(name, "kernel span us:", (max(r[3] for r in t) - t0) / 1e3)
    for c in (0, 73):
        r = t[c]
        print("  cta", c, "start+%.2f setup %.2f weights %.2f end %.2f" % ((r[0] - t0) / 1e3, (r[1] - r[0]) / 1e3, (r[2] - r[1]) / 1e3, (r[3] - t0) / 1e3))
        print("     tile: landed  pro_done  mma_saw  mma_issued  epi_saw  epi_done   (us after weights resident)")
        for i in range(8):
            e = r[4 + 6 * i: 10 + 6 * i]
            if e[5] > 0:
                print("     %d: " % i + "  ".join("%7.2f" % ((v - r[2]) / 1e3) if v > 0 else "      -" for v in e))
