"""Per-shape sustained timing of the 1x1-conv GEMM (vmb_pixlin) on the shapes of the light SISR net at B=8, 64x64.
Four rotating buffer sets (> L2 together for the big shapes), 12 launches per CUDA graph, 20 replays."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vmambair_b200 import ops

dev, dt = "cuda", torch.bfloat16
B, P = int(os.environ.get("PB_B", 8)), int(os.environ.get("PB_P", 4096))
SHAPES = [("in_conv96", 96, 192, "ln_act"), ("w_big96", 96, 256, "plain"), ("out_conv96", 96, 96, "gate_res"),
          ("pin96", 96, 510, "ln"), ("pout96", 255, 96, "res"),
          ("in_conv48", 48, 96, "ln_act"), ("w_big48", 48, 160, "plain"), ("out_conv48", 48, 48, "gate_res"),
          ("pin48", 48, 254, "ln"), ("pout48", 127, 48, "res")]
if os.environ.get("PB_TRAIN"):  # the GEMMs of one training block (forward + data gradients), C = 96 and C = 48
    SHAPES = [("in_conv96", 96, 192, "ln"), ("w_big96", 96, 512, "plain"), ("out_conv96", 96, 96, "gate_res"), ("pin96", 96, 510, "ln"),
              ("pout96", 255, 96, "res"), ("d_pout96", 96, 255, "plain"), ("d_pin96", 510, 96, "plain"), ("d_out96", 96, 96, "plain"),
              ("d_big96", 512, 96, "plain"), ("d_in96", 192, 96, "plain"),
              ("in_conv48", 48, 96, "ln"), ("w_big48", 48, 320, "plain"), ("out_conv48", 48, 48, "gate_res"), ("pin48", 48, 254, "ln"),
              ("pout48", 127, 48, "res"), ("d_pout48", 48, 127, "plain"), ("d_pin48", 254, 48, "plain"), ("d_out48", 48, 48, "plain"),
              ("d_big48", 320, 48, "plain"), ("d_in48", 96, 48, "plain")]
for name, K, M, kind in SHAPES:
    sets = []
    for _ in range(4):
        x = torch.randn(B, K, P, device=dev).to(dt)
        sets.append(dict(x=x, out=torch.empty(B, M, P, device=dev, dtype=dt), res=torch.randn(B, M, P, device=dev).to(dt)))
    w = ops.pad_weight((torch.randn(M, K, device=dev) / K ** 0.5).to(dt))
    bias = torch.randn(M, device=dev)
    lw, lb = torch.rand(K, device=dev) + 0.5, torch.randn(K, device=dev) * 0.1
    gate = torch.randn(B, K, device=dev) * 0.3

    def call(s):
        if kind == "ln_act":
            return ops.pixlin(s["x"], w, bias, ln=(1, lw, lb), act=(M // 2, M), out=s["out"])
        if kind == "plain":
            return ops.pixlin(s["x"], w, out=s["out"])
        if kind == "gate_res":
            return ops.pixlin(s["x"], w, bias, residual=s["res"], gate=gate, gate_mode=1, out=s["out"])
        if kind == "ln":
            return ops.pixlin(s["x"], w, bias, ln=(1, lw, lb), out=s["out"])
        return ops.pixlin(s["x"], w, bias, residual=s["res"], out=s["out"])

    nbytes = 2 * B * P * (K + M + (M if "res" in kind else 0))
    row = dict(shape=name, K=K, M=M, kind=kind, MB=round(nbytes / 1e6, 1))
    call(sets[0]); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(12):
            call(sets[i % 4])
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    for _ in range(20):
        g.replay()
    e.record(); torch.cuda.synchronize()
    us = s.elapsed_time(e) / (20 * 12) * 1e3
    row["us"] = round(us, 2); row["GBs"] = round(nbytes / us / 1e3, 0)
    print(json.dumps(row), flush=True)
