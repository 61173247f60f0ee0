"""A few launches of one pixlin shape (for ncu): PB_SHAPE in {pin96,in_conv96,w_big96,pout96}."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vmambair_b200 import ops
dev, dt, B, P = "cuda", torch.bfloat16, 8, 4096
K, M, kind = {"pin96": (96, 510, "ln"), "in_conv96": (96, 192, "ln_act"), "w_big96": (96, 256, "plain"), "pout96": (255, 96, "res")}[os.environ.get("PB_SHAPE", "pin96")]
x = torch.randn(B, K, P, device=dev).to(dt); res = torch.randn(B, M, P, device=dev).to(dt)
w = ops.pad_weight((torch.randn(M, K, device=dev) / K ** 0.5).to(dt)); bias = torch.randn(M, device=dev)
lw, lb = torch.rand(K, device=dev) + 0.5, torch.randn(K, device=dev) * 0.1
for _ in range(3):
    if kind == "ln": ops.pixlin(x, w, bias, ln=(1, lw, lb))
    elif kind == "ln_act": ops.pixlin(x, w, bias, ln=(1, lw, lb), act=(M // 2, M))
    elif kind == "plain": ops.pixlin(x, w)
    else: ops.pixlin(x, w, bias, residual=res)
torch.cuda.synchronize()
