"""Channel-branch kernel: v1 vs v2 sustained time (VMB_CH_V selects the version)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vmambair_b200 import archs, fused, ops
dim = 96
blk = archs.MamberBlock(dim=dim, num_heads=1, ffn_expansion_factor=2.66, bias=False, LayerNorm_type="WithBias", variant="sisr").cuda()
c = fused._prepare(blk, torch.bfloat16, torch.device("cuda"))
pooled = torch.randn(8, dim, device="cuda") * 40.0
for v in ("1", "2"):
    os.environ["VMB_CH_V"] = v
    ops.channel_branch(pooled, 1.0 / 4096, c["ch"], dim); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(20):
            ops.channel_branch(pooled, 1.0 / 4096, c["ch"], dim)
    g.replay(); torch.cuda.synchronize()
    s, e = torch.cuda.Event(True), torch.cuda.Event(True)
    s.record()
    for _ in range(10):
        g.replay()
    e.record(); torch.cuda.synchronize()
    print("v" + v, "us per launch: %.2f" % (s.elapsed_time(e) / 200 * 1e3))
