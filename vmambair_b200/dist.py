"""Batch-axis data parallelism: the only parallelism VmambaIR uses (reference: DistributedDataParallel in
Deraining/basicsr/models/base_model.py:67-85; loss reduce :369).  Images are independent units, so every rank
holds a replica and its own slice of the batch; the one collective of a training step is a single flat
all-reduce of the gradients (NCCL over NVLink/NVSwitch on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_batch(global_batch: int, rank: int, world: int):
    """contiguous slice [lo, hi) of the global batch owned by `rank` (EnlargedSampler-style even split)."""
    per = (global_batch + world - 1) // world
    lo = min(rank * per, global_batch)
    return lo, min(lo + per, global_batch)


class FlatGradAllReduce:
    """One all-reduce per step over a single flat buffer holding every gradient (48 MB fp32 for the full SR net)."""

    def __init__(self, params, dtype=torch.float32):
        self.params = [p for p in params if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(n, dtype=dtype, device=dev)
        self.views = []
        o = 0
        for p in self.params:
            self.views.append(self.flat[o:o + p.numel()].view_as(p))
            o += p.numel()

    def attach(self):
        """make every .grad a view of the flat buffer (no copies at reduce time)."""
        for p, v in zip(self.params, self.views):
            p.grad = v if v.dtype == p.dtype else None
        return self

    def reduce(self, world: int, group=None):
        """gathers whatever is not already a view (a parameter whose dtype differs from the flat buffer keeps its own .grad and is
        copied in; a parameter that received no gradient this step contributes zeros, not last step's values), then one all-reduce"""
        if any(p.grad is not v for p, v in zip(self.params, self.views)):
            for p, v in zip(self.params, self.views):
                if p.grad is None:
                    v.zero_()
                elif p.grad is not v:
                    v.copy_(p.grad)
                    if v.dtype == p.dtype:
                        p.grad = v
        if world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
            self.flat.div_(world)

    def zero(self):
        self.flat.zero_()


def broadcast_params(module: torch.nn.Module, src: int = 0):
    """identical replicas at start (DDP does this at construction).  The broadcast writes through p.data, whose version counter is
    not p's, so each parameter's version is bumped after it: the inference weight caches key on it."""
    if dist.is_initialized() and dist.get_world_size() > 1:
        for p in module.parameters():
            dist.broadcast(p.data, src)
            torch.autograd.graph.increment_version(p)
