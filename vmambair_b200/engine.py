"""Public inference / training entry points around the drop-in networks.

InferenceEngine: static-shape, CUDA-graph-replayed forward with pinned host staging -- the call a user
makes to upscale a batch of LQ tiles (host tensor in, host tensor out).
"""
from __future__ import annotations

import copy

import torch

from . import ops

# parameters that stay fp32 when the network runs in bf16 (the scan keeps state/params in fp32,
# reference: csrc/selective_scan/cus/selective_scan.cpp:165-172,203,211)
_FP32_PARAMS = ("A_logs", "Ac_logs", "Ds", "Dsc", "dt_projs_bias", "dtc_projs_bias")


def cast_for_inference(net: torch.nn.Module, dtype: torch.dtype) -> torch.nn.Module:
    """In-place cast of `net` (callers that keep training the same module pass a copy: InferenceEngine deep-copies).
    Parameters the fused kernels consume in fp32 (LayerNorm affine, conv biases, scan parameters) keep an un-rounded fp32
    master in `p._vmb_master`, so a bf16 engine does not round them twice."""
    for name, p in net.named_parameters():
        if name.rsplit(".", 1)[-1] in _FP32_PARAMS:
            p.data = p.data.float()
        else:
            master = p.data.float() if (p.dim() == 1 and dtype != torch.float32) else None
            p.data = p.data.to(dtype)
            if master is not None:
                p._vmb_master = master
    return net


def fork_join_batch(fn, x: torch.Tensor, chains: int, side_streams) -> torch.Tensor:
    """fn(x) evaluated on `chains` contiguous sub-batches, sub-batch i > 0 on side_streams[i-1] (forked from / joined
    back to the current stream with events, so the same code captures into parallel branches of a CUDA graph).
    Images are independent units of the path, so the result is that of fn(x)."""
    if chains <= 1 or x.shape[0] % chains != 0:
        return fn(x)
    cur = torch.cuda.current_stream(x.device)
    per = x.shape[0] // chains
    outs = [None] * chains
    fork = torch.cuda.Event()
    fork.record(cur)
    for i, st in enumerate(side_streams[:chains - 1]):
        st.wait_event(fork)
        with torch.cuda.stream(st):
            outs[i + 1] = fn(x[(i + 1) * per:(i + 2) * per])
    outs[0] = fn(x[:per])
    for st in side_streams[:chains - 1]:
        ev = torch.cuda.Event()
        ev.record(st)
        cur.wait_event(ev)
    return torch.cat(outs, 0)


class InferenceEngine:
    def __init__(self, net: torch.nn.Module, batch: int, height: int, width: int, dtype=torch.bfloat16,
                 device="cuda", in_channels: int = 3, use_graph: bool = True, chains: int = 1, lowres_chains: int = 1):
        """chains > 1: the batch is split into `chains` independent sub-batches whose kernel chains are captured on
        parallel streams of ONE graph -- images are independent, and most stages of a 64x64 tile are latency-bound
        single-wave launches, so two chains fill the GPU better than one.
        lowres_chains > 1: only the levels below full resolution (1/2, 1/4, 1/8: 9 of the 27 OSS blocks of the light net,
        every launch there a fraction of a wave) run as that many parallel sub-batch branches; the full-resolution
        stages, which fill the GPU on their own, keep the whole batch."""
        self.device = torch.device(device)
        # the caller's module is left untouched (it may be the training replica): the engine owns a cast copy
        self.net = cast_for_inference(copy.deepcopy(net).to(self.device).eval(), dtype)
        self.dtype = dtype
        self.x_dev = torch.zeros(batch, in_channels, height, width, device=self.device, dtype=dtype)
        self.x_host = torch.zeros(batch, in_channels, height, width, dtype=dtype).pin_memory()
        self.stream = torch.cuda.Stream(self.device)
        self.graph = None
        self.launches_per_step = 0
        self.chains = chains if (chains > 1 and batch % chains == 0) else 1
        self.side = [torch.cuda.Stream(self.device) for _ in range(self.chains - 1)]
        if lowres_chains > 1 and hasattr(self.net, "set_lowres_chains"):
            self.net.set_lowres_chains(lowres_chains, [torch.cuda.Stream(self.device) for _ in range(lowres_chains - 1)])
        with torch.cuda.device(self.device), torch.no_grad():
            with torch.cuda.stream(self.stream):
                for _ in range(2):  # warm-up (cuDNN autotune, lazy module load) before capture
                    y = self._forward()
                n0 = ops.launch_count()
                y = self._forward()
                self.launches_per_step = ops.launch_count() - n0
            self.stream.synchronize()
            self.y_dev = y
            if use_graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.stream):
                    self.y_dev = self._forward()
                self.graph = g
        self.y_host = torch.empty(self.y_dev.shape, dtype=self.y_dev.dtype).pin_memory()

    def _forward(self):
        """net(x_dev); with chains > 1 the sub-batches run on forked streams and are joined into one output."""
        if self.chains == 1:
            return self.net(self.x_dev)
        cur = torch.cuda.current_stream(self.device)
        per = self.x_dev.shape[0] // self.chains
        outs = [None] * self.chains
        fork = torch.cuda.Event()
        fork.record(cur)
        for i, st in enumerate(self.side):
            st.wait_event(fork)
            with torch.cuda.stream(st):
                outs[i + 1] = self.net(self.x_dev[(i + 1) * per:(i + 2) * per])
        outs[0] = self.net(self.x_dev[:per])
        for st in self.side:
            ev = torch.cuda.Event()
            ev.record(st)
            cur.wait_event(ev)
        return torch.cat(outs, 0)

    @torch.no_grad()
    def step_device(self):
        """one forward on the resident input (x_dev -> y_dev), on self.stream"""
        with torch.cuda.stream(self.stream):
            if self.graph is not None:
                self.graph.replay()
            else:
                self.y_dev = self._forward()
        return self.y_dev

    @torch.no_grad()
    def run(self, x_host: torch.Tensor) -> torch.Tensor:
        """host (pinned or pageable) batch in -> host result out; H2D + forward + D2H on one stream.
        Returns the engine's reused pinned output buffer: the next run() overwrites it (clone() to keep a result)."""
        with torch.cuda.stream(self.stream):
            self.x_dev.copy_(x_host, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.y_dev = self._forward()
            self.y_host.copy_(self.y_dev, non_blocking=True)
        self.stream.synchronize()
        return self.y_host
