"""Flat-buffer optimizer of the training step: ONE kernel for Adam/AdamW + gradient clipping + EMA over all parameters
(reference: optimizer_g.step() / clip_grad_norm_ / model_ema(), SRGAN/VmambaIR/models/MambaSISR_model.py:141-147,
Deraining/basicsr/models/image_restoration_model.py:165-173, base_model.py:54-62; hyper-parameters of
SRGAN/options/MambaSISR15_x4.yml:78-82: Adam lr 2e-4, betas (0.9, 0.99), no weight decay; EMA decay 0.999).

The parameters are re-pointed to views of one flat fp32 buffer and their .grad to views of a second one -- the same buffer
vmambair_b200.dist all-reduces -- so the step touches 5 contiguous arrays instead of ~1 500 small tensors.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class FlatAdam:
    def __init__(self, params, lr=2e-4, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.0, decoupled=False, ema_decay=0.0,
                 max_grad_norm=0.0):
        self.params = [p for p in params if p.requires_grad]
        assert self.params and all(p.dtype == torch.float32 and p.is_cuda for p in self.params), "fp32 CUDA parameters"
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.n = n
        self.flat_param = torch.empty(n, dtype=torch.float32, device=dev)
        self.flat_grad = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        self.state = torch.zeros(4, dtype=torch.float32, device=dev)
        o = 0
        with torch.no_grad():
            for p in self.params:
                k = p.numel()
                self.flat_param[o:o + k].copy_(p.data.reshape(-1))
                p.data = self.flat_param[o:o + k].view_as(p)       # parameters live in the flat buffer from here on
                p.grad = self.flat_grad[o:o + k].view_as(p)        # autograd accumulates straight into the flat gradient
                o += k
        self.ema = self.flat_param.clone() if ema_decay > 0 else None
        self.lr, self.betas, self.eps, self.weight_decay, self.decoupled = lr, betas, eps, weight_decay, decoupled
        self.ema_decay, self.max_grad_norm = ema_decay, max_grad_norm
        # the .grad views exist from here on: let the fused backward kernels add into them directly (no AccumulateGrad launch per
        # parameter -- ~1 500 tiny kernels per step on the full SR net)
        from . import fused_train
        fused_train.set_direct_grads(True)

    def check_views(self):
        """.grad must still alias the flat buffer (zero_grad(set_to_none=True) would break it)"""
        o = 0
        for p in self.params:
            if p.grad is None or p.grad.data_ptr() != self.flat_grad.data_ptr() + 4 * o:
                p.grad = self.flat_grad[o:o + p.numel()].view_as(p)
            o += p.numel()

    @torch.no_grad()
    def step(self, grad_scale: float = 1.0, zero_grad: bool = True, lr_device: torch.Tensor | None = None):
        """lr_device: a float32 CUDA tensor whose first element is the learning rate, read by the kernel on the device (so that a
        captured CUDA graph follows a schedule that a kernel earlier in the stream writes); None: self.lr"""
        from . import fused_train
        if lr_device is not None and not (lr_device.dtype == torch.float32 and lr_device.device == self.flat_param.device):
            raise ValueError(f"FlatAdam.step: lr_device must be a float32 tensor on {self.flat_param.device}")
        fused_train.join_side_stream()  # normally already joined by the end-of-backward callback
        a = _lib.AdamArgs(param=self.flat_param.data_ptr(), grad=self.flat_grad.data_ptr(), exp_avg=self.exp_avg.data_ptr(),
                          exp_avg_sq=self.exp_avg_sq.data_ptr(), ema=self.ema.data_ptr() if self.ema is not None else None,
                          state=self.state.data_ptr(), n=self.n, lr=self.lr, beta1=self.betas[0], beta2=self.betas[1], eps=self.eps,
                          weight_decay=self.weight_decay, decoupled_weight_decay=int(self.decoupled), grad_scale=grad_scale,
                          max_grad_norm=self.max_grad_norm, ema_decay=self.ema_decay, zero_grad=int(zero_grad),
                          lr_dev=lr_device.data_ptr() if lr_device is not None else None)
        with torch.cuda.device(self.flat_param.device):
            st = C.c_void_p(torch.cuda.current_stream(self.flat_param.device).cuda_stream)
            _lib.check(_lib.lib().vmb_fused_adam(C.byref(a), st), "fused_adam")
        self.mark_written()

    def mark_written(self):
        """bump every parameter's version counter after a write behind autograd's back (the kernel above, a CUDA-graph replay of
        it, a copy into flat_param): the inference weight caches (fused._prepare, unet._cached, the SR tail's channels-last copy)
        key on _version and data_ptr, and neither changes when the flat buffer is written through its pointer or a view of it"""
        torch.autograd.graph.increment_version(self.params)

    def ema_state_dict(self, module: torch.nn.Module):
        """EMA weights under the module's parameter names (the reference's net_g_ema / `params_ema` checkpoint entry)"""
        out, o = {}, 0
        names = {id(p): n for n, p in module.named_parameters()}
        for p in self.params:
            out[names[id(p)]] = self.ema[o:o + p.numel()].view_as(p).clone()
            o += p.numel()
        return out
