"""Training path of one OSS block on the fused kernels: forward AND backward of every stage as this library's kernels
(SURVEY.md 8 a15 -- the autograd of LayerNorm, in_conv, depthwise conv + SiLU, cross-scan, x_proj / dt_proj, the selective scan,
merge + out_norm + gate, out_conv, the EFFN), replacing the torch-autograd-over-eager-ops path of round 1.

Reference semantics: MamberBlock.forward under autograd, SRGAN/VmambaIR/archs/MambaSISR6_arch.py:486-515 (SS2D_1.forward :486-498,
forward_corev1 :395-436, FeedForward :201-218); the training step that drives it is MambaSISRModel.optimize_parameters
(SRGAN/VmambaIR/models/MambaSISR_model.py:120-147).

Structure (three autograd Functions):
    prepare_block: ONE launch per block and step -> every 1x1-conv weight in kernel layout + its transpose, the folded x_proj/dt_proj
             matrix, A = -exp(A_logs), the flipped depthwise taps (vmb_prep_block_weights)
    _Front:  x -> norm1 + in_conv -> dwconv + SiLU -> x_proj/dt_proj (folded GEMM) -> cross-scan -> selective scan (checkpoints)
             -> merge + out_norm + SiLU(z) gate -> (y2, pooled sums)
    _Channel: pooled sums -> channel-direction OSS -> c         (vmb_channel_branch / vmb_channel_branch_bwd, one CTA per image;
             levels whose (2 dc, 16, C) state history exceeds one CTA's shared memory (C = 384) keep torch autograd)
    _Tail:   (y2, c, x) -> channel gate + out_conv + residual -> norm2 + project_in -> dwconv + GELU gate -> project_out + residual
A standalone SS2D_1 (ss2d_forward) runs _Front without norm1, _Channel, and _OutConv (channel gate + out_conv, no residual; its backward
is _Tail's out_conv section, _out_conv_bwd); prepare_block then prepares the attn weights only.

Backward kernels: vmb_pixlin with the transposed weight (data gradients of the five 1x1 convs), vmb_pixlin_wgrad (their weight and bias
gradients: mma.sync, split over pixels), vmb_selective_scan_bwd, vmb_cross_scan (the gathers pi_k and their inverses = pi_k with H
and W swapped, bit-exact permutations), vmb_sum4_add, vmb_merge_norm_gate_bwd, vmb_layernorm_fwd/bwd, vmb_dwconv3x3_bwd +
vmb_dwconv3x3 (flipped taps), vmb_channel_gate_bwd.  Every fp32 gradient accumulator of a Function's backward is a slice of ONE
zero-filled workspace.  Activations are saved in the compute dtype (bf16 under autocast), parameters stay fp32 and receive fp32
gradients.  fp32 activations (parity mode) send the weight gradients to the library GEMM.
"""
from __future__ import annotations

import contextlib

import torch

from . import ops


def _f32(t):
    return None if t is None else t.detach().float().contiguous()


def _p16(n):
    return (n + 15) // 16 * 16


def _acc(param, fallback):
    """fp32 accumulator of a parameter gradient: the parameter's own .grad when it is a contiguous fp32 buffer on the same device (the
    kernels ADD into it -- what autograd's AccumulateGrad would do with one more launch per parameter; with optim.FlatAdam the .grad
    buffers are views of the flat gradient the all-reduce and the optimizer kernel read), else the zero-filled `fallback` slice.
    -> (buffer shaped like fallback, direct?)"""
    g = getattr(param, "grad", None) if param is not None else None
    if _DIRECT_GRADS and g is not None and g.dtype == torch.float32 and g.is_contiguous() and g.device == fallback.device and \
            g.numel() == fallback.numel() and not torch.is_grad_enabled():
        return g.view(fallback.shape), True
    return fallback, False


class _Side:
    """Second stream for the weight-gradient kernels of the backward pass.  Nothing downstream of a block waits for its weight
    gradients (with direct .grad accumulation not even autograd does), while the data-gradient chain is a sequence of small-grid,
    latency-bound launches at the training batch (4 images): the wgrad GEMMs and LayerNorm recomputations run beside it
    (fork: side waits for the current stream; join: one wait at the end of the backward pass, queued as an autograd callback --
    also under CUDA-graph capture, where this becomes a fork / join of graph branches)."""
    stream = {}      # device index -> torch.cuda.Stream
    keep = []        # tensors the side-stream kernels read: kept alive until the join
    armed = False
    on = True        # False: everything on the current stream (the single-stream comparison of the tests)


def join_side_stream():
    """make the current stream wait for the weight-gradient stream (idempotent; optim.FlatAdam.step calls it before it reads .grad).
    Nothing to do once the end-of-backward callback has joined it: waiting then would also tie a CUDA-graph capture to a stream the
    capture never forked (a graph whose backward did not use the side stream, after an earlier eager backward that did)."""
    if _Side.armed:
        _side_join()


def _side_join():
    _Side.armed = False
    for st in _Side.stream.values():
        torch.cuda.current_stream(st.device).wait_stream(st)
    _Side.keep.clear()


@contextlib.contextmanager
def _side(ok, dev, *keep):
    """run the enclosed launches on the side stream when `ok` (their results go nowhere but into .grad buffers)"""
    if not (ok and _Side.on and _DIRECT_GRADS and not torch.is_grad_enabled()):
        yield False
        return
    st = _Side.stream.get(dev.index)
    if st is None:
        st = _Side.stream[dev.index] = torch.cuda.Stream(dev)
    if not _Side.armed:
        torch.autograd.Variable._execution_engine.queue_callback(_side_join)
        _Side.armed = True
    _Side.keep.extend(keep)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        yield True


_DIRECT_GRADS = False  # opt-in (optim.FlatAdam turns it on): only valid for .backward()-style accumulation into .grad


def set_direct_grads(on: bool):
    """True: the backward kernels add the parameter gradients straight into existing fp32 .grad buffers and hand autograd None for
    them (valid for loss.backward() accumulation, NOT for torch.autograd.grad(...)); False: gradients are returned to autograd"""
    global _DIRECT_GRADS
    _DIRECT_GRADS = bool(on)


class _Arena:
    """views carved out of one flat tensor (16-element aligned offsets)"""

    def __init__(self, dtype, device):
        self.dtype, self.device, self.specs, self.n = dtype, device, [], 0

    def add(self, name, *shape):
        k = 1
        for s in shape:
            k *= s
        self.specs.append((name, self.n, shape, k))
        self.n += _p16(k)

    def build(self, zero=False):
        buf = (torch.zeros if zero else torch.empty)(max(self.n, 16), dtype=self.dtype, device=self.device)
        return {name: buf[o:o + k].view(*shape) for name, o, shape, k in self.specs}


def prepare_block(mod, dtype, device):
    """kernel-layout weights of one OSS block (or of a standalone SS2D_1: the attn weights only) for this step, ONE launch
    (vmb_prep_block_weights).  D = d_model, C = d_inner (the scanned width E)."""
    a = getattr(mod, "attn", mod)
    f = getattr(mod, "ffn", None)
    D, C, R, N = a.d_model, a.d_inner, a.dt_rank, a.d_state
    Mb = 4 * (C + 2 * N)
    w = _Arena(dtype, device)
    mats = [("Win", 2 * C, D), ("WinT", D, 2 * C), ("Wbig", Mb, C), ("WbigT", C, Mb), ("Wout", D, C), ("WoutT", C, D)]
    if f is not None:
        h = f.project_out.weight.shape[1]
        mats += [("Wpin", 2 * h, C), ("WpinT", C, 2 * h), ("Wpout", C, h), ("WpoutT", h, C)]
    for name, rows, cols in mats:
        w.add(name, rows, _p16(cols))
    W = w.build()
    g = _Arena(torch.float32, device)
    g.add("A", 4 * C, N)
    g.add("cwf", C, 9)
    if f is not None:
        g.add("fdwf", 2 * h, 9)
    G = g.build()
    d = lambda p: p.detach()
    Job = ops.PrepJob
    jobs = [
        Job(type=ops.PREP_PAD_COPY, src=d(a.in_conv.weight), dst=W["Win"], M=2 * C, K=D, ld=_p16(D)),
        Job(type=ops.PREP_TRANSPOSE, src=d(a.in_conv.weight), dst=W["WinT"], M=2 * C, K=D, ld=_p16(2 * C)),
        Job(type=ops.PREP_FOLD, src=d(a.x_proj_weight), src2=d(a.dt_projs_weight), dst=W["Wbig"], dst2=W["WbigT"], M=C, K=R, N2=2 * N,
            ld=_p16(C), ld2=_p16(Mb)),
        Job(type=ops.PREP_PAD_COPY, src=d(a.out_conv.weight), dst=W["Wout"], M=D, K=C, ld=_p16(C)),
        Job(type=ops.PREP_TRANSPOSE, src=d(a.out_conv.weight), dst=W["WoutT"], M=D, K=C, ld=_p16(D)),
    ]
    if f is not None:
        jobs += [
            Job(type=ops.PREP_PAD_COPY, src=d(f.project_in.weight), dst=W["Wpin"], M=2 * h, K=C, ld=_p16(C)),
            Job(type=ops.PREP_TRANSPOSE, src=d(f.project_in.weight), dst=W["WpinT"], M=2 * h, K=C, ld=_p16(2 * h)),
            Job(type=ops.PREP_PAD_COPY, src=d(f.project_out.weight), dst=W["Wpout"], M=C, K=h, ld=_p16(h)),
            Job(type=ops.PREP_TRANSPOSE, src=d(f.project_out.weight), dst=W["WpoutT"], M=C, K=h, ld=_p16(C)),
        ]
    jobs += [
        Job(type=ops.PREP_NEG_EXP, src=d(a.A_logs), dst=G["A"], M=4 * C, K=N),
        Job(type=ops.PREP_FLIP_TAPS, src=d(a.conv2d.weight), dst=G["cwf"], M=C, K=9),
    ]
    if f is not None:
        jobs.append(Job(type=ops.PREP_FLIP_TAPS, src=d(f.dwconv.weight), dst=G["fdwf"], M=2 * h, K=9))
    for j in jobs:
        assert j.src.dtype == torch.float32 and j.src.is_contiguous(), "fp32 contiguous parameters"
    ops.prep_block_weights(jobs, dtype)
    W.update(G)
    return W


class _Front(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, n1w, n1b, w_in, b_in, cw, cb, x_proj_w, dt_w, dt_b, A_logs, Ds, on_w, on_b, Win, WinT, Wbig, WbigT, A, cwf):
        with torch.autocast("cuda", enabled=False):
            B, D, H, W = x.shape
            L = H * W
            C, N, R = cw.shape[0], A_logs.shape[1], dt_w.shape[2]
            ln_mode = 0 if n1w is None else 1 if n1b is not None else 2  # 0: standalone SS2D_1, no norm1 in front of in_conv
            x3 = x.contiguous().view(B, D, L)
            xz = ops.pixlin(x3, Win, _f32(b_in), ln=(ln_mode, _f32(n1w), _f32(n1b)) if ln_mode else None)  # (B,2C,L): [x_pre | z_pre]
            cw9 = _f32(cw.view(C, 9))
            xc = ops.dwconv3x3(xz[:, :C], cw9, _f32(cb), C, H, W, 0)
            dbl4 = ops.pixlin(xc, Wbig).view(B, 4, C + 2 * N, L)   # delta, B, C of the four directions, pixel order
            xs, dts, bc = ops.cross_scan_multi([([xc] * 4, C, None), ([dbl4[:, k, :C] for k in range(4)], C, None),
                                                ([dbl4[:, k, C:] for k in range(4)], 2 * N, None)], H, W)  # one launch
            ys, ckpt = ops.selective_scan_fwd(xs.view(B, 4 * C, L), dts.view(B, 4 * C, L), A, bc[:, :, :N], bc[:, :, N:], _f32(Ds),
                                              _f32(dt_b.reshape(-1)), True, need_ckpt=True)
            y2, pooled, ws = ops.merge_norm_gate(ys.view(B, 4, C, L), xz[:, C:], _f32(on_w), _f32(on_b), C, H, W,
                                                 z_preact=True, return_ws=True)
            ctx.save_for_backward(x3, xz, xc, xs, dts, bc, ckpt, ws, A, n1w, n1b, w_in, cw, cb, x_proj_w, dt_w, dt_b, Ds, on_w, on_b,
                                  WinT, WbigT, cwf, b_in)
            ctx.geom = (B, D, C, H, W, N, R, ln_mode)
        return y2.view(B, C, H, W), pooled

    @staticmethod
    def backward(ctx, dy2, dpooled):
        with torch.autocast("cuda", enabled=False):
            (x3, xz, xc, xs, dts, bc, ckpt, ws, A, n1w, n1b, w_in, cw, cb, x_proj_w, dt_w, dt_b, Ds, on_w, on_b,
             WinT, WbigT, cwf, b_in) = ctx.saved_tensors
            B, D, C, H, W, N, R, ln_mode = ctx.geom
            L, dt_, dev = H * W, x3.dtype, x3.device
            Mb = 4 * (C + 2 * N)
            z = _Arena(torch.float32, dev)  # every fp32 accumulator of this backward: one zero fill
            for name, shape in (("onw", (C,)), ("onb", (C,)), ("dA", (4 * C, N)), ("dD", (4 * C,)), ("dbias", (4 * C,)), ("dbig", (Mb, C)),
                                ("dcw", (C, 9)), ("dcb", (C,)), ("dwin", (2 * C, D)), ("dbin", (2 * C,)), ("n1w", (D,)), ("n1b", (D,))):
                z.add(name, *shape)
            Z = z.build(zero=True)
            dy2 = dy2.to(dt_).contiguous().view(B, C, L)
            dpooled = None if dpooled is None else dpooled.float().contiguous()
            dxz = torch.empty_like(xz)  # [d x_pre | d z_pre]
            (g_onw, k_onw), (g_onb, k_onb) = _acc(on_w, Z["onw"]), _acc(on_b, Z["onb"])
            dm = ops.merge_norm_gate_bwd(ws, xz[:, C:], dy2, dpooled, _f32(on_w), _f32(on_b), C, L, dz_out=dxz[:, C:], phase="data")
            with _side(k_onw and k_onb, dev, ws, xz, dy2, dpooled):
                d_onw, d_onb = ops.merge_norm_gate_bwd(ws, xz[:, C:], dy2, dpooled, _f32(on_w), _f32(on_b), C, L, dz_out=None,
                                                       zeroed=(g_onw, g_onb), phase="params")
            dys = ops.cross_scan([dm] * 4, C, H, W)  # gradient of the merged output, gathered into the four scan orders
            (g_dD, k_dD), (g_dbias, k_dbias) = _acc(Ds, Z["dD"]), _acc(dt_b, Z["dbias"])
            du, ddelta, dA, dB, dC, dD, dbias = ops.selective_scan_bwd(
                xs.view(B, 4 * C, L), dts.view(B, 4 * C, L), A, bc[:, :, :N], bc[:, :, N:], _f32(Ds), _f32(dt_b.reshape(-1)),
                dys.view(B, 4 * C, L), ckpt, True, zeroed=(Z["dA"], g_dD, g_dbias), deterministic=False)
            # back to pixel order: pi_k^-1 is pi_k with H and W swapped
            ddbl = torch.empty((B, 4, C + 2 * N, L), dtype=dt_, device=dev)
            dxc4 = ops.cross_scan_multi([([du.view(B, 4, C, L)[:, k] for k in range(4)], C, None),
                                         ([ddelta.view(B, 4, C, L)[:, k] for k in range(4)], C, ddbl[:, :, :C]),
                                         ([dB[:, k] for k in range(4)], N, ddbl[:, :, C:C + N]),
                                         ([dC[:, k] for k in range(4)], N, ddbl[:, :, C + N:])], W, H)[0]  # one launch
            ddbl = ddbl.view(B, Mb, L)
            dxc = ops.sum4_add(dxc4, ops.pixlin(ddbl, WbigT))  # x_proj data gradient + the four direction gradients of u
            xw, dtw = x_proj_w.detach(), dt_w.detach()
            gx, gd = getattr(x_proj_w, "grad", None), getattr(dt_w, "grad", None)
            k_big = _DIRECT_GRADS and gx is not None and gd is not None and gx.dtype == gd.dtype == torch.float32 and not torch.is_grad_enabled()
            with _side(k_big, dev, ddbl, xc, Z["dbig"]):
                dbig = ops.pixlin_wgrad(ddbl, xc, out=Z["dbig"], deterministic=False).view(4, C + 2 * N, C)
                d_xproj = torch.cat([torch.bmm(dtw.transpose(1, 2), dbig[:, :C]), dbig[:, C:]], 1)  # [W_dt^T dW ; dW[C:]]
                d_dtw = torch.bmm(dbig[:, :C], xw[:, :R].transpose(1, 2))                            # dW W_x[:R]^T
                if k_big:
                    gx.add_(d_xproj)
                    gd.add_(d_dtw)
                    d_xproj = d_dtw = None
            # depthwise conv + SiLU
            (g_cw, k_cw), (g_cb, k_cb) = _acc(cw, Z["dcw"]), _acc(cb, Z["dcb"])
            dv = ops.dwconv3x3_bwd(xz[:, :C], _f32(cw.view(C, 9)), _f32(cb), dxc, C, H, W, 0, phase="data")
            with _side(k_cw and (cb is None or k_cb), dev, xz, dv):
                d_cw, d_cb = ops.dwconv3x3_bwd(xz[:, :C], _f32(cw.view(C, 9)), _f32(cb), None, C, H, W, 0, zeroed=(g_cw, g_cb),
                                               phase="params", dv=dv)
            ops.dwconv3x3(dv, cwf, None, C, H, W, 2, out=dxz[:, :C])
            # in_conv + norm1
            dxn = ops.pixlin(dxz, WinT)
            (g_win, k_win), (g_bin, k_bin) = _acc(w_in, Z["dwin"]), _acc(b_in, Z["dbin"])
            with _side(k_win and (b_in is None or k_bin), dev, x3, dxz):
                xn = ops.layernorm_fwd(x3, ln_mode, _f32(n1w), _f32(n1b)) if ln_mode else x3
                d_win = ops.pixlin_wgrad(dxz, xn, out=g_win, dbias=g_bin, deterministic=False).view_as(w_in)
            (g_n1w, k_n1w), (g_n1b, k_n1b) = _acc(n1w, Z["n1w"]), _acc(n1b, Z["n1b"])
            if ln_mode:
                dx, st1 = ops.layernorm_bwd(x3, dxn, ln_mode, _f32(n1w), phase="data")
                with _side(k_n1w and (n1b is None or k_n1b), dev, x3, dxn, st1):
                    d_n1w, d_n1b = ops.layernorm_bwd(x3, dxn, ln_mode, _f32(n1w), zeroed=(g_n1w, g_n1b), phase="params", stats=st1)
            else:
                dx, d_n1w, d_n1b = dxn, None, None
            dA_logs = dA * A  # A = -exp(A_logs)
        drop = lambda t, direct: None if direct else t  # accumulated straight into .grad: nothing for autograd to add
        return (dx.view(B, D, H, W), drop(d_n1w, k_n1w), drop(d_n1b, k_n1b), drop(d_win, k_win), drop(g_bin, k_bin),
                drop(d_cw.view_as(cw), k_cw), drop(d_cb, k_cb), d_xproj, d_dtw, drop(dbias.view_as(dt_b), k_dbias),
                dA_logs, drop(dD, k_dD), drop(d_onw, k_onw), drop(d_onb, k_onb), None, None, None, None, None, None)


class _Tail(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y2, c, x, w_out, b_out, n2w, n2b, w_pin, b_pin, fdw, fdwb, w_pout, b_pout, gate_mode,
                Wout, WoutT, Wpin, WpinT, Wpout, WpoutT, fdwf):
        with torch.autocast("cuda", enabled=False):
            B, C, H, W = x.shape
            L = H * W
            h = w_pout.shape[1]
            ln_mode = 1 if n2b is not None else 2
            x3, y23 = x.contiguous().view(B, C, L), y2.contiguous().view(B, C, L)
            cg = c.detach().float().contiguous()
            x1 = ops.pixlin(y23, Wout, _f32(b_out), residual=x3, gate=cg, gate_mode=gate_mode)
            t = ops.pixlin(x1, Wpin, _f32(b_pin), ln=(ln_mode, _f32(n2w), _f32(n2b)))
            gg = ops.dwconv3x3(t, _f32(fdw.view(2 * h, 9)), _f32(fdwb), h, H, W, 1)
            out = ops.pixlin(gg, Wpout, _f32(b_pout), residual=x1)
            ctx.save_for_backward(y23, cg, x1, t, gg, w_out, b_out, n2w, n2b, w_pin, b_pin, fdw, fdwb, w_pout, b_pout,
                                  WoutT, WpinT, WpoutT, fdwf)
            ctx.geom = (B, C, H, W, h, ln_mode, gate_mode)
        return out.view(B, C, H, W)

    @staticmethod
    def backward(ctx, dout):
        with torch.autocast("cuda", enabled=False):
            (y23, cg, x1, t, gg, w_out, b_out, n2w, n2b, w_pin, b_pin, fdw, fdwb, w_pout, b_pout,
             WoutT, WpinT, WpoutT, fdwf) = ctx.saved_tensors
            B, C, H, W, h, ln_mode, gate_mode = ctx.geom
            L, dt_, dev = H * W, x1.dtype, x1.device
            z = _Arena(torch.float32, dev)
            for name, shape in (("wpout", (C, h)), ("bpout", (C,)), ("fdw", (2 * h, 9)), ("fdwb", (2 * h,)), ("wpin", (2 * h, C)),
                                ("bpin", (2 * h,)), ("n2w", (C,)), ("n2b", (C,)), ("wb", (B, C, C)), ("bout", (C,))):
                z.add(name, *shape)
            Z = z.build(zero=True)
            dout3 = dout.to(dt_).contiguous().view(B, C, L)
            # project_out
            dgg = ops.pixlin(dout3, WpoutT)
            (g_wpout, k_wpout), (g_bpout, k_bpout) = _acc(w_pout, Z["wpout"]), _acc(b_pout, Z["bpout"])
            with _side(k_wpout and (b_pout is None or k_bpout), dev, dout3, gg):
                d_wpout = ops.pixlin_wgrad(dout3, gg, out=g_wpout, dbias=g_bpout if b_pout is not None else None, deterministic=False).view_as(w_pout)
            # depthwise conv + GELU gate
            (g_fdw, k_fdw), (g_fdwb, k_fdwb) = _acc(fdw, Z["fdw"]), _acc(fdwb, Z["fdwb"])
            dv = ops.dwconv3x3_bwd(t, _f32(fdw.view(2 * h, 9)), _f32(fdwb), dgg, h, H, W, 1, phase="data")
            with _side(k_fdw and (fdwb is None or k_fdwb), dev, t, dv):
                d_fdw, d_fdwb = ops.dwconv3x3_bwd(t, _f32(fdw.view(2 * h, 9)), _f32(fdwb), None, h, H, W, 1, zeroed=(g_fdw, g_fdwb),
                                                  phase="params", dv=dv)
            dt = ops.dwconv3x3(dv, fdwf, None, 2 * h, H, W, 2)
            # project_in + norm2 (+ the residual branch of the EFFN)
            dx1n = ops.pixlin(dt, WpinT)
            (g_wpin, k_wpin), (g_bpin, k_bpin) = _acc(w_pin, Z["wpin"]), _acc(b_pin, Z["bpin"])
            with _side(k_wpin and (b_pin is None or k_bpin), dev, x1, dt):
                x1n = ops.layernorm_fwd(x1, ln_mode, _f32(n2w), _f32(n2b))
                d_wpin = ops.pixlin_wgrad(dt, x1n, out=g_wpin, dbias=g_bpin if b_pin is not None else None, deterministic=False).view_as(w_pin)
            (g_n2w, k_n2w), (g_n2b, k_n2b) = _acc(n2w, Z["n2w"]), _acc(n2b, Z["n2b"])
            dx1, st2 = ops.layernorm_bwd(x1, dx1n, ln_mode, _f32(n2w), add=dout3, phase="data")
            with _side(k_n2w and (n2b is None or k_n2b), dev, x1, dx1n, st2):
                d_n2w, d_n2b = ops.layernorm_bwd(x1, dx1n, ln_mode, _f32(n2w), zeroed=(g_n2w, g_n2b), phase="params", stats=st2)
            # out_conv with the channel gate in front, residual behind
            dy2, dc, d_wout, d_bout = _out_conv_bwd(dx1, y23, cg, w_out, b_out, WoutT, gate_mode, Z["wb"], Z["bout"])
        drop = lambda t, direct: None if direct else t
        return (dy2.view(B, C, H, W), dc, dx1.view(B, C, H, W), d_wout, d_bout,
                drop(d_n2w, k_n2w), drop(d_n2b, k_n2b), drop(d_wpin, k_wpin), drop(g_bpin, k_bpin) if b_pin is not None else None,
                drop(d_fdw.view_as(fdw), k_fdw), drop(d_fdwb, k_fdwb), drop(d_wpout, k_wpout),
                drop(g_bpout, k_bpout) if b_pout is not None else None, None, None, None, None, None, None, None, None)


def _out_conv_bwd(dx1, y23, cg, w_out, b_out, WoutT, gate_mode, wb_acc, bout_acc):
    """backward of the channel gate + out_conv: dx1 (B,D,L) contiguous, the gradient of out_conv's output; y23 (B,E,L) its gated input
    before the gate; cg (B,E) fp32 the gate; wb_acc (B,D,E) / bout_acc (D) zero-filled fp32 accumulators.
    -> (dy2 (B,E,L), dgate (B,E) fp32, d out_conv.weight, d out_conv.bias), the last two None when added straight into .grad"""
    dev = dx1.device
    dyg = ops.pixlin(dx1, WoutT)
    dy2, dc = ops.channel_gate_bwd(dyg, y23, cg, gate_mode)
    g_bout, k_bout = _acc(b_out, bout_acc)
    g_wout = getattr(w_out, "grad", None)
    k_wout = _DIRECT_GRADS and g_wout is not None and g_wout.dtype == torch.float32 and not torch.is_grad_enabled()
    with _side(k_wout and (b_out is None or k_bout), dev, dx1, y23, cg, wb_acc):
        wb = ops.pixlin_wgrad(dx1, y23, per_batch=True, out=wb_acc, dbias=g_bout, deterministic=False)  # (B, C_out, C_in): scaled per image by the gate
        if gate_mode == 1:
            d_wout = (wb * (1.0 + cg)[:, None, :]).sum(0)
        else:  # y + c: the gate adds c[b,k] * sum_p dx1[b,m,p]  (per-image row sums: B*C values)
            d_wout = wb.sum(0) + torch.einsum("bm,bk->mk", dx1.float().sum(2), cg)
        if k_wout:
            g_wout.add_(d_wout.view_as(g_wout))
            d_wout = None
    return dy2, dc, None if d_wout is None else d_wout.view_as(w_out), None if b_out is None or k_bout else g_bout


class _OutConv(torch.autograd.Function):
    """channel gate + out_conv of a standalone SS2D_1 (no residual behind): (y2 (B,E,H,W), c (B,E) fp32) -> (B,D,H,W)"""

    @staticmethod
    def forward(ctx, y2, c, w_out, b_out, gate_mode, Wout, WoutT):
        with torch.autocast("cuda", enabled=False):
            B, C, H, W = y2.shape
            D = w_out.shape[0]
            y23 = y2.contiguous().view(B, C, H * W)
            cg = c.detach().float().contiguous()
            out = ops.pixlin(y23, Wout, _f32(b_out), gate=cg, gate_mode=gate_mode)
            ctx.save_for_backward(y23, cg, w_out, b_out, WoutT)
            ctx.geom = (B, C, D, H, W, gate_mode)
        return out.view(B, D, H, W)

    @staticmethod
    def backward(ctx, dout):
        with torch.autocast("cuda", enabled=False):
            y23, cg, w_out, b_out, WoutT = ctx.saved_tensors
            B, C, D, H, W, gate_mode = ctx.geom
            z = _Arena(torch.float32, y23.device)
            z.add("wb", B, D, C)
            z.add("bout", D)
            Z = z.build(zero=True)
            dout3 = dout.to(y23.dtype).contiguous().view(B, D, H * W)
            dy2, dc, d_wout, d_bout = _out_conv_bwd(dout3, y23, cg, w_out, b_out, WoutT, gate_mode, Z["wb"], Z["bout"])
        return dy2.view(B, C, H, W), dc, d_wout, d_bout, None, None, None


class _Channel(torch.autograd.Function):
    """channel-direction OSS on the pooled sums: vmb_channel_branch forward, vmb_channel_branch_bwd backward (one CTA per image each)"""

    @staticmethod
    def forward(ctx, pooled, inv_count, C, dc, Rc, N, cin_w, cin_b, xc_proj, dtc_w, dtc_b, Ac_logs, Dsc, cout_w, cout_b, cn_w, cn_b):
        prm = dict(cin_w=_f32(cin_w.view(-1)) if cin_w is not None else None, cin_b=_f32(cin_b), xc_proj=_f32(xc_proj), dtc_w=_f32(dtc_w),
                   dtc_b=_f32(dtc_b), Ac_logs=_f32(Ac_logs), Dsc=_f32(Dsc), cout_w=_f32(cout_w.view(-1)) if cout_w is not None else None,
                   cout_b=_f32(cout_b), cn_w=_f32(cn_w), cn_b=_f32(cn_b), dc=dc, Rc=Rc, N=N)
        pooled = pooled.detach().float().contiguous()
        ctx.prm, ctx.inv_count, ctx.C = prm, inv_count, C
        ctx.params = (cin_w, cin_b, xc_proj, dtc_w, dtc_b, Ac_logs, Dsc, cout_w, cout_b, cn_w, cn_b)  # leaves: their .grad is the accumulator
        ctx.save_for_backward(pooled)
        ctx.shapes = [None if t is None else t.shape for t in (cin_w, cin_b, xc_proj, dtc_w, dtc_b, Ac_logs, Dsc, cout_w, cout_b, cn_w, cn_b)]
        return ops.channel_branch(pooled, inv_count, prm, C)

    @staticmethod
    def backward(ctx, dc_out):
        (pooled,) = ctx.saved_tensors
        keys = ("cin_w", "cin_b", "xc_proj", "dtc_w", "dtc_b", "Ac_logs", "Dsc", "cout_w", "cout_b", "cn_w", "cn_b")
        into = {}
        if _DIRECT_GRADS and not torch.is_grad_enabled():
            for k, prm in zip(keys, ctx.params):
                g = getattr(prm, "grad", None) if prm is not None else None
                if g is not None and g.dtype == torch.float32 and g.is_contiguous() and g.device == pooled.device:
                    into[k] = g.view(-1)
        dpooled, g = ops.channel_branch_bwd(pooled, ctx.inv_count, ctx.prm, ctx.C, dc_out, into=into)
        grads = [None if (shp is None or k in into) else g[k].view(shp) for k, shp in zip(keys, ctx.shapes)]
        return (dpooled, None, None, None, None, None, *grads)


def channel_gate(a, pooled, L):
    """c (B, C) fp32 from the pooled sums: the fused kernels when the level fits one CTA's shared memory, else torch autograd"""
    C = pooled.shape[1]
    prm_probe = dict(dc=a.dc_inner, Rc=a.dtc_rank, N=a.dc_state)
    if ops.channel_branch_bwd_supported(C, prm_probe):
        has_cio = hasattr(a, "conv_cin")
        cn = a.channel_norm.body
        return _Channel.apply(pooled, 1.0 / L, C, a.dc_inner, a.dtc_rank, a.dc_state,
                              a.conv_cin.weight if has_cio else None, a.conv_cin.bias if has_cio else None, a.xc_proj_weight,
                              a.dtc_projs_weight, a.dtc_projs_bias, a.Ac_logs, a.Dsc,
                              a.conv_cout.weight if has_cio else None, a.conv_cout.bias if has_cio else None, cn.weight, cn.bias)
    with torch.autocast("cuda", enabled=False):
        return a.cforward_pooled(pooled * (1.0 / L))


def _front(a, x, P, norm=None):
    """_Front of attn module `a` (norm: the block's norm1 LayerNorm, fused into in_conv) -> (y2, pooled sums)"""
    on = a.out_norm.body
    return _Front.apply(x, None if norm is None else norm.weight, getattr(norm, "bias", None), a.in_conv.weight, a.in_conv.bias,
                        a.conv2d.weight, a.conv2d.bias, a.x_proj_weight, a.dt_projs_weight, a.dt_projs_bias, a.A_logs, a.Ds, on.weight,
                        on.bias, P["Win"], P["WinT"], P["Wbig"], P["WbigT"], P["A"], P["cwf"])


def block_forward(block, x: torch.Tensor) -> torch.Tensor:
    """MamberBlock.forward with autograd on the fused kernels (x: (B,C,H,W) CUDA tensor in the compute dtype)."""
    a, f = block.attn, block.ffn
    L = x.shape[2] * x.shape[3]
    n2 = block.norm2.body
    with torch.no_grad():
        P = prepare_block(block, x.dtype, x.device)
    y2, pooled = _front(a, x, P, block.norm1.body)
    c = channel_gate(a, pooled, L)  # (B, C) fp32: channel-direction OSS on the pooled descriptor
    return _Tail.apply(y2, c, x, a.out_conv.weight, a.out_conv.bias, n2.weight, getattr(n2, "bias", None), f.project_in.weight,
                       f.project_in.bias, f.dwconv.weight, f.dwconv.bias, f.project_out.weight, f.project_out.bias,
                       1 if a.gate == "mul" else 2, P["Wout"], P["WoutT"], P["Wpin"], P["WpinT"], P["Wpout"], P["WpoutT"], P["fdwf"])


def ss2d_forward(a, x: torch.Tensor) -> torch.Tensor:
    """SS2D_1.forward of a standalone module with autograd on the fused kernels (x: (B,D,H,W) CUDA tensor in the compute dtype):
    _Front without norm1, the channel gate, then _OutConv (gate + out_conv, no residual)."""
    L = x.shape[2] * x.shape[3]
    with torch.no_grad():
        P = prepare_block(a, x.dtype, x.device)
    y2, pooled = _front(a, x, P)
    c = channel_gate(a, pooled, L)  # (B, E) fp32
    return _OutConv.apply(y2, c, a.out_conv.weight, a.out_conv.bias, 1 if a.gate == "mul" else 2, P["Wout"], P["WoutT"])
