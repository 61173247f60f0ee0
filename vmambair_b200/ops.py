"""Thin torch-tensor front-end of the C-ABI (device pointers + strides -> library call).

Mirrors the reference binding `selective_scan_cuda_core.fwd/bwd`
(Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan.cpp:157-349): same argument
meaning, same checks, same RuntimeError behaviour.  `selective_scan_fwd_z` and `scan_gate_bwd` add what mamba_ssm's
`selective_scan_cuda` has on top (the z gate and its backward, pair-layout checkpoints holding the last state); the module
`vmambair_b200.selective_scan_cuda` composes them with `selective_scan_bwd` into that module's fwd / bwd.  Outputs are allocated here with torch (the
library owns nothing), on the input's device and current stream.
"""
from __future__ import annotations

import collections
import ctypes as C
import math

import torch

from . import _lib

_DT = {torch.float32: _lib.DT_F32, torch.bfloat16: _lib.DT_BF16, torch.float16: _lib.DT_F16}


_LAUNCHES = 0          # kernels of this library launched so far (host-side count)
_TIMING = None         # when a list: (tag, bytes, start_event, end_event) per library call (bench roofline)


def launch_count() -> int:
    return _LAUNCHES


def set_timing(records):
    """records: None (off) or a list that receives (tag, algorithmic_bytes, start_event, end_event)."""
    global _TIMING
    _TIMING = records


class _timed:
    def __init__(self, tag, nbytes, dev, kernels):
        self.tag, self.nbytes, self.dev, self.kernels = tag, nbytes, dev, kernels

    def __enter__(self):
        if _TIMING is not None and self.tag is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record(torch.cuda.current_stream(self.dev))

    def __exit__(self, *a):
        global _LAUNCHES
        _LAUNCHES += self.kernels
        if _TIMING is not None and self.tag is not None:
            self.e.record(torch.cuda.current_stream(self.dev))
            _TIMING.append((self.tag, self.nbytes, self.s, self.e))


def _run(name, t, tag, *args, nbytes=0, kernels=1):
    """The one way this module calls the library: `name`(*args, stream) on t's device and current stream, its status checked and
    its `kernels` launches counted.  Under set_timing the call is recorded as (tag, nbytes, events); tag None: counted, not timed.
    A struct argument is passed by reference (the argtypes in _lib.SYMBOLS declare a pointer)."""
    fn = getattr(_lib.lib(), name)
    with torch.cuda.device(t.device), _timed(tag, nbytes, t.device, kernels):
        _lib.check(fn(*args, _stream(t)), name)


def _stream(t: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _ptr4(ts):
    """up to four tensors -> a `void* [4]` member, zero-padded"""
    return (C.c_void_p * 4)(*[t.data_ptr() for t in ts])


def _rev4(revs):
    """up to four direction flags -> an `int rev[4]` member, zero-padded"""
    return (C.c_int * 4)(*map(int, revs))


def _check_common(u, delta, A, B, C_, D, delta_bias, who):
    if u.dtype not in _DT:
        raise RuntimeError(f"{who}: input dtype must be float32/float16/bfloat16, got {u.dtype}")
    if A.dtype != torch.float32:
        raise RuntimeError(f"{who}: A must be float32")
    for n, t in (("delta", delta), ("B", B), ("C", C_)):
        if t.dtype != u.dtype:
            raise RuntimeError(f"{who}: {n}.dtype {t.dtype} != u.dtype {u.dtype}")
    for n, t in (("u", u), ("delta", delta), ("A", A), ("B", B), ("C", C_)):
        if not t.is_cuda:
            raise RuntimeError(f"{who}: {n} must be a CUDA tensor")
    if u.dim() != 3 or B.dim() != 4 or C_.dim() != 4 or A.dim() != 2:
        raise RuntimeError(f"{who}: expected u (B,D,L), A (D,N), B/C (B,G,N,L)")
    b, d, l = u.shape
    n = A.shape[1]
    g = B.shape[1]
    if tuple(delta.shape) != (b, d, l) or tuple(A.shape) != (d, n) or tuple(B.shape) != (b, g, n, l) \
            or tuple(C_.shape) != (b, g, n, l):
        raise RuntimeError(f"{who}: shape mismatch u{tuple(u.shape)} delta{tuple(delta.shape)} A{tuple(A.shape)} "
                           f"B{tuple(B.shape)} C{tuple(C_.shape)}")
    for nme, t in (("u", u), ("delta", delta), ("B", B), ("C", C_)):
        if t.stride(-1) != 1 and t.size(-1) != 1:
            raise RuntimeError(f"{who}: {nme}.stride(-1) must be 1")
    if not A.is_contiguous():
        raise RuntimeError(f"{who}: A must be contiguous")
    for nme, t in (("D", D), ("delta_bias", delta_bias)):
        if t is not None:
            if t.dtype != torch.float32 or not t.is_cuda or tuple(t.shape) != (d,) or not t.is_contiguous():
                raise RuntimeError(f"{who}: {nme} must be a contiguous float32 CUDA tensor of shape ({d},)")
    return b, d, l, n, g


def _deterministic(flag) -> bool:
    """None: follow torch.use_deterministic_algorithms(); True / False: override it."""
    return torch.are_deterministic_algorithms_enabled() if flag is None else bool(flag)


def _workspace(nbytes, given, dev, who):
    """uint8 device buffer of at least nbytes: the caller's (16 B aligned, contiguous), else a fresh one.  Its contents never matter."""
    if nbytes < 0:
        raise RuntimeError(f"{who}: {_lib.lib().vmb_last_error().decode()}")
    if given is None:
        return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    if not given.is_cuda or not given.is_contiguous() or given.numel() * given.element_size() < nbytes or given.data_ptr() % 16:
        raise RuntimeError(f"{who}: workspace must be a contiguous, 16 B aligned CUDA tensor of at least {nbytes} bytes")
    return given


def ckpt_interval() -> int:
    return _lib.lib().vmb_scan_ckpt_interval()


def selective_scan_fwd(u, delta, A, B, C_, D=None, delta_bias=None, delta_softplus=False, need_ckpt=True, out_float=False):
    """-> (out, ckpt).  out has delta's dtype/shape; ckpt is the opaque fp32 checkpoint tensor.
    out_float: out is fp32 whatever the input dtype -- with bf16 / fp16 inputs the fp32 accumulator is stored without rounding
    (the reference's selective_scan_cuda_oflex, cusoflex/selective_scan_oflex.cpp:219,235-239)."""
    b, d, l, n, g = _check_common(u, delta, A, B, C_, D, delta_bias, "selective_scan_fwd")
    out_f32 = bool(out_float) and u.dtype != torch.float32
    if out_f32:
        out = torch.empty(delta.shape, dtype=torch.float32, device=delta.device)
    else:
        out = torch.empty_like(delta)
        if out.stride(-1) != 1:
            out = torch.empty(delta.shape, dtype=delta.dtype, device=delta.device)
    ck = ckpt_interval()
    ckpt = torch.empty((b, d, (l + ck - 1) // ck, n), dtype=torch.float32, device=u.device) if need_ckpt else None
    a = _lib.ScanFwdArgs(
        u=_ptr(u), delta=_ptr(delta), A=_ptr(A), Bm=_ptr(B), Cm=_ptr(C_), D=_ptr(D), delta_bias=_ptr(delta_bias), out=_ptr(out),
        ckpt=_ptr(ckpt), batch=b, dim=d, seqlen=l, dstate=n, ngroups=g,
        u_bs=u.stride(0), u_ds=u.stride(1), delta_bs=delta.stride(0), delta_ds=delta.stride(1), out_bs=out.stride(0), out_ds=out.stride(1),
        B_bs=B.stride(0), B_gs=B.stride(1), B_ns=B.stride(2), C_bs=C_.stride(0), C_gs=C_.stride(1), C_ns=C_.stride(2),
        delta_softplus=int(bool(delta_softplus)), dtype=_DT[u.dtype], out_f32=int(out_f32))
    es = u.element_size()
    nbytes = es * (2 * b * d * l + 2 * b * g * n * l) + out.element_size() * b * d * l + 4 * (d * n + 2 * d)  # SURVEY.md 8(d): every operand once
    _run("vmb_selective_scan_fwd", u, "scan_fwd", a, nbytes=nbytes)
    return out, ckpt


def selective_scan_bwd(u, delta, A, B, C_, D, delta_bias, dout, ckpt, delta_softplus=False, zeroed=None, dout_float=False,
                       deterministic=None, workspace=None):
    """-> (du, ddelta, dA, dB, dC, dD, ddelta_bias); dB/dC returned in B/C dtype (reference cpp:347).
    dout has u's dtype (cus/selective_scan.cpp:259).  dout_float=True also accepts an fp32 dout against bf16 / fp16 u (the gradient
    of an out_float forward; the reference's selective_scan_cuda_oflex.bwd, cusoflex/selective_scan_oflex.cpp:257-260,349-355):
    du, ddelta, dB, dC keep u's dtype.
    zeroed: optional (dA, dD, dbias) pre-zeroed fp32 buffers (the training path hands out slices of one zeroed workspace).
    deterministic: None follows torch.are_deterministic_algorithms_enabled().  True runs the bitwise-reproducible kernels: every CTA
    stores its partial sums in its own workspace slot and a second kernel sums them in a fixed order, then ADDS one sum to each
    element of dA / dD / dbias (timing tag "scan_bwd_det").  False: fp32 atomics (tag "scan_bwd").
    workspace: optional uint8 CUDA tensor used as the library's scratch (its contents are irrelevant); else one is allocated."""
    b, d, l, n, g = _check_common(u, delta, A, B, C_, D, delta_bias, "selective_scan_bwd")
    det = _deterministic(deterministic)
    dout_f32 = bool(dout_float) and dout.dtype == torch.float32 and u.dtype != torch.float32
    if (dout.dtype != u.dtype and not dout_f32) or tuple(dout.shape) != (b, d, l) or (dout.stride(-1) != 1 and dout.size(-1) != 1):
        raise RuntimeError("selective_scan_bwd: dout must match u in dtype (or be float32) and shape, with stride(-1)==1")
    L = _lib.lib()
    du = torch.empty((b, d, l), dtype=u.dtype, device=u.device)
    ddelta = torch.empty((b, d, l), dtype=u.dtype, device=u.device)
    dA = torch.zeros_like(A) if zeroed is None else zeroed[0]
    dB = torch.empty((b, g, n, l), dtype=u.dtype, device=u.device)
    dC = torch.empty((b, g, n, l), dtype=u.dtype, device=u.device)
    dD = (torch.zeros_like(D) if zeroed is None else zeroed[1]) if D is not None else None
    dbias = (torch.zeros_like(delta_bias) if zeroed is None else zeroed[2]) if delta_bias is not None else None
    a = _lib.ScanBwdArgs(
        u=_ptr(u), delta=_ptr(delta), A=_ptr(A), Bm=_ptr(B), Cm=_ptr(C_), D=_ptr(D), delta_bias=_ptr(delta_bias), dout=_ptr(dout),
        ckpt=_ptr(ckpt), du=_ptr(du), ddelta=_ptr(ddelta), dA=_ptr(dA), dB=_ptr(dB), dC=_ptr(dC), dD=_ptr(dD), ddelta_bias=_ptr(dbias),
        batch=b, dim=d, seqlen=l, dstate=n, ngroups=g,
        u_bs=u.stride(0), u_ds=u.stride(1), delta_bs=delta.stride(0), delta_ds=delta.stride(1), dout_bs=dout.stride(0),
        dout_ds=dout.stride(1), du_bs=du.stride(0), du_ds=du.stride(1), ddelta_bs=ddelta.stride(0), ddelta_ds=ddelta.stride(1),
        B_bs=B.stride(0), B_gs=B.stride(1), B_ns=B.stride(2), C_bs=C_.stride(0), C_gs=C_.stride(1), C_ns=C_.stride(2),
        delta_softplus=int(bool(delta_softplus)), dtype=_DT[u.dtype], dout_f32=int(dout_f32), deterministic=int(det))
    with torch.cuda.device(u.device):
        nws = L.vmb_scan_bwd_det_workspace_bytes(C.byref(a)) if det else L.vmb_scan_bwd_workspace_bytes(b, g, n, l)
    ws = _workspace(nws, workspace, u.device, "selective_scan_bwd")
    a.workspace = ws.data_ptr()
    es = u.element_size()
    nbytes = es * (4 * b * d * l + 4 * b * g * n * l) + dout.element_size() * b * d * l + 4 * b * d * ((l + 63) // 64) * n
    _run("vmb_selective_scan_bwd", u, "scan_bwd_det" if det else "scan_bwd", a, nbytes=nbytes, kernels=2)
    return du, ddelta, dA, dB, dC, dD, dbias


def _check_io(t, like, name, who):
    if t.dtype != like.dtype or tuple(t.shape) != tuple(like.shape) or not t.is_cuda or (t.stride(-1) != 1 and t.size(-1) != 1):
        raise RuntimeError(f"{who}: {name} must be a CUDA tensor of shape {tuple(like.shape)} and dtype {like.dtype} with stride(-1)==1")


def selective_scan_fwd_z(u, delta, A, B, C_, D=None, z=None, delta_bias=None, delta_softplus=False, need_ckpt=True):
    """The forward of mamba_ssm's selective_scan_cuda.fwd -> (out, x, out_z).
    out: the ungated result, delta's dtype.  out_z = out * SiLU(z) from the fp32 accumulator, rounded once (None without z): the
    same launch writes both.  x: fp32 (B, D, ceil(L/64), 2N) pair-layout checkpoints, x[:, :, -1, 1::2] the state after the last
    position (None when need_ckpt is False).  The gradient path is selective_scan_bwd on x[..., 1::2] (after scan_gate_bwd with z)."""
    b, d, l, n, g = _check_common(u, delta, A, B, C_, D, delta_bias, "selective_scan_fwd")
    if z is not None:
        _check_io(z, u, "z", "selective_scan_fwd")
    out = torch.empty((b, d, l), dtype=u.dtype, device=u.device)
    out_z = torch.empty_like(out) if z is not None else None
    ck = ckpt_interval()
    x = torch.empty((b, d, (l + ck - 1) // ck, 2 * n), dtype=torch.float32, device=u.device) if need_ckpt else None
    a = _lib.ScanFwdArgs(
        u=_ptr(u), delta=_ptr(delta), A=_ptr(A), Bm=_ptr(B), Cm=_ptr(C_), D=_ptr(D), delta_bias=_ptr(delta_bias), out=_ptr(out),
        ckpt=_ptr(x), batch=b, dim=d, seqlen=l, dstate=n, ngroups=g,
        u_bs=u.stride(0), u_ds=u.stride(1), delta_bs=delta.stride(0), delta_ds=delta.stride(1), out_bs=out.stride(0), out_ds=out.stride(1),
        B_bs=B.stride(0), B_gs=B.stride(1), B_ns=B.stride(2), C_bs=C_.stride(0), C_gs=C_.stride(1), C_ns=C_.stride(2),
        delta_softplus=int(bool(delta_softplus)), dtype=_DT[u.dtype], out_f32=0,
        z=_ptr(z), out_z=_ptr(out_z), z_bs=z.stride(0) if z is not None else 0, z_ds=z.stride(1) if z is not None else 0,
        out_z_bs=out_z.stride(0) if z is not None else 0, out_z_ds=out_z.stride(1) if z is not None else 0,
        ckpt_pairs=int(need_ckpt))
    es = u.element_size()
    nbytes = es * ((2 + (3 if z is not None else 1)) * b * d * l + 2 * b * g * n * l) + 4 * (d * n + 2 * d)
    _run("vmb_selective_scan_fwd", u, "scan_fwd_z" if z is not None else "scan_fwd", a, nbytes=nbytes)
    return out, x, out_z


def scan_gate_bwd(dout, out, z, dz=None, recompute_out_z=False):
    """Backward of out_z = out * SiLU(z) (the gate of selective_scan_fwd_z), one launch -> (dout_eff, dz, out_z).
    dout_eff = dout * SiLU(z), fp32: the gradient w.r.t. the ungated out, for selective_scan_bwd(..., dout_float=True).
    dz = dout * out * s * (1 + z (1 - s)), s = sigmoid(z), in z's dtype, written into `dz` when given (any view with stride(-1)==1).
    out_z: out * SiLU(z) when recompute_out_z, else None."""
    who = "scan_gate_bwd"
    _check_io(z, z, "z", who)
    _check_io(dout, z, "dout", who)
    _check_io(out, z, "out", who)
    b, d, l = z.shape
    if dz is None:
        dz = torch.empty((b, d, l), dtype=z.dtype, device=z.device)
    else:
        _check_io(dz, z, "dz", who)
    dout_eff = torch.empty((b, d, l), dtype=torch.float32, device=z.device)
    out_z = torch.empty((b, d, l), dtype=z.dtype, device=z.device) if recompute_out_z else None
    a = _lib.ScanGateArgs(
        dout=_ptr(dout), out=_ptr(out), z=_ptr(z), dout_eff=_ptr(dout_eff), dz=_ptr(dz), out_z=_ptr(out_z), batch=b, dim=d, seqlen=l,
        dout_bs=dout.stride(0), dout_ds=dout.stride(1), out_bs=out.stride(0), out_ds=out.stride(1), z_bs=z.stride(0), z_ds=z.stride(1),
        dz_bs=dz.stride(0), dz_ds=dz.stride(1), out_z_bs=out_z.stride(0) if recompute_out_z else 0,
        out_z_ds=out_z.stride(1) if recompute_out_z else 0, dtype=_DT[z.dtype])
    es = z.element_size()
    _run("vmb_scan_gate_bwd", z, "scan_gate_bwd", a, nbytes=(es * (4 + int(bool(recompute_out_z))) + 4) * b * d * l)
    return dout_eff, dz, out_z


# ----------------------------------------------------------------------------- fused OSS-block stages
def pixlin(x, w, bias=None, residual=None, ln=None, gate=None, gate_mode=0, act=(0, 0), out_dtype=None, out=None):
    """out[b,m,p] = epi(sum_k w[m,k] pro(x)[b,k,p]).  x: (B,K,P) view with stride(-1)==1; w: (M,>=K) x.dtype, rows may be
    zero-padded to a multiple of 16 (pad_weight) for vector loads.
    ln = (mode, weight_fp32, bias_fp32|None); gate: (B,K) fp32; residual: (B,M,P) view."""
    B, K, P = x.shape
    M = w.shape[0]
    assert w.shape[1] >= K and w.dtype == x.dtype and w.stride(1) == 1 and x.stride(2) == 1
    out_dtype = out_dtype or x.dtype
    if out is None:
        out = torch.empty((B, M, P), dtype=out_dtype, device=x.device)
    ln_mode, ln_w, ln_b = ln if ln is not None else (0, None, None)
    a = _lib.PixlinArgs(
        x=_ptr(x), w=_ptr(w), bias=_ptr(bias), residual=_ptr(residual), out=_ptr(out), ln_w=_ptr(ln_w), ln_b=_ptr(ln_b),
        gate=_ptr(gate), ln_mode=ln_mode, gate_mode=gate_mode if gate is not None else 0, act_from=act[0], act_to=act[1],
        batch=B, K=K, M=M, P=P, x_bs=x.stride(0), x_cs=x.stride(1), r_bs=residual.stride(0) if residual is not None else 0,
        r_cs=residual.stride(1) if residual is not None else 0, o_bs=out.stride(0), o_cs=out.stride(1),
        g_bs=gate.stride(0) if gate is not None else 0, w_ld=w.stride(0), dtype=_DT[x.dtype], out_dtype=_DT[out_dtype])
    _run("vmb_pixlin", x, "pixlin", a)
    return out


def pad_weight(w: torch.Tensor) -> torch.Tensor:
    """(M,K) -> (M, ceil16(K)) zero-padded copy: rows 16 B aligned for the vectorised weight staging."""
    M, K = w.shape
    kp = (K + 15) // 16 * 16
    if kp == K:
        return w.contiguous()
    out = torch.zeros((M, kp), dtype=w.dtype, device=w.device)
    out[:, :K] = w
    return out


def dwconv3x3(x, w9, bias, c_out, H, W, mode, out=None):
    """x: (B, Cin, H*W) view; mode 0: SiLU(dw(x[:c_out])); mode 1: gelu(dw(x[:c_out])) * dw(x[c_out:2c_out]);
    mode 2: dw(x[:c_out]) (no activation: the transposed conv of the backward pass, called with flipped taps)."""
    B = x.shape[0]
    if out is None:
        out = torch.empty((B, c_out, H * W), dtype=x.dtype, device=x.device)
    _run("vmb_dwconv3x3", x, "dwconv", _dwconv_args(x, w9, bias, out, c_out, H, W, mode))
    return out


def _dwconv_args(x, w9, bias, out, c_out, H, W, mode):
    return _lib.DwconvArgs(x=_ptr(x), w=_ptr(w9), bias=_ptr(bias), out=_ptr(out), batch=x.shape[0], c_out=c_out, H=H, W=W, mode=mode,
                           x_bs=x.stride(0), x_cs=x.stride(1), o_bs=out.stride(0), o_cs=out.stride(1), dtype=_DT[x.dtype])


def dwconv3x3_t(x, w9, bias, c_out, H, W):
    """SiLU(dw(x[:c_out])) and its (W,H)-transposed copy from ONE launch -> (out (B,c_out,H*W), out_t (B,c_out,W*H))."""
    B = x.shape[0]
    out = torch.empty((B, c_out, H * W), dtype=x.dtype, device=x.device)
    out_t = torch.empty_like(out)
    _run("vmb_dwconv3x3_t", x, "dwconv", _dwconv_args(x, w9, bias, out, c_out, H, W, 0), _ptr(out_t))
    return out, out_t


def cross_scan(srcs, rows, H, W, out=None):
    """srcs: 4 views (B, rows, L) sharing strides -> (B, 4, rows, L) in scan order.  `out`: optional (B, 4, rows, L) view
    (e.g. a channel slice of a wider tensor) with contiguous rows.  The inverse orders are the same call with H and W swapped."""
    s0 = srcs[0]
    B = s0.shape[0]
    if out is None:
        out = torch.empty((B, 4, rows, H * W), dtype=s0.dtype, device=s0.device)
    assert out.shape == (B, 4, rows, H * W) and out.stride(3) == 1 and out.stride(2) == H * W and out.dtype == s0.dtype
    for t in srcs:
        assert t.stride() == s0.stride() and t.stride(2) == 1
    _run("vmb_cross_scan", s0, "cross_scan", _cross_scan_args(srcs, out, rows, H, W))
    return out


def _cross_scan_args(srcs, out, rows, H, W):
    s0 = srcs[0]
    return _lib.CrossScanArgs(src=_ptr4(srcs), out=_ptr(out), batch=s0.shape[0], rows=rows, H=H, W=W, src_bs=s0.stride(0),
                              src_rs=s0.stride(1), out_bs=out.stride(0), dtype=_DT[s0.dtype], out_ks=out.stride(1))


def pixel_shuffle2_nhwc(x, bias=None):
    """nn.PixelShuffle(2) on a channels-last tensor: x logical (B,4C,H,W) with NHWC storage -> (B,C,2H,2W), NHWC storage.
    Bit-identical to F.pixel_shuffle(x, 2).  bias: optional fp32 (4C), added to x first (the bias of the conv that produced x)."""
    B, C4, H, W = x.shape
    assert C4 % 4 == 0 and x.is_contiguous(memory_format=torch.channels_last)
    out = torch.empty((B, C4 // 4, 2 * H, 2 * W), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    a = _lib.PixelShuffleArgs(x=_ptr(x), out=_ptr(out), batch=B, H=H, W=W, C=C4 // 4, dtype=_DT[x.dtype])
    if bias is None:
        _run("vmb_pixel_shuffle2_nhwc", x, "pixel_shuffle", a)
    else:
        assert bias.dtype == torch.float32 and bias.numel() == C4 and bias.is_contiguous() and bias.device == x.device
        _run("vmb_pixel_shuffle2_nhwc_bias", x, "pixel_shuffle", a, _ptr(bias))
    return out


def cross_scan_multi(segs, H, W):
    """segs: up to 4 tuples (srcs, rows, out|None) as for cross_scan, all of one geometry -> list of outputs, ONE launch."""
    assert 1 <= len(segs) <= 4
    arr = (_lib.CrossScanArgs * len(segs))()
    outs = []
    s00 = segs[0][0][0]
    B = s00.shape[0]
    for i, (srcs, rows, out) in enumerate(segs):
        s0 = srcs[0]
        if out is None:
            out = torch.empty((B, 4, rows, H * W), dtype=s0.dtype, device=s0.device)
        assert out.shape == (B, 4, rows, H * W) and out.stride(3) == 1 and out.stride(2) == H * W and out.dtype == s00.dtype
        for t in srcs:
            assert t.stride() == s0.stride() and t.stride(2) == 1 and t.dtype == s00.dtype and t.shape[0] == B
        arr[i] = _cross_scan_args(srcs, out, rows, H, W)
        outs.append(out)
    _run("vmb_cross_scan_multi", s00, "cross_scan", arr, len(segs))
    return outs


CONV_PLAIN, CONV_UNSHUFFLE2, CONV_SHUFFLE2, CONV_ADD_NEAREST = 0, 1, 2, 3


def pack_conv3x3_weight(w: torch.Tensor, dtype) -> torch.Tensor:
    """nn.Conv2d weight (Cout, Cin, 3, 3) -> the kernel layout [tap = 3 ky + kx][Cout rounded up to 64][Cin rounded up to 16], zero
    padded, in the I/O dtype (include/vmambair_b200.h, vmb_conv3x3)."""
    Cout, Cin = w.shape[0], w.shape[1]
    assert w.shape[2:] == (3, 3)
    out = torch.zeros((9, (Cout + 63) // 64 * 64, (Cin + 15) // 16 * 16), dtype=dtype, device=w.device)
    out[:, :Cout, :Cin] = w.detach().permute(2, 3, 0, 1).reshape(9, Cout, Cin).to(dtype)
    return out


def conv3x3(x, wp, bias, c_out, mode=CONV_PLAIN, out=None, add=None, add_scale=1, nhwc=False):
    """Dense 3x3 conv (stride 1, pad 1) with the PixelUnshuffle(2) / PixelShuffle(2) / channel-slice / "+ nearest-upsampled image"
    store folded in.  x: (B, Cin, H, W), NCHW view with dense planes (any batch / channel stride) or, nhwc=True, channels_last
    contiguous.  wp: pack_conv3x3_weight(...).  bias: fp32 (c_out) or None.  out: optional NCHW destination with dense planes (e.g.
    a channel slice of the decoder's concatenation buffer).  add (mode CONV_ADD_NEAREST): (B, c_out, H/s, W/s), x.dtype."""
    B, Cin, H, W = x.shape
    if nhwc:
        assert x.is_contiguous(memory_format=torch.channels_last)
        x_bs, x_cs = H * W * Cin, 1
    else:
        assert x.stride(3) == 1 and x.stride(2) == W, "conv3x3: NCHW input planes must be dense"
        x_bs, x_cs = x.stride(0), x.stride(1)
    assert wp.dtype == x.dtype and wp.is_contiguous() and wp.shape == (9, (c_out + 63) // 64 * 64, (Cin + 15) // 16 * 16)
    shape = {CONV_PLAIN: (B, c_out, H, W), CONV_UNSHUFFLE2: (B, 4 * c_out, H // 2, W // 2),
             CONV_SHUFFLE2: (B, c_out // 4, 2 * H, 2 * W), CONV_ADD_NEAREST: (B, c_out, H, W)}[mode]
    if out is None:
        out = torch.empty(shape, dtype=x.dtype, device=x.device)
    assert tuple(out.shape) == shape and out.dtype == x.dtype and out.stride(3) == 1 and out.stride(2) == shape[3]
    add_bs = add_cs = 0
    if mode == CONV_ADD_NEAREST:
        assert add is not None and add.dtype == x.dtype and add.shape == (B, c_out, H // add_scale, W // add_scale)
        add = add.contiguous()
        add_bs, add_cs = add.stride(0), add.stride(1)
    a = _lib.Conv3x3Args(x=_ptr(x), w=_ptr(wp), bias=_ptr(bias), out=_ptr(out), add=_ptr(add) if mode == CONV_ADD_NEAREST else None,
                         batch=B, Cin=Cin, Cout=c_out, H=H, W=W, in_nhwc=int(nhwc), mode=mode, add_scale=add_scale, x_bs=x_bs, x_cs=x_cs,
                         o_bs=out.stride(0), o_cs=out.stride(1), add_bs=add_bs, add_cs=add_cs, dtype=_DT[x.dtype])
    _run("vmb_conv3x3", x, "conv3x3", a)
    return out


def transpose_hw(x, H, W):
    """x: (B, C, H*W) contiguous -> (B, C, W*H) with every plane transposed."""
    assert x.is_contiguous()
    out = torch.empty_like(x)
    a = _lib.TransposeArgs(x=_ptr(x), out=_ptr(out), planes=x.shape[0] * x.shape[1], H=H, W=W, dtype=_DT[x.dtype])
    _run("vmb_transpose_hw", x, "transpose", a)
    return out


def selective_scan_fwd_grouped(us, deltas, Bs, Cs, revs, A, D, delta_bias, delta_softplus=True, need_ckpt=False):
    """Direction-aware forward: group g reads us[g] (B,R,L), deltas[g] (B,R,L), Bs[g]/Cs[g] (B,N,L) (views sharing
    strides) and walks them backwards when revs[g]; returns (B, G, R, L) with group g written in ITS SOURCE's memory order.
    need_ckpt: -> (out, ckpt) with the fp32 checkpoints (B, G*R, n_ckpt, N) that selective_scan_bwd_grouped consumes."""
    G = len(us)
    b, R, L = us[0].shape
    N = A.shape[1]
    for lst in (us, deltas, Bs, Cs):
        for t in lst:
            assert t.stride() == lst[0].stride() and t.stride(2) == 1 and t.dtype == us[0].dtype
    out = torch.empty((b, G, R, L), dtype=us[0].dtype, device=us[0].device)
    ck = ckpt_interval()
    ckpt = torch.empty((b, G * R, (L + ck - 1) // ck, N), dtype=torch.float32, device=us[0].device) if need_ckpt else None
    a = _lib.ScanGroupedArgs(
        u=_ptr4(us), delta=_ptr4(deltas), Bm=_ptr4(Bs), Cm=_ptr4(Cs), out=_ptr4([out[:, g] for g in range(G)]), rev=_rev4(revs),
        A=_ptr(A), D=_ptr(D), delta_bias=_ptr(delta_bias), batch=b, dim=G * R, seqlen=L, dstate=N, ngroups=G,
        u_bs=us[0].stride(0), u_ds=us[0].stride(1), delta_bs=deltas[0].stride(0), delta_ds=deltas[0].stride(1),
        out_bs=out.stride(0), out_ds=out.stride(2), B_bs=Bs[0].stride(0), B_ns=Bs[0].stride(1), C_bs=Cs[0].stride(0),
        C_ns=Cs[0].stride(1), delta_softplus=int(bool(delta_softplus)), dtype=_DT[us[0].dtype], ckpt=_ptr(ckpt))
    es = us[0].element_size()
    n_u = len({t.data_ptr() for t in us})  # forward and reversed directions share one source tensor: counted once
    nbytes = es * b * L * (n_u * R + G * R + G * R + 2 * G * N) + 4 * (G * R * N + 2 * G * R)  # every unique operand / result once
    if ckpt is not None:
        nbytes += 4 * ckpt.numel()
    _run("vmb_selective_scan_fwd_grouped", us[0], "scan_fwd", a, nbytes=nbytes)
    return (out, ckpt) if need_ckpt else out


def selective_scan_bwd_grouped(us, deltas, Bs, Cs, douts, revs, A, D, delta_bias, ckpt, delta_softplus=True, zeroed=None, out=None,
                               deterministic=None, workspace=None):
    """Backward of selective_scan_fwd_grouped (checkpoints from its need_ckpt=True call): douts[g] (B,R,L) is the gradient of group
    g's output in that group's memory order.  -> (dus, ddeltas, dA, dBs, dCs, dD, ddelta_bias): dus / ddeltas lists of (B,R,L), dBs / dCs
    lists of (B,N,L), every one in the memory order of group g's sources; dA (G*R,N), dD, ddelta_bias (G*R) fp32.
    zeroed: optional (dA, dD, dbias) pre-zeroed fp32 accumulators.  out: optional (dus, ddeltas, dBs, dCs) destination views (each list
    sharing strides, rows contiguous), e.g. slices of the buffers the next kernels read.
    deterministic / workspace: as in selective_scan_bwd."""
    det = _deterministic(deterministic)
    G = len(us)
    b, R, L = us[0].shape
    N = A.shape[1]
    dev, dt = us[0].device, us[0].dtype
    for lst in (us, deltas, Bs, Cs, douts):
        for t in lst:
            assert t.stride() == lst[0].stride() and t.stride(2) == 1 and t.dtype == dt and t.is_cuda
    if out is None:
        du = torch.empty((b, G, R, L), dtype=dt, device=dev)
        ddelta = torch.empty((b, G, R, L), dtype=dt, device=dev)
        dBm = torch.empty((b, G, N, L), dtype=dt, device=dev)
        dCm = torch.empty((b, G, N, L), dtype=dt, device=dev)
        out = ([du[:, g] for g in range(G)], [ddelta[:, g] for g in range(G)], [dBm[:, g] for g in range(G)], [dCm[:, g] for g in range(G)])
    dus, dds, dBs, dCs = out
    for lst in out:
        for t in lst:
            assert t.stride() == lst[0].stride() and t.stride(2) == 1 and t.dtype == dt
    Lb = _lib.lib()
    dA = torch.zeros_like(A) if zeroed is None else zeroed[0]
    dD = (torch.zeros_like(D) if zeroed is None else zeroed[1]) if D is not None else None
    dbias = (torch.zeros_like(delta_bias) if zeroed is None else zeroed[2]) if delta_bias is not None else None
    a = _lib.ScanGroupedBwdArgs(
        u=_ptr4(us), delta=_ptr4(deltas), Bm=_ptr4(Bs), Cm=_ptr4(Cs), dout=_ptr4(douts), du=_ptr4(dus), ddelta=_ptr4(dds),
        dB=_ptr4(dBs), dC=_ptr4(dCs), rev=_rev4(revs), A=_ptr(A), D=_ptr(D), delta_bias=_ptr(delta_bias), ckpt=_ptr(ckpt),
        dA=_ptr(dA), dD=_ptr(dD), ddelta_bias=_ptr(dbias), batch=b, dim=G * R, seqlen=L, dstate=N, ngroups=G,
        u_bs=us[0].stride(0), u_ds=us[0].stride(1), delta_bs=deltas[0].stride(0), delta_ds=deltas[0].stride(1),
        dout_bs=douts[0].stride(0), dout_ds=douts[0].stride(1), du_bs=dus[0].stride(0), du_ds=dus[0].stride(1),
        ddelta_bs=dds[0].stride(0), ddelta_ds=dds[0].stride(1), B_bs=Bs[0].stride(0), B_ns=Bs[0].stride(1),
        C_bs=Cs[0].stride(0), C_ns=Cs[0].stride(1), dB_bs=dBs[0].stride(0), dB_ns=dBs[0].stride(1), dC_bs=dCs[0].stride(0),
        dC_ns=dCs[0].stride(1), delta_softplus=int(bool(delta_softplus)), dtype=_DT[dt], deterministic=int(det))
    with torch.cuda.device(dev):
        nws = Lb.vmb_scan_grouped_bwd_det_workspace_bytes(C.byref(a)) if det else Lb.vmb_scan_bwd_workspace_bytes(b, G, N, L)
    ws = _workspace(nws, workspace, dev, "selective_scan_bwd_grouped")
    a.workspace = ws.data_ptr()
    es = us[0].element_size()
    uniq = lambda lst: len({t.data_ptr() for t in lst})  # directions that share a source tensor read it once
    nbytes = es * b * L * (R * (uniq(us) + G + uniq(douts) + 2 * G) + 4 * G * N) + (4 * ckpt.numel() if ckpt is not None else 0)
    _run("vmb_selective_scan_bwd_grouped", us[0], "scan_bwd_det" if det else "scan_bwd", a, nbytes=nbytes, kernels=2)
    return dus, dds, dA, dBs, dCs, dD, dbias


_CSC_SMEM_LIMIT = 227 * 1024


def cross_scan_c_supported(D, L, R, N) -> bool:
    """True when vmb_cross_selective_scan_c_fwd / _bwd take (D, L, R, N) on one CTA per image: d_state <= 16, D <= 16 and the
    backward's shared memory within 227 KB (the library's own check)."""
    s = _lib.lib().vmb_cross_selective_scan_c_smem_bytes(int(D), int(L), int(R), int(N))
    return 0 < s <= _CSC_SMEM_LIMIT


def _csc_args(x, xw, xb, dtw, dtb, A_logs, Ds, y, delta_softplus):
    b, D, L = x.shape
    K, RN, D2 = xw.shape
    N = A_logs.shape[1]
    R = RN - 2 * N
    if x.dtype not in _DT or not x.is_cuda or x.stride(2) != 1:
        raise RuntimeError("cross_selective_scan_c: x must be a float32/bfloat16/float16 CUDA tensor (B, D, L) with stride(-1) == 1")
    for n, t, shp in (("x_proj_weight", xw, (2, RN, D)), ("x_proj_bias", xb, (2, RN)), ("dt_projs_weight", dtw, (2, D, R)),
                      ("dt_projs_bias", dtb, (2 * D,)), ("A_logs", A_logs, (2 * D, N)), ("Ds", Ds, (2 * D,))):
        if t is None and n == "x_proj_bias":
            continue
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != x.device or tuple(t.shape) != shp:
            raise RuntimeError(f"cross_selective_scan_c: {n} must be a contiguous float32 tensor of shape {shp} on x's device")
    return _lib.CrossScanCArgs(x=_ptr(x), x_proj_weight=_ptr(xw), x_proj_bias=_ptr(xb), dt_projs_weight=_ptr(dtw),
                               dt_projs_bias=_ptr(dtb), A_logs=_ptr(A_logs), Ds=_ptr(Ds), y=_ptr(y), batch=b, D=D, L=L, R=R, N=N,
                               x_bs=x.stride(0), x_ds=x.stride(1), delta_softplus=int(bool(delta_softplus)), dtype=_DT[x.dtype])


def cross_selective_scan_c_fwd(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, delta_softplus=True):
    """Two-direction channel scan, one launch: x (B, D, L) any of the three dtypes; parameters fp32 contiguous, x_proj_weight (2, R+2N, D),
    x_proj_bias (2, R+2N) or None, dt_projs_weight (2, D, R), dt_projs_bias (2D), A_logs (2D, N), Ds (2D).
    -> y fp32 (B, L, D) = y_0 + flip(y_1) (include/vmambair_b200.h, vmb_cross_selective_scan_c_fwd)."""
    b, D, L = x.shape
    y = torch.empty((b, L, D), dtype=torch.float32, device=x.device)
    a = _csc_args(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, y, delta_softplus)
    _run("vmb_cross_selective_scan_c_fwd", x, "cscan_c_fwd", a)
    return y


def cross_selective_scan_c_bwd(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, dy, delta_softplus=True):
    """Backward of cross_selective_scan_c_fwd (two launches: the per-image kernel and the fixed-order batch sum).  dy: fp32 (B, L, D).
    -> (dx (B, D, L) in x's dtype, {name: fp32 gradient shaped like the parameter}); "x_proj_bias" only when the bias is given."""
    b, D, L = x.shape
    K, RN, _ = x_proj_weight.shape
    N = A_logs.shape[1]
    R = RN - 2 * N
    if dy.dtype != torch.float32 or tuple(dy.shape) != (b, L, D) or not dy.is_contiguous() or dy.device != x.device:
        raise RuntimeError(f"cross_selective_scan_c_bwd: dy must be a contiguous float32 tensor of shape {(b, L, D)}")
    dx = torch.empty((b, D, L), dtype=x.dtype, device=x.device)
    sizes = [("x_proj_weight", (2, RN, D)), ("x_proj_bias", (2, RN)), ("dt_projs_weight", (2, D, R)), ("dt_projs_bias", (2 * D,)),
             ("A_logs", (2 * D, N)), ("Ds", (2 * D,))]
    flat = torch.empty(sum(math.prod(s) for _, s in sizes), dtype=torch.float32, device=x.device)
    ws = torch.empty(_lib.lib().vmb_cross_selective_scan_c_workspace_bytes(b, D, R, N) // 4, dtype=torch.float32, device=x.device)
    a = _lib.CrossScanCBwdArgs(
        fwd=_csc_args(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, None, delta_softplus),
        dy=_ptr(dy), dx=_ptr(dx), d_params=_ptr(flat), workspace=_ptr(ws))
    _run("vmb_cross_selective_scan_c_bwd", x, "cscan_c_bwd", a, kernels=2)
    grads, o = {}, 0
    for n, s in sizes:
        k = math.prod(s)
        if n != "x_proj_bias" or x_proj_bias is not None:
            grads[n] = flat[o:o + k].view(s)
        o += k
    return dx, grads


def merge_sum(ys, C_, H, W, in_place_order=False, out=None):
    """ys: (B,4,C,L) contiguous, four scan directions -> fp32 (B,C,L): (y0 + y2') + T y1' + T y3' in pixel order, where ' is the
    inverse order of the direction (in_place_order: ys[0], ys[2] hold natural (H,W) pixel order and ys[1], ys[3] the transposed (W,H)
    order, as the grouped scan writes them; else every ys[k] is in scan order, k = 2, 3 reversed).  out: optional fp32 (B,C,L) dense."""
    B = ys.shape[0]
    assert ys.is_contiguous() and ys.shape == (B, 4, C_, H * W)
    if out is None:
        out = torch.empty((B, C_, H * W), dtype=torch.float32, device=ys.device)
    assert out.dtype == torch.float32 and out.is_contiguous()
    ws = torch.empty(_lib.lib().vmb_merge_workspace_bytes(B, C_, H, W), dtype=torch.uint8, device=ys.device)
    a = _lib.MergeArgs(ys=_ptr(ys), batch=B, C=C_, H=H, W=W, dtype=_DT[ys.dtype], workspace=_ptr(ws), in_place_order=int(in_place_order))
    _run("vmb_merge_sum", ys, "merge", a, _ptr(out), nbytes=ys.element_size() * ys.numel() + 4 * out.numel())
    return out


def merge_norm_gate(ys, z, ln_w, ln_b, C_, H, W, in_place_order=False, z_preact=False, return_ws=False):
    """ys: (B,4,C,L) contiguous; z: (B,C,L) view -> (y2 (B,C,L), pooled sums (B,C) fp32 [, workspace]).
    z_preact: z holds the pre-activation (SiLU applied here); return_ws: also return the fp32 workspace (merged scan output
    (B,C,L) followed by the per-pixel (sum, sum of squares)) that vmb_merge_norm_gate_bwd consumes."""
    B = ys.shape[0]
    assert ys.is_contiguous() and z.stride(2) == 1
    y2 = torch.empty((B, C_, H * W), dtype=ys.dtype, device=ys.device)
    pooled = torch.empty((B, C_), dtype=torch.float32, device=ys.device)
    ws = torch.empty(_lib.lib().vmb_merge_workspace_bytes(B, C_, H, W), dtype=torch.uint8, device=ys.device)
    a = _lib.MergeArgs(ys=_ptr(ys), z=_ptr(z), ln_w=_ptr(ln_w), ln_b=_ptr(ln_b), y2=_ptr(y2), pooled=_ptr(pooled), batch=B, C=C_, H=H,
                       W=W, z_bs=z.stride(0), z_cs=z.stride(1), dtype=_DT[ys.dtype], workspace=_ptr(ws),
                       in_place_order=int(in_place_order), z_preact=int(z_preact), save_ws=int(return_ws))
    _run("vmb_merge_norm_gate", ys, "merge", a, kernels=2)
    return (y2, pooled, ws) if return_ws else (y2, pooled)


def _channel_args(pooled, inv_count, prm, C_, c_out):
    return _lib.ChannelArgs(pooled=_ptr(pooled), inv_count=inv_count, cin_w=_ptr(prm["cin_w"]), cin_b=_ptr(prm["cin_b"]),
                            xc_proj=_ptr(prm["xc_proj"]), dtc_w=_ptr(prm["dtc_w"]), dtc_b=_ptr(prm["dtc_b"]), Ac_logs=_ptr(prm["Ac_logs"]),
                            Dsc=_ptr(prm["Dsc"]), cout_w=_ptr(prm["cout_w"]), cout_b=_ptr(prm["cout_b"]), cn_w=_ptr(prm["cn_w"]),
                            cn_b=_ptr(prm["cn_b"]), c_out=_ptr(c_out), batch=pooled.shape[0], C=C_, dc=prm["dc"], Rc=prm["Rc"], N=prm["N"])


def channel_branch(pooled, inv_count, prm, C_):
    B = pooled.shape[0]
    c = torch.empty((B, C_), dtype=torch.float32, device=pooled.device)
    _run("vmb_channel_branch", pooled, "channel", _channel_args(pooled, inv_count, prm, C_, c))
    return c


# ----------------------------------------------------------------------------- training path: backward stages
def layernorm_fwd(x, mode, w, b):
    """x: (B,C,L) view -> LayerNorm over C per pixel, materialised (B,C,L) contiguous (mode 1 WithBias / 2 BiasFree)."""
    B, C_, L = x.shape
    assert x.stride(2) == 1
    y = torch.empty((B, C_, L), dtype=x.dtype, device=x.device)
    a = _lib.LnFwdArgs(x=_ptr(x), w=_ptr(w), b=_ptr(b), y=_ptr(y), batch=B, C=C_, L=L, mode=mode, x_bs=x.stride(0), x_cs=x.stride(1),
                       y_bs=y.stride(0), y_cs=y.stride(1), dtype=_DT[x.dtype])
    _run("vmb_layernorm_fwd", x, "ln_fwd", a)
    return y


def layernorm_bwd(x, g, mode, w, add=None, need_param_grads=True, zeroed=None, phase="both", stats=None):
    """-> (dx (B,C,L), dw (C) fp32, db (C) fp32 | None): LayerNorm backward of g [+ add] (the residual branch's gradient).
    phase "data": dx only -> (dx, stats);  phase "params" (stats of the "data" call): dw / db only -> (dw, db)."""
    B, C_, L = x.shape
    assert x.stride(2) == 1 and g.stride(2) == 1 and g.dtype == x.dtype and (add is None or (add.stride(2) == 1 and add.dtype == x.dtype))
    assert phase in ("both", "data", "params") and (phase != "params" or stats is not None)
    dx = torch.empty((B, C_, L), dtype=x.dtype, device=x.device) if phase != "params" else None
    if stats is None:
        stats = torch.empty((B, L, 2), dtype=torch.float32, device=x.device)
    dw = db = None
    if phase != "data":
        if zeroed is not None:
            dw, db = zeroed[0], (zeroed[1] if mode == 1 else None)
        elif need_param_grads:
            dw = torch.zeros(C_, dtype=torch.float32, device=x.device)
            db = torch.zeros(C_, dtype=torch.float32, device=x.device) if mode == 1 else None
    a = _lib.LnBwdArgs(x=_ptr(x), g=_ptr(g), add=_ptr(add), w=_ptr(w), dx=_ptr(dx), dw=_ptr(dw), db=_ptr(db), stats=_ptr(stats),
                       batch=B, C=C_, L=L, mode=mode, x_bs=x.stride(0), x_cs=x.stride(1), g_bs=g.stride(0), g_cs=g.stride(1),
                       a_bs=add.stride(0) if add is not None else 0, a_cs=add.stride(1) if add is not None else 0,
                       dx_bs=dx.stride(0) if dx is not None else 0, dx_cs=dx.stride(1) if dx is not None else 0, dtype=_DT[x.dtype])
    _run("vmb_layernorm_bwd", x, "ln_bwd", a, kernels=(1 if dx is not None else 0) + (1 if dw is not None else 0))
    if phase == "data":
        return dx, stats
    if phase == "params":
        return dw, db
    return dx, dw, db


def merge_norm_gate_bwd(ws, z, dy2, dpooled, ln_w, ln_b, C_, L, dz_out, zeroed=None, phase="both"):
    """backward of merge_norm_gate(z_preact=True).  ws: the forward's workspace; dy2 (B,C,L) contiguous; dpooled (B,C) fp32|None;
    dz_out: (B,C,L) view receiving the gradient w.r.t. the pre-activation z.  -> (dm (B,C,L), d ln_w, d ln_b).
    phase "data": -> dm (dz_out written);  phase "params": -> (d ln_w, d ln_b) only."""
    B = dy2.shape[0]
    assert dy2.is_contiguous() and z.stride(2) == 1 and (dz_out is None or dz_out.stride(2) == 1) and phase in ("both", "data", "params")
    merged = ws.view(torch.float32)
    stats = merged[B * C_ * L:]
    dm = torch.empty((B, C_, L), dtype=dy2.dtype, device=dy2.device) if phase != "params" else None
    dz = dz_out if phase != "params" else None
    dw = db = None
    if phase != "data":
        dw = torch.zeros(C_, dtype=torch.float32, device=dy2.device) if zeroed is None else zeroed[0]
        db = torch.zeros(C_, dtype=torch.float32, device=dy2.device) if zeroed is None else zeroed[1]
    a = _lib.MergeBwdArgs(merged=_ptr(merged), stats=_ptr(stats), z=_ptr(z), dy2=_ptr(dy2), dpooled=_ptr(dpooled), w=_ptr(ln_w),
                          b=_ptr(ln_b), dm=_ptr(dm), dz=_ptr(dz), dw=_ptr(dw), db=_ptr(db), batch=B, C=C_, L=L, z_bs=z.stride(0),
                          z_cs=z.stride(1), dz_bs=dz.stride(0) if dz is not None else 0, dz_cs=dz.stride(1) if dz is not None else 0,
                          dtype=_DT[dy2.dtype])
    _run("vmb_merge_norm_gate_bwd", dy2, "merge_bwd", a, kernels=(1 if dm is not None else 0) + (1 if dw is not None else 0))
    if phase == "data":
        return dm
    if phase == "params":
        return dw, db
    return dm, dw, db


def dwconv3x3_bwd(x, w9, bias, g, c_out, H, W, mode, zeroed=None, phase="both", dv=None):
    """backward of dwconv3x3 (mode 0 / 1) up to the conv output: -> (dv (B, channels, L), dw9 (channels, 9) fp32, dbias (channels) fp32|None);
    the input gradient is dwconv3x3(dv, w9.flip(-1), None, channels, H, W, 2).
    phase "data": -> dv only;  phase "params" (dv of the "data" call, g unused): -> (dw9, dbias) only."""
    B = x.shape[0]
    ch = c_out * (2 if mode else 1)
    assert x.stride(2) == 1 and phase in ("both", "data", "params")
    if phase == "params":
        assert dv is not None and dv.dtype == x.dtype
        g = None
    else:
        assert g.stride(2) == 1 and g.dtype == x.dtype
        dv = torch.empty((B, ch, H * W), dtype=x.dtype, device=x.device)
    dw = dbias = None
    if phase != "data":
        dw = torch.zeros((ch, 9), dtype=torch.float32, device=x.device) if zeroed is None else zeroed[0]
        dbias = (torch.zeros(ch, dtype=torch.float32, device=x.device) if zeroed is None else zeroed[1]) if bias is not None else None
    a = _lib.DwconvBwdArgs(x=_ptr(x), w=_ptr(w9), bias=_ptr(bias), g=_ptr(g), dv=_ptr(dv), dw=_ptr(dw), dbias=_ptr(dbias), batch=B,
                           c_out=c_out, H=H, W=W, mode=mode, x_bs=x.stride(0), x_cs=x.stride(1),
                           g_bs=g.stride(0) if g is not None else 0, g_cs=g.stride(1) if g is not None else 0,
                           dv_bs=dv.stride(0), dv_cs=dv.stride(1), dtype=_DT[x.dtype])
    _run("vmb_dwconv3x3_bwd", x, "dwconv_bwd", a, kernels=(1 if g is not None else 0) + (1 if dw is not None else 0))
    if phase == "data":
        return dv
    if phase == "params":
        return dw, dbias
    return dv, dw, dbias


def channel_gate_bwd(dyg, y2, gate, mode):
    """dyg, y2: (B,C,L) contiguous; gate (B,C) fp32 -> (dy2 (B,C,L), dgate (B,C) fp32)."""
    B, C_, L = y2.shape
    assert dyg.is_contiguous() and y2.is_contiguous() and gate.is_contiguous() and gate.dtype == torch.float32
    dy2 = torch.empty_like(y2)
    dg = torch.empty((B, C_), dtype=torch.float32, device=y2.device)
    a = _lib.GateBwdArgs(dyg=_ptr(dyg), y2=_ptr(y2), gate=_ptr(gate), dy2=_ptr(dy2), dgate=_ptr(dg), batch=B, C=C_, L=L, mode=mode,
                         dtype=_DT[y2.dtype])
    _run("vmb_channel_gate_bwd", y2, "gate_bwd", a)
    return dy2, dg


def pixlin_wgrad(dy, x, per_batch=False, out=None, dbias=None, deterministic=None, workspace=None):
    """dW[m,k] = sum_{b,p} dy[b,m,p] x[b,k,p] -> fp32 (M,K)  (or (B,M,K) without the batch sum).  16-bit activations with 16 B aligned
    rows run this library's mma.sync split-pixel kernel; fp32 (parity mode) or unaligned rows go to the library GEMM.
    out: optional fp32 accumulator (the result is ADDED: pre-zero it for a plain result); dbias: optional (M) fp32 accumulator receiving
    sum_{b,p} dy (the bias gradient).
    deterministic: None follows torch.are_deterministic_algorithms_enabled().  True: every CTA stores its partial in its own workspace
    slot and a second kernel adds their fixed-order sum once to out / dbias (bitwise reproducible; timing tag "wgrad_det").  False:
    fp32 atomics (tag "wgrad").  The fp32 / unaligned fallback is a torch GEMM either way.  workspace: as in selective_scan_bwd."""
    B, M, L = dy.shape
    K = x.shape[1]
    ok = (dy.dtype in (torch.bfloat16, torch.float16) and x.dtype == dy.dtype and dy.stride(2) == 1 and x.stride(2) == 1
          and all(s % 8 == 0 for s in (dy.stride(0), dy.stride(1), x.stride(0), x.stride(1)))
          and dy.data_ptr() % 16 == 0 and x.data_ptr() % 16 == 0)
    if not ok:
        wb = torch.bmm(dy.float(), x.float().transpose(1, 2))  # fp32 operands: a 16-bit bmm would round dW to 16 bits
        if dbias is not None:
            dbias += dy.float().sum((0, 2))
        res = wb if per_batch else wb.sum(0)
        if out is not None:
            out.add_(res)  # same contract as the kernel: ADD into the (pre-zeroed or accumulating) buffer
            return out
        return res
    if out is None:
        out = torch.zeros((B, M, K) if per_batch else (M, K), dtype=torch.float32, device=dy.device)
    det = _deterministic(deterministic)
    a = _lib.WgradArgs(dy=_ptr(dy), x=_ptr(x), out=_ptr(out), batch=B, M=M, K=K, L=L, dy_bs=dy.stride(0), dy_cs=dy.stride(1),
                       x_bs=x.stride(0), x_cs=x.stride(1), per_batch=int(per_batch), dtype=_DT[dy.dtype], dbias=_ptr(dbias),
                       deterministic=int(det))
    if not det:
        _run("vmb_pixlin_wgrad", dy, "wgrad", a)
        return out
    with torch.cuda.device(dy.device):
        ws = _workspace(_lib.lib().vmb_pixlin_wgrad_workspace_bytes(C.byref(a)), workspace, dy.device, "pixlin_wgrad")
    a.workspace = ws.data_ptr()
    _run("vmb_pixlin_wgrad", dy, "wgrad_det", a, kernels=2)
    return out


# vmb_prep_job types (include/vmambair_b200.h, vmb_prep_block_weights): (M,K) -> (M,ld) converted, columns >= K zero;  (M,K) ->
# (K,ld) transposed, columns >= M zero;  x_proj and dt_proj folded into one matrix and its transpose;  -exp(src);  taps flipped
PREP_PAD_COPY, PREP_TRANSPOSE, PREP_FOLD, PREP_NEG_EXP, PREP_FLIP_TAPS = 0, 1, 2, 3, 4

# one vmb_prep_job, tensors in place of its pointers.  type, src, dst, M and K are always given; src2, dst2, N2 and ld2 only for
# PREP_FOLD, ld (the padded row length) only for the 16-bit outputs
PrepJob = collections.namedtuple("PrepJob", "type src src2 dst dst2 M K N2 ld ld2", defaults=(None, None, None, 0, 0, 0, 0, 0))


def prep_block_weights(jobs, dtype):
    """jobs: PrepJob or (type, src, src2, dst, dst2, M, K, N2, ld, ld2) tuples -- see vmb_prep_block_weights; one launch."""
    jobs = [PrepJob._make(j) for j in jobs]
    a = _lib.PrepArgs(njobs=len(jobs), dtype=_DT[dtype])
    for i, j in enumerate(jobs):
        a.jobs[i] = _lib.PrepJob(src=_ptr(j.src), src2=_ptr(j.src2), dst=_ptr(j.dst), dst2=_ptr(j.dst2), type=j.type, M=j.M, K=j.K,
                                 N2=j.N2, ld=j.ld, ld2=j.ld2)
    _run("vmb_prep_block_weights", jobs[0].src, "prep", a)


def sum4_add(x4, add):
    """x4 (B,4,C,L) contiguous, add (B,C,L) contiguous -> add + x4.sum(1) (fp32 accumulation, result in the input dtype).
    The kernel moves 16 B vectors; C*L not a multiple of the vector width, or an operand not 16 B aligned, takes the same sum in torch."""
    B = x4.shape[0]
    assert x4.is_contiguous() and add.is_contiguous() and x4.dtype == add.dtype
    if add[0].numel() % (16 // add.element_size()) or x4.data_ptr() % 16 or add.data_ptr() % 16:
        return (add.float() + x4.float().sum(1)).to(add.dtype)
    out = torch.empty_like(add)
    _run("vmb_sum4_add", x4, None, _ptr(x4), _ptr(add), _ptr(out), B, add[0].numel(), _DT[x4.dtype])  # counted, not timed
    return out


def channel_branch_bwd_supported(C_, prm) -> bool:
    return prm["N"] <= 16 and 2 * prm["dc"] * 16 <= 512 and \
        _lib.lib().vmb_channel_branch_bwd_smem_bytes(C_, prm["dc"], prm["Rc"], prm["N"]) <= 227 * 1024


def channel_branch_bwd(pooled, inv_count, prm, C_, dc_out, into=None):
    """backward of channel_branch: -> (dpooled (B,C) fp32, dict of fp32 parameter gradients keyed like prm).
    into: optional {key: contiguous fp32 accumulator} -- those gradients are ADDED there (e.g. the parameters' .grad buffers)"""
    B = pooled.shape[0]
    dev = pooled.device
    dc, Rc, N = prm["dc"], prm["Rc"], prm["N"]
    RN = Rc + 2 * N
    sizes = dict(cin_w=dc, cin_b=dc, xc_proj=2 * RN * dc, dtc_w=2 * dc * Rc, dtc_b=2 * dc, Ac_logs=2 * dc * N, Dsc=2 * dc, cout_w=dc,
                 cout_b=1, cn_w=C_, cn_b=C_)
    into = into or {}
    own = {k: n for k, n in sizes.items() if k not in into}
    g, o = {}, 0
    if own:
        flat = torch.zeros(sum(own.values()), dtype=torch.float32, device=dev)  # one zero fill for every accumulator
        for k, n in own.items():
            g[k] = flat[o:o + n]
            o += n
    for k, t in into.items():
        assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == sizes[k]
        g[k] = t
    has_cin, has_cout = prm["cin_w"] is not None, prm["cout_w"] is not None
    dpooled = torch.empty((B, C_), dtype=torch.float32, device=dev)
    scratch = torch.empty(_lib.lib().vmb_channel_branch_bwd_scratch_bytes(B, dc, C_) // 4, dtype=torch.float32, device=dev)
    dc_out = dc_out.float().contiguous()
    a = _lib.ChannelBwdArgs(fwd=_channel_args(pooled, inv_count, prm, C_, None), dc_out=_ptr(dc_out), d_pooled=_ptr(dpooled),
                            d_cin_w=_ptr(g["cin_w"]) if has_cin else None, d_cin_b=_ptr(g["cin_b"]) if has_cin else None,
                            d_xc_proj=_ptr(g["xc_proj"]), d_dtc_w=_ptr(g["dtc_w"]), d_dtc_b=_ptr(g["dtc_b"]), d_Ac_logs=_ptr(g["Ac_logs"]),
                            d_Dsc=_ptr(g["Dsc"]), d_cout_w=_ptr(g["cout_w"]) if has_cout else None,
                            d_cout_b=_ptr(g["cout_b"]) if has_cout else None, d_cn_w=_ptr(g["cn_w"]), d_cn_b=_ptr(g["cn_b"]),
                            scratch=_ptr(scratch))
    _run("vmb_channel_branch_bwd", pooled, "channel_bwd", a)
    return dpooled, g


# ---- image-level I/O (vmambair_b200.enhance; RealSR/VmambaIR/utils.py:174-243) ----

def _image_geom(img, who):
    """(H, W, channels, u16, row / pixel / channel element strides) of a uint8 / uint16 (H, W) or (H, W, C) CUDA tensor"""
    if img.dtype not in (torch.uint8, torch.uint16):
        raise RuntimeError(f"{who}: image dtype must be uint8 or uint16, got {img.dtype}")
    if not img.is_cuda:
        raise RuntimeError(f"{who}: image must be a CUDA tensor")
    if img.dim() == 2:
        (H, W), (rs, ps), c, cs = img.shape, img.stride(), 1, 0
    elif img.dim() == 3 and img.shape[2] in (1, 3, 4):
        (H, W, c), (rs, ps, cs) = img.shape, img.stride()
    else:
        raise RuntimeError(f"{who}: image must be (H, W) or (H, W, C) with C in 1, 3, 4; got {tuple(img.shape)}")
    return H, W, c, int(img.dtype == torch.uint16), rs, ps, cs


def image_max(img):
    """largest value of a uint8 / uint16 image as a 1-element int32 CUDA tensor (read it back once: enhance's 16-bit test)"""
    H, W, c, u16, rs, ps, cs = _image_geom(img, "image_max")
    out = torch.empty(1, dtype=torch.int32, device=img.device)
    a = _lib.ImageMaxArgs(img=_ptr(img), H=H, W=W, channels=c, u16=u16, row_stride=rs, pixel_stride=ps, channel_stride=cs,
                          max_out=_ptr(out))
    _run("vmb_image_max", img, "image_max", a, nbytes=H * W * c * img.element_size())
    return out


def image_to_planes(img, max_range, pad_h=(0, 0, 0), pad_w=(0, 0, 0), alpha_plane=False, dtype=torch.float32):
    """uint8 / uint16 HWC image -> (1 + alpha_plane, 3, H + sum(pad_h), W + sum(pad_w)) planes in `dtype`: img / max_range, BGR -> RGB
    (gray repeated), three successive bottom / right reflect pads; alpha_plane: image 1 of the batch is the alpha channel x 3."""
    H, W, c, u16, rs, ps, cs = _image_geom(img, "image_to_planes")
    Hp, Wp = H + sum(pad_h), W + sum(pad_w)
    out = torch.empty((1 + int(alpha_plane), 3, Hp, Wp), dtype=dtype, device=img.device)
    a = _lib.ImageToPlanesArgs(img=_ptr(img), out=_ptr(out), H=H, W=W, channels=c, u16=u16, row_stride=rs, pixel_stride=ps,
                               channel_stride=cs, max_range=float(max_range), pad_h=(C.c_int * 3)(*pad_h),
                               pad_w=(C.c_int * 3)(*pad_w), alpha_plane=int(bool(alpha_plane)), dtype=_DT[dtype])
    _run("vmb_image_to_planes", img, "image_to_planes", a, nbytes=H * W * c * img.element_size() + out.numel() * out.element_size())
    return out


def planes_to_image(planes, H, W, channels, max_range, out_dtype, alpha_src=None, out=None):
    """(batch, 3, >= H, >= W) planes (pixel-contiguous rows) -> uint8 / uint16 image (H, W) for channels 1, else (H, W, channels):
    top-left crop, clamp to [0, 1], RGB -> BGR, BGR2GRAY for channels 1; channels 4: alpha from planes image 1 (BGR2GRAY), or, with
    alpha_src (the source image's alpha channel, (h, w) uint8 / uint16 view), cv2 INTER_LINEAR from it; x max_range, rounded half to
    even, saturated."""
    if planes.dtype not in _DT or planes.dim() != 4 or planes.shape[1] != 3 or planes.stride(3) != 1 or not planes.is_cuda:
        raise RuntimeError("planes_to_image: planes must be a (B, 3, H, W) float32 / bf16 / fp16 CUDA tensor with stride(3) == 1")
    if planes.shape[2] < H or planes.shape[3] < W or (channels == 4 and alpha_src is None and planes.shape[0] < 2):
        raise RuntimeError(f"planes_to_image: planes {tuple(planes.shape)} too small for a {H} x {W} x {channels} image")
    shape = (H, W) if channels == 1 else (H, W, channels)
    if out is None:
        out = torch.empty(shape, dtype=out_dtype, device=planes.device)
    if tuple(out.shape) != shape or out.dtype not in (torch.uint8, torch.uint16) or (channels > 1 and out.stride(2) != 1):
        raise RuntimeError(f"planes_to_image: out must be a uint8 / uint16 {shape} tensor with contiguous channels")
    ah = aw = ars = aps = au16 = 0
    if alpha_src is not None:
        ah, aw, _, au16, ars, aps, _ = _image_geom(alpha_src, "planes_to_image")
    a = _lib.PlanesToImageArgs(planes=_ptr(planes), out=_ptr(out), alpha_src=_ptr(alpha_src), H=H, W=W, channels=channels,
                               u16=int(out.dtype == torch.uint16), p_bs=planes.stride(0), p_cs=planes.stride(1), p_rs=planes.stride(2),
                               out_rs=out.stride(0), out_ps=out.stride(1), alpha_mode=int(alpha_src is not None), alpha_H=ah,
                               alpha_W=aw, alpha_u16=au16, alpha_rs=ars, alpha_ps=aps, max_range=float(max_range),
                               dtype=_DT[planes.dtype])
    _run("vmb_planes_to_image", planes, "planes_to_image", a,
         nbytes=H * W * (planes.element_size() * 3 * (1 + int(channels == 4 and alpha_src is None)) + channels * out.element_size()))
    return out


def resize_lanczos4(img, width, height):
    """cv2.resize(img, (width, height), interpolation=cv2.INTER_LANCZOS4) of a uint8 / uint16 (H, W) or (H, W, C) CUDA image"""
    H, W, c, u16, rs, ps, cs = _image_geom(img, "resize_lanczos4")
    if c > 1 and cs != 1:
        raise RuntimeError("resize_lanczos4: the channels of a pixel must be contiguous")
    out = torch.empty((height, width) if img.dim() == 2 else (height, width, c), dtype=img.dtype, device=img.device)
    a = _lib.ResizeLanczos4Args(src=_ptr(img), dst=_ptr(out), sH=H, sW=W, dH=height, dW=width, channels=c, u16=u16,
                                src_rs=rs, src_ps=ps, dst_rs=out.stride(0), dst_ps=out.stride(1))
    _run("vmb_resize_lanczos4", img, "resize_lanczos4", a, nbytes=(H * W + height * width) * c * img.element_size())
    return out


# ---- image metrics (csrc/metrics.cu): PSNR / SSIM of the reference's psnr_ssim.py and Deraining/utils.py ----
MSRC = {torch.uint8: 0, torch.uint16: 1, torch.float32: 2, torch.float64: 3}   # VMB_MSRC_*: the value itself
MSRC_Q = {torch.float32: 4, torch.bfloat16: 5, torch.float16: 6}                 # VMB_MSRC_Q_*: tensor2img's uint8 of the value
SSIM_MODES = {"valid": 0, "replicate": 1, "replicate3d": 2}                       # VMB_SSIM_*


def metric_src(t, offset, strides, quantize=False):
    """vmb_metric_src of the (batch, H, W, channels) view of CUDA tensor t's storage that starts `offset` elements after t.data_ptr()
    with element strides (batch, row, pixel, channel); a stride may be negative (an RGB planar tensor read as BGR)."""
    table = MSRC_Q if quantize else MSRC
    if t.dtype not in table:
        raise RuntimeError(f"metrics: {'quantized ' if quantize else ''}source dtype {t.dtype} not in {list(table)}")
    return _lib.MetricSrc(img=C.c_void_p(t.data_ptr() + offset * t.element_size()), dtype=table[t.dtype], batch_stride=strides[0],
                          row_stride=strides[1], pixel_stride=strides[2], channel_stride=strides[3])


def to_y_channel_planes(t, src, batch, H, W, channels):
    """to_y_channel of `src` (a metric_src view of CUDA tensor t) -> (batch, H, W) float32"""
    out = torch.empty((batch, H, W), dtype=torch.float32, device=t.device)
    a = _lib.ToYArgs(src=src, batch=batch, H=H, W=W, channels=channels, out=_ptr(out))
    _run("vmb_to_y_channel", t, "to_y_channel", a, nbytes=batch * H * W * (channels * t.element_size() + 4))
    return out


def psnr_sums(t, src1, src2, batch, H, W, channels, y_channel):
    """-> (mse, max of image 1, psnr), three (batch,) float64 tensors on t's device (vmb_psnr)"""
    out = torch.empty((3, batch), dtype=torch.float64, device=t.device)
    a = _lib.PsnrArgs(img1=src1, img2=src2, batch=batch, H=H, W=W, channels=channels, y_channel=int(y_channel),
                      mse=_ptr(out[0]), max_value=_ptr(out[1]), psnr=_ptr(out[2]))
    ws = torch.empty(_lib.lib().vmb_psnr_workspace_bytes(C.byref(a)), dtype=torch.uint8, device=t.device)
    a.workspace = _ptr(ws)
    _run("vmb_psnr", t, "psnr", a, nbytes=2 * batch * H * W * channels * t.element_size(), kernels=2)
    return out[0], out[1], out[2]


def ssim_mean(t, src1, src2, batch, H, W, channels, y_channel, mode, taps, mix=None, max_value=None):
    """-> (batch,) float64: the mean SSIM map of each pair (vmb_ssim; mode a key of SSIM_MODES; taps: 11 floats; mix: the
    channels x channels filter across channels of 'replicate3d', with max_value (batch,) float64 for its constants)"""
    out = torch.empty(batch, dtype=torch.float64, device=t.device)
    mix9 = [0.0] * 9
    for i, v in enumerate([] if mix is None else [v for row in mix for v in row]):
        mix9[i] = float(v)
    a = _lib.SsimArgs(img1=src1, img2=src2, batch=batch, H=H, W=W, channels=channels, y_channel=int(y_channel), mode=SSIM_MODES[mode],
                      taps=(C.c_double * 11)(*taps), mix=(C.c_double * 9)(*mix9), max_value=_ptr(max_value), ssim=_ptr(out))
    ws = torch.empty(_lib.lib().vmb_ssim_workspace_bytes(C.byref(a)), dtype=torch.uint8, device=t.device)
    a.workspace = _ptr(ws)
    empty = mode == "valid" and (H <= 10 or W <= 10)  # no map: only the kernel that writes nan runs
    _run("vmb_ssim", t, "ssim", a, nbytes=2 * batch * H * W * channels * t.element_size(), kernels=1 if empty else 2)
    return out


# ---- NIQE (csrc/niqe.cu): calculate_niqe of the reference's niqe.py; nothing read on the host ----
NIQE_CONVERT = {"y": _lib.NIQE_Y, "gray": _lib.NIQE_GRAY, None: _lib.NIQE_PLANE}


def niqe_table(device):
    """-> (9801,) float64 on `device`: r(gamma) of estimate_aggd_param over gam = np.arange(0.2, 10.001, 0.001)"""
    out = torch.empty(_lib.NIQE_TABLE, dtype=torch.float64, device=device)
    _run("vmb_niqe_table", out, "niqe_table", _ptr(out), nbytes=out.numel() * 8)
    return out


def niqe_prep(t, src, batch, H, W, channels, convert):
    """-> (plane (batch, H, W), half (batch, H / 2, W / 2)), float32: `src` (a metric_src view of CUDA tensor t, already cut to whole
    96 x 96 blocks) as the plane NIQE filters, under `convert` (a key of NIQE_CONVERT), and its 2 x 2 mean"""
    plane = torch.empty((batch, H, W), dtype=torch.float32, device=t.device)
    half = torch.empty((batch, H // 2, W // 2), dtype=torch.float32, device=t.device)
    a = _lib.NiqePrepArgs(src=src, batch=batch, H=H, W=W, channels=channels, convert=NIQE_CONVERT[convert], plane=_ptr(plane),
                          half=_ptr(half))
    _run("vmb_niqe_prep", t, "niqe_prep", a, nbytes=batch * H * W * (channels * t.element_size() + 5))
    return plane, half


def niqe_features(plane, half, table, window, mscn=False):
    """-> (batch, blocks, 36) float64 features (the reference's distparam) of the prep planes; window: 49 floats (the 7 x 7 Gaussian,
    row-major).  mscn=True: also the normalised planes, (features, mscn (batch, H, W), mscn_half (batch, H / 2, W / 2))."""
    batch, H, W = plane.shape
    nb = (H // _lib.NIQE_BLOCK) * (W // _lib.NIQE_BLOCK)
    feats = torch.empty((batch, nb, _lib.NIQE_FEATURES), dtype=torch.float64, device=plane.device)
    m1 = torch.empty_like(plane) if mscn else None
    m2 = torch.empty_like(half) if mscn else None
    a = _lib.NiqeFeaturesArgs(plane=_ptr(plane), half=_ptr(half), table=_ptr(table), features=_ptr(feats), mscn=_ptr(m1),
                              mscn_half=_ptr(m2), window=(C.c_double * 49)(*window), batch=batch, H=H, W=W)
    _run("vmb_niqe_features", plane, "niqe_features", a, nbytes=(plane.numel() + half.numel()) * 4 + feats.numel() * 8)
    return (feats, m1, m2) if mscn else feats


def niqe_score(feats, mu_pris, cov_pris):
    """-> (batch,) float64 NIQE scores of (batch, blocks, 36) features against the pristine model (36,) / (36, 36) float64"""
    batch, nb, _ = feats.shape
    out = torch.empty(batch, dtype=torch.float64, device=feats.device)
    a = _lib.NiqeScoreArgs(features=_ptr(feats) if nb else None, mu_pris=_ptr(mu_pris), cov_pris=_ptr(cov_pris), score=_ptr(out),
                           batch=batch, blocks=nb)
    _run("vmb_niqe_score", feats, "niqe_score", a, nbytes=feats.numel() * 8)
    return out


# ---- degradations (csrc/degrade.cu): basicsr's Real-ESRGAN synthesis operators; float32 NCHW, contiguous, nothing read on the host ----
NOISE_GAUSSIAN, NOISE_POISSON = 0, 1  # VMB_NOISE_*


def filter2d(img, kernel, per_image, quantize_out=False):
    """(b, c, H, W) img cross-correlated with the (k, k) kernel(s) `kernel` ((1, k, k) shared or (b, k, k) per image), reflect pads"""
    b, c, H, W = img.shape
    k = kernel.shape[-1]
    out = torch.empty_like(img)
    a = _lib.Filter2dArgs(img=_ptr(img), out=_ptr(out), kernel=_ptr(kernel), batch=b, channels=c, H=H, W=W, k=k,
                          per_image=int(per_image), quantize_out=int(quantize_out))
    _run("vmb_filter2d", img, "filter2d", a, nbytes=2 * img.numel() * 4)
    return out


def usm_sharp(img, taps, weight, threshold):
    """USMSharp of (b, c, H, W) img with the separable kernel outer(taps, taps)"""
    b, c, H, W = img.shape
    out, ws = torch.empty_like(img), torch.empty_like(img)
    a = _lib.UsmSharpArgs(img=_ptr(img), out=_ptr(out), workspace=_ptr(ws), batch=b, channels=c, H=H, W=W, k=len(taps),
                          taps=(C.c_float * 51)(*taps), weight=float(weight), threshold=float(threshold))
    _run("vmb_usm_sharp", img, "usm_sharp", a, nbytes=7 * img.numel() * 4, kernels=2)
    return out


def jpeg(img, quality=None, factor=0.0, clamp_in=False, quantize_out=False):
    """DiffJPEG(differentiable=False) of (b, 3, H, W) img: quality a (b,) float32 device tensor, or None and the scalar `factor`"""
    b, _, H, W = img.shape
    out = torch.empty_like(img)
    a = _lib.JpegArgs(img=_ptr(img), out=_ptr(out), quality=_ptr(quality), factor=float(factor), batch=b, H=H, W=W,
                      clamp_in=int(clamp_in), quantize_out=int(quantize_out))
    _run("vmb_jpeg", img, "jpeg", a, nbytes=2 * img.numel() * 4)
    return out


def noise_levels(img):
    """-> (rates (b, 3, H, W), rates_gray (b, 1, H, W), vals (b,), vals_gray (b,)) of generate_poisson_noise_pt, on the device"""
    b, _, H, W = img.shape
    rates = torch.empty_like(img)
    rates_gray = torch.empty((b, 1, H, W), dtype=torch.float32, device=img.device)
    vals = torch.empty((2, b), dtype=torch.float32, device=img.device)
    ws = torch.empty(64 * b, dtype=torch.uint8, device=img.device)
    a = _lib.NoiseLevelsArgs(img=_ptr(img), rates=_ptr(rates), rates_gray=_ptr(rates_gray), vals=_ptr(vals[0]), vals_gray=_ptr(vals[1]),
                             workspace=_ptr(ws), batch=b, H=H, W=W)
    _run("vmb_noise_levels", img, "noise_levels", a, nbytes=(2 * img.numel() + rates.numel() + rates_gray.numel()) * 4, kernels=2)
    return rates, rates_gray, vals[0], vals[1]


def noise_apply(img, kind, noise, noise_gray, u_param, u_gray, param_range, gray_prob, clip, rounds, vals=None, vals_gray=None):
    """img + the Gaussian / Poisson noise of basicsr from torch's draws (vmb_noise_apply_args); -> a new tensor"""
    b, c, H, W = img.shape
    out = torch.empty_like(img)
    lo, hi = param_range
    a = _lib.NoiseApplyArgs(img=_ptr(img), out=_ptr(out), noise=_ptr(noise), noise_gray=_ptr(noise_gray), u_param=_ptr(u_param),
                            u_gray=_ptr(u_gray), param_lo=float(lo), param_span=float(hi - lo), gray_prob=float(gray_prob),
                            vals=_ptr(vals), vals_gray=_ptr(vals_gray), kind=kind, batch=b, channels=c, H=H, W=W, clip=int(clip),
                            rounds=int(rounds))
    _run("vmb_noise_apply", img, "noise_apply", a, nbytes=(3 * img.numel() + noise_gray.numel()) * 4)
    return out


# ---- GAN stage (csrc/gan.cu): UNetDiscriminatorSN between its convolutions and the vanilla GAN loss; fp32 or bf16 activations,
# contiguous; every reduction in a fixed order (bitwise reproducible), nothing read on the host ----
def _gan_dt(t):
    if t.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"the GAN kernels take float32 or bfloat16 tensors, not {t.dtype}")
    return _DT[t.dtype]


def _rows_cols(ws):
    n = len(ws)
    rows, cols = (C.c_int * _lib.SN_MAX_LAYERS)(), (C.c_int * _lib.SN_MAX_LAYERS)()
    for i, w in enumerate(ws):
        rows[i], cols[i] = w.shape[0], w[0].numel()
    return n, rows, cols


def spectral_norm(ws, us, vs, train, dtype, eps=1e-12):
    """torch.nn.utils.spectral_norm of the fp32 weights `ws` (weight_orig, contiguous) with their u / v buffers `us` / `vs`, all
    layers in one call: train advances u and v in place.  -> (W / sigma per layer in `dtype`, sigma (layers,), the u and v used)"""
    n, rows, cols = _rows_cols(ws)
    dev = ws[0].device
    wn_flat = torch.empty(sum(w.numel() for w in ws), dtype=dtype, device=dev)
    uv_flat = torch.empty(sum(rows[:n]) + sum(cols[:n]), dtype=torch.float32, device=dev)
    sigma = torch.empty(n, dtype=torch.float32, device=dev)
    ws_bytes = _lib.lib().vmb_sn_workspace_bytes(n, rows, cols)
    work = torch.empty(ws_bytes // 4, dtype=torch.float32, device=dev)
    wns, us_save, vs_save, o, ouv = [], [], [], 0, 0
    for i, w in enumerate(ws):
        wns.append(wn_flat[o:o + w.numel()].view(w.shape))
        us_save.append(uv_flat[ouv:ouv + rows[i]])
        vs_save.append(uv_flat[ouv + rows[i]:ouv + rows[i] + cols[i]])
        o, ouv = o + w.numel(), ouv + rows[i] + cols[i]
    P = lambda ts: (C.c_void_p * _lib.SN_MAX_LAYERS)(*[t.data_ptr() for t in ts])
    a = _lib.SnFwdArgs(w=P(ws), wn=P(wns), u=P(us), v=P(vs), u_save=P(us_save), v_save=P(vs_save), rows=rows, cols=cols,
                       sigma=_ptr(sigma), workspace=_ptr(work), layers=n, train=int(train), dtype=_gan_dt(wn_flat), eps=float(eps))
    _run("vmb_sn_fwd", ws[0], "sn_fwd", a, nbytes=(2 if train else 1) * 4 * o + wn_flat.numel() * wn_flat.element_size(),
         kernels=4 if train else 2)
    return wns, sigma, us_save, vs_save


def spectral_norm_bwd(gs, ws, us, vs, sigma, grads, accumulate):
    """dW_orig of every layer of `spectral_norm` from the gradients `gs` of its outputs W / sigma (u, v, sigma: the saved ones),
    written to the fp32 tensors `grads`, or added to those where accumulate[i]"""
    n, rows, cols = _rows_cols(ws)
    work = torch.empty(_lib.lib().vmb_sn_bwd_workspace_bytes(n, rows, cols) // 4, dtype=torch.float32, device=ws[0].device)
    P = lambda ts: (C.c_void_p * _lib.SN_MAX_LAYERS)(*[t.data_ptr() for t in ts])
    acc = (C.c_int * _lib.SN_MAX_LAYERS)(*map(int, accumulate))
    a = _lib.SnBwdArgs(g=P(gs), w=P(ws), u=P(us), v=P(vs), grad=P(grads), rows=rows, cols=cols, accumulate=acc, sigma=_ptr(sigma),
                       workspace=_ptr(work), layers=n, dtype=_gan_dt(gs[0]))
    nel = sum(w.numel() for w in ws)
    _run("vmb_sn_bwd", ws[0], "sn_bwd", a, nbytes=nel * (2 * gs[0].element_size() + 4 * 4), kernels=2)


def gan_up(pre, skip=None):
    """F.interpolate(leaky_relu(pre, 0.2) [+ skip], scale_factor=2, mode='bilinear', align_corners=False) of (b, c, h, w) tensors"""
    b, c, h, w = pre.shape
    out = torch.empty((b, c, 2 * h, 2 * w), dtype=pre.dtype, device=pre.device)
    a = _lib.GanUpArgs(pre=_ptr(pre), skip=_ptr(skip), out=_ptr(out), planes=b * c, H=h, W=w, dtype=_gan_dt(pre))
    _run("vmb_gan_up", pre, "gan_up", a, nbytes=(pre.numel() * (2 if skip is not None else 1) + out.numel()) * pre.element_size())
    return out


def gan_up_bwd(dout, pre, want_skip):
    """-> (dpre, dskip or None) of gan_up from its output gradient: the adjoint of up2 gathered, times leaky'(pre) for dpre"""
    b, c, h, w = pre.shape
    dpre = torch.empty_like(pre)
    dskip = torch.empty_like(pre) if want_skip else None
    a = _lib.GanUpBwdArgs(dout=_ptr(dout), pre=_ptr(pre), dpre=_ptr(dpre), dskip=_ptr(dskip), planes=b * c, H=h, W=w, dtype=_gan_dt(pre))
    _run("vmb_gan_up_bwd", pre, "gan_up_bwd", a, nbytes=(dout.numel() + pre.numel() * (3 if want_skip else 2)) * pre.element_size())
    return dpre, dskip


def gan_act(x, skip=None, out=None):
    """leaky_relu(x, 0.2) [+ skip] into `out` (default: x itself, in place)"""
    out = x if out is None else out
    a = _lib.GanActArgs(x=_ptr(x), skip=_ptr(skip), out=_ptr(out), n=x.numel(), dtype=_gan_dt(x))
    _run("vmb_gan_act", x, "gan_act", a, nbytes=x.numel() * x.element_size() * (3 if skip is not None else 2))
    return out


def gan_act_bwd(g, ref, g2=None, out=None):
    """(g [+ g2]) * leaky'(ref) into `out` (default: g itself, in place)"""
    out = g if out is None else out
    a = _lib.GanActBwdArgs(g=_ptr(g), g2=_ptr(g2), ref=_ptr(ref), dx=_ptr(out), n=g.numel(), dtype=_gan_dt(g))
    _run("vmb_gan_act_bwd", g, "gan_act_bwd", a, nbytes=g.numel() * g.element_size() * (4 if g2 is not None else 3))
    return out


def bce_logits(x, target, weight):
    """weight * mean(BCEWithLogits(x, full_like(x, target))) -> 0-dim float32 tensor"""
    n = x.numel()
    loss = torch.empty((), dtype=torch.float32, device=x.device)
    work = torch.empty(_lib.lib().vmb_bce_logits_workspace_bytes(n) // 4, dtype=torch.float32, device=x.device)
    a = _lib.BceLogitsArgs(x=_ptr(x), loss=_ptr(loss), workspace=_ptr(work), n=n, target=float(target), weight=float(weight),
                           dtype=_gan_dt(x))
    _run("vmb_bce_logits", x, "bce_logits", a, nbytes=n * x.element_size(), kernels=2)
    return loss


def bce_logits_bwd(x, grad_loss, target, weight):
    """gradient of bce_logits with respect to x, for the upstream 0-dim float32 gradient grad_loss (read on the device)"""
    gx = torch.empty_like(x)
    a = _lib.BceLogitsBwdArgs(x=_ptr(x), grad_loss=_ptr(grad_loss), grad_x=_ptr(gx), n=x.numel(), target=float(target),
                              weight=float(weight), dtype=_gan_dt(x))
    _run("vmb_bce_logits_bwd", x, "bce_logits_bwd", a, nbytes=2 * x.numel() * x.element_size())
    return gx


# ---- GAN training step (csrc/gan_step.cu): pixel loss, logit means, the generator's output-gradient junction, the learning-rate
# schedule and the EMA alone; fixed-order sums, nothing read on the host ----
def mean_loss(x, y=None, weight=1.0, out=None):
    """weight * mean(|x - y|) (the recipes' L1Loss), or weight * mean(x) when y is None -> 0-dim float32 tensor (`out` if given).
    x, y: contiguous tensors of one dtype (float32 or bfloat16) and element count (the kernel indexes them linearly)"""
    if y is not None and (y.dtype != x.dtype or y.numel() != x.numel()):
        raise ValueError(f"mean_loss: x {x.dtype} {tuple(x.shape)} and y {y.dtype} {tuple(y.shape)} differ")
    if not x.is_contiguous() or (y is not None and (not y.is_contiguous() or y.device != x.device)):
        raise ValueError("mean_loss: x and y must be contiguous tensors on one device")
    n = x.numel()
    out = torch.empty((), dtype=torch.float32, device=x.device) if out is None else out
    work = torch.empty(_lib.lib().vmb_mean_loss_workspace_bytes(n) // 4, dtype=torch.float32, device=x.device)
    a = _lib.MeanLossArgs(x=_ptr(x), y=_ptr(y), out=_ptr(out), workspace=_ptr(work), n=n, weight=float(weight), dtype=_gan_dt(x))
    _run("vmb_mean_loss", x, "mean_loss", a, nbytes=n * x.element_size() * (1 if y is None else 2), kernels=2)
    return out


def gan_out_grad(out, gt, g_percep, g_gan, w_pix, dtype):
    """the generator's output gradient w_pix * sign(out - gt) / n + g_percep + g_gan, in `dtype`.  out, gt: contiguous, one dtype
    (float32 or bfloat16); g_percep, g_gan: contiguous float32 or None (term absent).  The kernel indexes all of them linearly."""
    if gt.dtype != out.dtype or gt.numel() != out.numel():
        raise ValueError(f"gan_out_grad: out {out.dtype} {tuple(out.shape)} and gt {gt.dtype} {tuple(gt.shape)} differ")
    for g in (g_percep, g_gan):
        if g is not None and (g.dtype != torch.float32 or g.numel() != out.numel()):
            raise ValueError(f"gan_out_grad: a loss gradient is {g.dtype} {tuple(g.shape)}, not float32 {tuple(out.shape)}")
    if not all(t.is_contiguous() and t.device == out.device for t in (out, gt, g_percep, g_gan) if t is not None):
        raise ValueError("gan_out_grad: out, gt and the loss gradients must be contiguous tensors on one device")
    dout = torch.empty(out.shape, dtype=dtype, device=out.device)
    a = _lib.GanOutGradArgs(out=_ptr(out), gt=_ptr(gt), g_percep=_ptr(g_percep), g_gan=_ptr(g_gan), dout=_ptr(dout), n=out.numel(),
                            w_pix=float(w_pix), in_dtype=_gan_dt(out), out_dtype=_gan_dt(dout))
    nb = out.numel() * (2 * out.element_size() + 4 * sum(g is not None for g in (g_percep, g_gan)) + dout.element_size())
    _run("vmb_gan_out_grad", out, "gan_out_grad", a, nbytes=nb)
    return dout


def lr_rule(base, step_gamma=1.0, step_size=0, milestones=(), milestone_gamma=1.0, periods=(), restart_weights=(), eta_mins=()):
    """one optimizer's schedule for lr_schedule: base * step_gamma ** (it // step_size) * milestone_gamma ** #{m <= it - 1}; or, when
    `periods` is given, basicsr's cosine annealing with restarts at last_epoch it - 1 (one restart weight and eta_min per period;
    CosineAnnealingRestartLR is the case of equal eta_mins), which the step decay and milestones cannot be combined with"""
    if len(milestones) > _lib.LR_MAX_MILESTONES:
        raise ValueError(f"lr_rule: {len(milestones)} milestones, at most {_lib.LR_MAX_MILESTONES}")
    if not len(periods) == len(restart_weights) == len(eta_mins) <= _lib.LR_MAX_PERIODS or any(int(p) < 1 for p in periods):
        raise ValueError(f"lr_rule: periods {tuple(periods)}, restart_weights {tuple(restart_weights)} and eta_mins {tuple(eta_mins)} "
                         f"must have one length, at most {_lib.LR_MAX_PERIODS}, and positive periods")
    if periods and (milestones or step_size > 0):
        raise ValueError("lr_rule: a cosine schedule takes no step decay or milestones")
    n = _lib.LR_MAX_PERIODS
    return _lib.LrRule(base=float(base), step_gamma=float(step_gamma), milestone_gamma=float(milestone_gamma), step_size=int(step_size),
                       milestones=(_lib.i64 * _lib.LR_MAX_MILESTONES)(*map(int, milestones)), n_milestones=len(milestones),
                       n_periods=len(periods), periods=(_lib.i64 * n)(*map(int, periods)),
                       restart_weights=(C.c_double * n)(*map(float, restart_weights)), eta_mins=(C.c_double * n)(*map(float, eta_mins)))


def lr_schedule(it, lr, rules):
    """one thread on the device: it += 1 (int64, 1 element), then lr[k] = rules[k] at the new it (lr: float32, len(rules) elements)"""
    if it.dtype != torch.int64 or lr.dtype != torch.float32 or lr.numel() < len(rules) or not 1 <= len(rules) <= 2:
        raise ValueError("lr_schedule: it must be int64, lr float32 with one element per rule, 1 or 2 rules")
    a = _lib.LrScheduleArgs(iter=_ptr(it), lr=_ptr(lr), rule=(_lib.LrRule * 2)(*rules), n_rules=len(rules))
    _run("vmb_lr_schedule", it, "lr_schedule", a)


def ema_update(ema, param, decay):
    """ema = decay * ema + (1 - decay) * param over two float32 buffers of one size, in place"""
    if ema.dtype != torch.float32 or param.dtype != torch.float32 or ema.numel() != param.numel():
        raise ValueError("ema_update: ema and param must be float32 buffers of one size")
    _run("vmb_ema_update", ema, "ema_update", _ptr(ema), _ptr(param), ema.numel(), float(decay), nbytes=12 * ema.numel())


# ---- restoration step's input preparation (csrc/restore_step.cu): progressive subset / crop and mixup of lq and gt ----
def batch_crop_mix(lq, gt, idx, row0, col0, size, scale, lam=None, perm=None, out=None):
    """lq[idx][:, :, row0:row0 + size, col0:col0 + size] and gt's window at scale x those coordinates, mixed when lam is given:
    out[i] = lam * s[i] + (1 - lam) * s[perm[i]], rounded as torch evaluates that expression with Python-float lam (fp32 products of
    lam and of float32(1 - lam), one fp32 sum), else a pure gather.  lq, gt: float32 CUDA tensors (B, C, H, W) on one device, any
    strides; size None: the whole of lq.  idx: up to 64 source images (repeats allowed); perm: a permutation of range(len(idx)).
    out: (lq_out, gt_out), contiguous float32 tensors of the result's shapes to write into (e.g. a CUDA graph's inputs).
    -> (lq_out, gt_out)"""
    if any(t.dim() != 4 or t.dtype != torch.float32 or not t.is_cuda or t.device != lq.device for t in (lq, gt)):
        raise ValueError("batch_crop_mix: lq and gt must be 4-d float32 CUDA tensors on one device")
    B, scale = lq.shape[0], int(scale)
    idx = [int(i) for i in idx]
    k = len(idx)
    size = (lq.shape[2], lq.shape[3]) if size is None else (int(size), int(size))
    if gt.shape[0] != B or not 1 <= k <= _lib.CROP_MIX_MAX_IMAGES or not all(0 <= i < B for i in idx):
        raise ValueError(f"batch_crop_mix: {k} indices {idx} into batches of {B} and {gt.shape[0]} images "
                         f"(1 to {_lib.CROP_MIX_MAX_IMAGES})")
    if scale < 1 or row0 < 0 or col0 < 0 or min(size) < 1 or row0 + size[0] > lq.shape[2] or col0 + size[1] > lq.shape[3] or \
            scale * (row0 + size[0]) > gt.shape[2] or scale * (col0 + size[1]) > gt.shape[3]:
        raise ValueError(f"batch_crop_mix: window {size} at ({row0}, {col0}), scale {scale}, leaves lq {tuple(lq.shape)} or "
                         f"gt {tuple(gt.shape)}")
    perm = list(range(k)) if perm is None else [int(p) for p in perm]
    if sorted(perm) != list(range(k)):
        raise ValueError(f"batch_crop_mix: perm {perm} is not a permutation of range({k})")
    shapes = [(k, lq.shape[1], *size), (k, gt.shape[1], scale * size[0], scale * size[1])]
    if out is None:
        out = tuple(torch.empty(sh, dtype=torch.float32, device=lq.device) for sh in shapes)
    if any(tuple(o.shape) != sh or o.dtype != torch.float32 or not o.is_contiguous() or o.device != lq.device
           for o, sh in zip(out, shapes)):
        raise ValueError(f"batch_crop_mix: out must be contiguous float32 tensors of shapes {shapes} on {lq.device}")

    def tensor(src, dst, s):
        return _lib.CropMixTensor(src=_ptr(src), dst=_ptr(dst), stride_n=src.stride(0), stride_c=src.stride(1), stride_h=src.stride(2),
                                  stride_w=src.stride(3), c=dst.shape[1], h=dst.shape[2], w=dst.shape[3], row0=s * row0, col0=s * col0)

    n = _lib.CROP_MIX_MAX_IMAGES
    a = _lib.BatchCropMixArgs(t=(_lib.CropMixTensor * 2)(tensor(lq, out[0], 1), tensor(gt, out[1], scale)), n_tensors=2, batch=k,
                              idx=(C.c_int * n)(*idx), perm=(C.c_int * n)(*perm), lam=1.0 if lam is None else float(lam),
                              one_minus_lam=0.0 if lam is None else 1.0 - float(lam), mix=int(lam is not None))
    _run("vmb_batch_crop_mix", lq, "batch_crop_mix", a, nbytes=4 * sum(o.numel() for o in out) * (3 if lam is not None else 2))
    return out


# ---- perceptual loss (csrc/perceptual.cu): basicsr's PerceptualLoss between the VGG convolutions; output and ground truth as one
# 2B batch, fp32 or bf16 activations, contiguous; every reduction in a fixed order, nothing read on the host ----
PERCEP_CRIT = {"l1": _lib.PERCEP_L1, "l2": _lib.PERCEP_L2, "fro": _lib.PERCEP_FRO}


def percep_norm(x, gt, mean, std, range_norm, dtype):
    """(B, 3, H, W) fp32 x and gt, any strides -> (2B, 3, H, W) `dtype`: [x; gt] through (v + 1) / 2 (range_norm) and
    (v - mean) / std (mean, std: the (1, 3, 1, 1) fp32 buffers, or None)"""
    B, _, H, W = x.shape
    out = torch.empty((2 * B, 3, H, W), dtype=dtype, device=x.device)
    a = _lib.PercepNormArgs(x=_ptr(x), gt=_ptr(gt), x_stride=(C.c_int64 * 4)(*x.stride()), gt_stride=(C.c_int64 * 4)(*gt.stride()),
                            mean=_ptr(mean), std=_ptr(std), out=_ptr(out), B=B, H=H, W=W, range_norm=int(range_norm),
                            dtype=_gan_dt(out))
    _run("vmb_percep_norm", x, "percep_norm", a, nbytes=2 * x.numel() * (4 + out.element_size()))
    return out


def percep_norm_bwd(g, std, range_norm):
    """gradient at x (fp32, contiguous) of percep_norm from the gradient g (B, 3, H, W) at its x half"""
    B, _, H, W = g.shape
    dx = torch.empty(g.shape, dtype=torch.float32, device=g.device)
    a = _lib.PercepNormBwdArgs(g=_ptr(g), dx=_ptr(dx), std=_ptr(std), B=B, H=H, W=W, range_norm=int(range_norm), dtype=_gan_dt(g))
    _run("vmb_percep_norm_bwd", g, "percep_norm_bwd", a, nbytes=g.numel() * (4 + g.element_size()))
    return dx


def percep_stage_ctas(B, C, H, W):
    """CTAs of vmb_percep_stage at this x-half shape: the partials it writes per feature site"""
    return _lib.lib().vmb_percep_stage_ctas(B, C, H, W)


def percep_stage(y, relu, pool, feat, partial, crit, save):
    """One stage after a VGG convolution, y (2B, C, H, W) = [x half; gt half]: ReLU in place (relu), the 2 x 2 max-pool (pool), and
    at each feature site k (0 conv, 1 relu, 2 pool) with feat[k] the criterion's per-CTA partials into partial[k].  With `save`, the
    backward's state for the x half.  -> (pooled or None, code or None, [save of each site or None])"""
    B2, Cc, H, W = y.shape
    B = B2 // 2
    dev = y.device
    pooled = torch.empty((B2, Cc, H // 2, W // 2), dtype=y.dtype, device=dev) if pool else None
    cells = (B, Cc, (H + 1) // 2, (W + 1) // 2)
    code = torch.empty(cells, dtype=torch.uint8, device=dev) if save and relu else None
    saves = [None] * 3
    if save:
        for k in range(3):
            if not feat[k]:
                continue
            if crit == "l1":  # a byte of sign codes per cell, or per pooled element
                saves[k] = torch.empty((B, Cc, H // 2, W // 2) if k == 2 else cells, dtype=torch.uint8, device=dev)
            else:
                saves[k] = torch.empty((B, Cc, H // 2, W // 2) if k == 2 else (B, Cc, H, W), dtype=torch.float32, device=dev)
    a = _lib.PercepStageArgs(y=_ptr(y), pooled=_ptr(pooled), code=_ptr(code), save=(C.c_void_p * 3)(*[0 if s is None else s.data_ptr()
                             for s in saves]), partial=(C.c_void_p * 3)(*[0 if p is None else p.data_ptr() for p in partial]),
                             feat=(C.c_int * 3)(*map(int, feat)), B=B, C=Cc, H=H, W=W, relu=int(relu), pool=int(pool),
                             crit=PERCEP_CRIT[crit], dtype=_gan_dt(y))
    nbytes = y.numel() * y.element_size() * (1 if pool or not relu else 2) + (pooled.numel() * y.element_size() if pool else 0)
    _run("vmb_percep_stage", y, "percep_stage", a, nbytes=nbytes)
    return pooled, code, saves


def percep_loss(partial, offsets, numels, weights, crit, perceptual_weight):
    """perceptual_weight * sum_k weights[k] crit_k from the features' partials (feature k at partial[offsets[k]:offsets[k + 1]])
    -> (0-dim fp32 loss, per-feature criterion values (fp32, the norms the fro backward divides by))"""
    n = len(weights)
    loss = torch.empty((), dtype=torch.float32, device=partial.device)
    value = torch.empty(n, dtype=torch.float32, device=partial.device)
    a = _lib.PercepLossArgs(partial=_ptr(partial), loss=_ptr(loss), value=_ptr(value),
                            offset=(C.c_int * (_lib.PERCEP_MAX_FEATS + 1))(*offsets),
                            numel=(C.c_int64 * _lib.PERCEP_MAX_FEATS)(*numels), weight=(C.c_float * _lib.PERCEP_MAX_FEATS)(*weights),
                            feats=n, crit=PERCEP_CRIT[crit], perceptual_weight=float(perceptual_weight))
    _run("vmb_percep_loss", partial, "percep_loss", a, nbytes=partial.numel() * 4)
    return loss, value


def percep_stage_bwd(g_in, code, saves, feat, feat_index, scale, grad_loss, value, shape, relu, pool, crit, dtype):
    """Gradient at a stage's conv output, x half (B, C, H, W) = `shape`, from the gradient g_in at its output (None at the deepest
    stage) and the saved state of percep_stage; the loss terms' factors are grad_loss (device scalar) * scale[k]"""
    dev = grad_loss.device
    g_out = torch.empty(shape, dtype=dtype, device=dev)
    B, Cc, H, W = shape
    a = _lib.PercepStageBwdArgs(g_in=_ptr(g_in), g_out=_ptr(g_out), code=_ptr(code),
                                save=(C.c_void_p * 3)(*[0 if s is None else s.data_ptr() for s in saves]), grad_loss=_ptr(grad_loss),
                                value=_ptr(value), feat=(C.c_int * 3)(*map(int, feat)), feat_index=(C.c_int * 3)(*feat_index),
                                scale=(C.c_float * 3)(*scale), B=B, C=Cc, H=H, W=W, relu=int(relu), pool=int(pool),
                                crit=PERCEP_CRIT[crit], dtype=_gan_dt(g_out))
    nbytes = g_out.numel() * g_out.element_size() + (g_in.numel() * g_in.element_size() if g_in is not None else 0)
    _run("vmb_percep_stage_bwd", grad_loss, "percep_stage_bwd", a, nbytes=nbytes)
    return g_out


# ---- perceptual metrics (csrc/percep_metrics.cu): LPIPS (VGG) and DISTS between the VGG16 convolutions; the two images of each
# pair as one 2B batch, fp32 activations, contiguous; every reduction in a fixed order, nothing read on the host ----
PMETRIC = {"lpips": _lib.PMETRIC_LPIPS, "dists": _lib.PMETRIC_DISTS}


def pmetric_src(t, offset, strides):
    """vmb_pmetric_src of the (B, 3, H, W) view (RGB channel order) of CUDA tensor t's storage that starts `offset` elements after
    t.data_ptr(), element strides (b, c, h, w); t is float32 or uint8"""
    if t.dtype not in (torch.float32, torch.uint8):
        raise RuntimeError(f"perceptual metrics: source dtype {t.dtype} is not float32 or uint8")
    return _lib.PmetricSrc(data=C.c_void_p(t.data_ptr() + offset * t.element_size()), stride=(C.c_int64 * 4)(*strides),
                           u8=int(t.dtype == torch.uint8))


def pmetric_tiles(planes, items):
    """CTAs per plane of the statistics kernels (vmb_pmetric_tiles)"""
    return _lib.lib().vmb_pmetric_tiles(planes, items)


def pmetric_prep(t, src0, src1, B, H, W, metric, shift, scale, normalize=False, stats=None):
    """-> (2B, 3, H, W) fp32: [prep(src0); prep(src1)] for `metric` ('lpips' or 'dists'); shift, scale: the (1, 3, 1, 1) fp32
    buffers; stats: DISTS's fp64 layer-0 statistics buffer, or None.  t: a tensor on the sources' device (stream and count)."""
    out = torch.empty((2 * B, 3, H, W), dtype=torch.float32, device=t.device)
    a = _lib.PmetricPrepArgs(src=(_lib.PmetricSrc * 2)(src0, src1), shift=_ptr(shift), scale=_ptr(scale), out=_ptr(out),
                             stats=_ptr(stats), B=B, H=H, W=W, metric=PMETRIC[metric], normalize=int(normalize))
    _run("vmb_pmetric_prep", t, "pmetric_prep", a, nbytes=2 * B * 3 * H * W * (t.element_size() + 4))
    return out


def lpips_layer_ctas(B, H, W):
    """CTAs per image of vmb_lpips_layer at this shape: its partials per image"""
    return _lib.lib().vmb_lpips_layer_ctas(B, H, W)


def lpips_layer(y, w, partial):
    """LPIPS's per-CTA partials of one feature layer into `partial` (B * lpips_layer_ctas): y (2B, C, H, W) the conv output before
    the ReLU, w the (1, C, 1, 1) lin weight"""
    B2, Cc, H, W = y.shape
    a = _lib.LpipsLayerArgs(y=_ptr(y), w=_ptr(w), partial=_ptr(partial), B=B2 // 2, C=Cc, H=H, W=W)
    _run("vmb_lpips_layer", y, "lpips_layer", a, nbytes=y.numel() * 4)


def lpips_final(partial, offsets, ctas, hws, B):
    """-> (val (B,), per-layer values (layers, B)), fp32: each layer's partials added in order, / H W, summed over the layers"""
    n = len(ctas)
    layer = torch.empty((n + 1, B), dtype=torch.float32, device=partial.device)
    L = _lib.PMETRIC_MAX_LAYERS
    a = _lib.LpipsFinalArgs(partial=_ptr(partial), layer=_ptr(layer), out=_ptr(layer[n]), offset=(C.c_int * L)(*offsets),
                            ctas=(C.c_int * L)(*ctas), hw=(C.c_int64 * L)(*hws), B=B, layers=n)
    _run("vmb_lpips_final", partial, "lpips_final", a, nbytes=partial.numel() * 4)
    return layer[n], layer[:n]


def dists_layer(y, stats, pool):
    """DISTS's fp64 statistics of one feature layer into `stats`, and with `pool` -> the L2-pooled (2B, C, ceil(H/2), ceil(W/2))
    input of the next convolution (else None); y (2B, C, H, W) the conv output before the ReLU"""
    B2, Cc, H, W = y.shape
    pooled = torch.empty((B2, Cc, (H + 1) // 2, (W + 1) // 2), dtype=torch.float32, device=y.device) if pool else None
    a = _lib.DistsLayerArgs(y=_ptr(y), pooled=_ptr(pooled), stats=_ptr(stats), B=B2 // 2, C=Cc, H=H, W=W)
    _run("vmb_dists_layer", y, "dists_layer", a, nbytes=y.numel() * 4 + (pooled.numel() * 4 if pool else 0))
    return pooled


def dists_final(stats, alpha, beta, offsets, channels, tiles, ns, B, batch_average):
    """-> the (B,) fp32 scores, and with batch_average their mean (0-dim) as well (else None)"""
    score = torch.empty(B + 1, dtype=torch.float32, device=stats.device)
    L = _lib.PMETRIC_MAX_LAYERS
    a = _lib.DistsFinalArgs(stats=_ptr(stats), alpha=_ptr(alpha), beta=_ptr(beta), score=_ptr(score),
                            mean=_ptr(score[B]) if batch_average else None, offset=(C.c_int64 * L)(*offsets), n=(C.c_int64 * L)(*ns),
                            C=(C.c_int * L)(*channels), tiles=(C.c_int * L)(*tiles), B=B, layers=len(channels))
    _run("vmb_dists_final", stats, "dists_final", a, nbytes=stats.numel() * 8)
    return score[:B], (score[B] if batch_average else None)
