"""Four-direction 2-D selective scan as a differentiable operator: `cross_selective_scan`, `CrossScan`, `CrossMerge`; and the
two-direction channel scan next to it: `cross_selective_scanC`, `CrossScanC`, `CrossMergeC` (at the end of this module).

Reference: RealSR/VmambaIR/archs/MambaRealSR11_arch.py:325-434 (CrossScan, CrossMerge, cross_selective_scan), called by
SS2D_1.forward_corev2 (:791-804) and by VMamba-style code directly.

`cross_selective_scan` runs x -> merged fp32 y on this library's kernels in one autograd Function, without the four gathered
(B, 4, D, L) copies of u, delta, B and C that the reference builds in both directions:

    forward   vmb_transpose_hw (x^T) -> vmb_pixlin on x (directions 0/2) and on x^T (directions 1/3), x_proj and dt_proj folded into
              one matrix per direction -> vmb_selective_scan_fwd_grouped with checkpoints (directions 2/3 walk backwards inside the
              kernel) -> vmb_merge_sum (four-way fp32 sum in pixel order)
    backward  vmb_transpose_hw (dy^T) -> vmb_selective_scan_bwd_grouped (du, ddelta, dB, dC of every direction in its source's
              memory order) -> vmb_pixlin with the transposed folded weights (x_proj data gradients, added to du0 / du1 in the
              epilogue) -> vmb_merge_sum (dx = du0 + du2 + T(du1 + du3) + the x_proj data gradients) -> vmb_pixlin_wgrad (weight and
              bias gradients of the folded matrices, unfolded as fused_train._Front does)

Shapes the grouped kernels reject (16-bit I/O with H*W % 8 != 0, fp32 with H*W % 4 != 0, d_state > 16, odd D) take the gathered path
inside the same Function: vmb_cross_scan, the flat vmb_selective_scan_fwd / _bwd and the inverse gathers, as fused.py does at inference.
`out_norm` is applied afterwards by calling the module the caller passed, as the reference does.
"""
from __future__ import annotations

import torch

from . import ops

_DTYPES = (torch.float32, torch.bfloat16, torch.float16)


def _check_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("cross_selective_scan: every tensor must be a CUDA tensor")


def grouped_supported(D, L, N, dtype) -> bool:
    """True when the direction-aware kernels take (D, L = H*W, N, dtype): 16 B-aligned rows, d_state <= 16, an even row count."""
    v = 4 if dtype == torch.float32 else 8
    return L % v == 0 and N <= 16 and D % 2 == 0


def _fold(x_proj_weight, x_proj_bias, dt_projs_weight, D, R):
    """-> big (4, D+2N, D) = [W_dt,k W_x,k[:R] ; W_x,k[R:]] and bias (4, D+2N) = [W_dt,k b_k[:R] ; b_k[R:]] (or None), fp32"""
    xw, dtw = x_proj_weight.detach().float(), dt_projs_weight.detach().float()
    big = torch.cat([torch.bmm(dtw, xw[:, :R]), xw[:, R:]], 1)
    bias = None
    if x_proj_bias is not None:
        xb = x_proj_bias.detach().float()
        bias = torch.cat([torch.bmm(dtw, xb[:, :R, None])[..., 0], xb[:, R:]], 1)
    return big, bias


def _wT(w, dtype):
    """(M, K) fp32 -> the transposed weight (K, ceil16(M)) in `dtype` for the data-gradient GEMM"""
    return ops.pad_weight(w.t().to(dtype))


class _CrossSelectiveScan(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, delta_softplus):
        B, D, H, W = x.shape
        L = H * W
        K, _, R = dt_projs_weight.shape
        N = A_logs.shape[1]
        dt_ = x.dtype
        RN = D + 2 * N
        big, bias = _fold(x_proj_weight, x_proj_bias, dt_projs_weight, D, R)  # (4, RN, D), (4, RN)
        A = (-torch.exp(A_logs.detach().float())).contiguous()
        Df = Ds.detach().float().contiguous()
        dtb = dt_projs_bias.detach().float().reshape(-1).contiguous()
        xc = x.detach().contiguous().view(B, D, L)
        grouped = grouped_supported(D, L, N, dt_)
        if grouped:
            xt = ops.transpose_hw(xc, H, W)  # the (W,H)-ordered copy that directions 1 and 3 scan
            w02, w13 = big[0::2].reshape(2 * RN, D), big[1::2].reshape(2 * RN, D)
            b02 = bias[0::2].reshape(-1).contiguous() if bias is not None else None
            b13 = bias[1::2].reshape(-1).contiguous() if bias is not None else None
            d02 = ops.pixlin(xc, ops.pad_weight(w02.to(dt_)), b02).view(B, 2, RN, L)
            d13 = ops.pixlin(xt, ops.pad_weight(w13.to(dt_)), b13).view(B, 2, RN, L)
            src = [(xc, d02[:, 0]), (xt, d13[:, 0]), (xc, d02[:, 1]), (xt, d13[:, 1])]
            ys, ckpt = ops.selective_scan_fwd_grouped([s[0] for s in src], [s[1][:, :D] for s in src], [s[1][:, D:D + N] for s in src],
                                                      [s[1][:, D + N:] for s in src], [0, 0, 1, 1], A, Df, dtb, delta_softplus,
                                                      need_ckpt=True)
            y = ops.merge_sum(ys, D, H, W, in_place_order=True)
            ctx.save_for_backward(xc, xt, d02, d13, ckpt, A, Df, dtb, big, bias, x_proj_weight, dt_projs_weight, x_proj_bias)
        else:
            dbl4 = ops.pixlin(xc, ops.pad_weight(big.reshape(4 * RN, D).to(dt_)),
                              bias.reshape(-1).contiguous() if bias is not None else None).view(B, 4, RN, L)
            xs, dts, bc = ops.cross_scan_multi([([xc] * 4, D, None), ([dbl4[:, k, :D] for k in range(4)], D, None),
                                                ([dbl4[:, k, D:] for k in range(4)], 2 * N, None)], H, W)
            ys, ckpt = ops.selective_scan_fwd(xs.view(B, 4 * D, L), dts.view(B, 4 * D, L), A, bc[:, :, :N], bc[:, :, N:], Df, dtb,
                                              delta_softplus, need_ckpt=True)
            y = ops.merge_sum(ys.view(B, 4, D, L), D, H, W)
            ctx.save_for_backward(xc, xs, dts, bc, ckpt, A, Df, dtb, big, bias, x_proj_weight, dt_projs_weight, x_proj_bias)
        ctx.geom = (B, D, H, W, N, R, grouped, bool(delta_softplus))
        ctx.param_meta = {k: (t.shape, t.dtype) for k, t in (("xw", x_proj_weight), ("xb", x_proj_bias), ("dtw", dt_projs_weight),
                                                             ("dtb", dt_projs_bias), ("A_logs", A_logs), ("Ds", Ds)) if t is not None}
        return y.view(B, D, H, W)

    @staticmethod
    def backward(ctx, dy):
        B, D, H, W, N, R, grouped, softplus = ctx.geom
        L, RN = H * W, D + 2 * N
        if grouped:
            xc, xt, d02, d13, ckpt, A, Df, dtb, big, bias, x_proj_weight, dt_projs_weight, x_proj_bias = ctx.saved_tensors
        else:
            xc, xs, dts, bc, ckpt, A, Df, dtb, big, bias, x_proj_weight, dt_projs_weight, x_proj_bias = ctx.saved_tensors
        dt_, dev = xc.dtype, xc.device
        dm = dy.to(dt_).contiguous().view(B, D, L)  # gradient of every direction's scan output (the merge is a plain sum)
        if grouped:
            dmt = ops.transpose_hw(dm, H, W)
            # du / ddelta / dB / dC straight into the buffers the next kernels read: S holds du2, du3 and (after the epilogue adds)
            # du0 + x_proj grad (0/2), du1 + x_proj grad (1/3); P holds du0, du1 until then; ddbl02 / ddbl13 the x_proj output grads
            S = torch.empty((B, 4, D, L), dtype=dt_, device=dev)
            P = torch.empty((B, 4, D, L), dtype=dt_, device=dev)
            ddbl02 = torch.empty((B, 2, RN, L), dtype=dt_, device=dev)
            ddbl13 = torch.empty((B, 2, RN, L), dtype=dt_, device=dev)
            dst = [ddbl02[:, 0], ddbl13[:, 0], ddbl02[:, 1], ddbl13[:, 1]]
            src = [(xc, d02[:, 0]), (xt, d13[:, 0]), (xc, d02[:, 1]), (xt, d13[:, 1])]
            _, _, dA, _, _, dD, dbias = ops.selective_scan_bwd_grouped(
                [s[0] for s in src], [s[1][:, :D] for s in src], [s[1][:, D:D + N] for s in src], [s[1][:, D + N:] for s in src],
                [dm, dmt, dm, dmt], [0, 0, 1, 1], A, Df, dtb, ckpt, softplus,
                out=([P[:, 0], P[:, 1], S[:, 2], S[:, 3]], [t[:, :D] for t in dst], [t[:, D:D + N] for t in dst],
                     [t[:, D + N:] for t in dst]))
            w02, w13 = big[0::2].reshape(2 * RN, D), big[1::2].reshape(2 * RN, D)
            ops.pixlin(ddbl02.view(B, 2 * RN, L), _wT(w02, dt_), residual=P[:, 0], out=S[:, 0])
            ops.pixlin(ddbl13.view(B, 2 * RN, L), _wT(w13, dt_), residual=P[:, 1], out=S[:, 1])
            dx = ops.merge_sum(S, D, H, W, in_place_order=True)  # du0 + du2 + T(du1 + du3) + both x_proj data gradients
            dbias02 = torch.zeros(2 * RN, dtype=torch.float32, device=dev) if x_proj_bias is not None else None
            dbias13 = torch.zeros(2 * RN, dtype=torch.float32, device=dev) if x_proj_bias is not None else None
            g02 = ops.pixlin_wgrad(ddbl02.view(B, 2 * RN, L), xc, dbias=dbias02).view(2, RN, D)
            g13 = ops.pixlin_wgrad(ddbl13.view(B, 2 * RN, L), xt, dbias=dbias13).view(2, RN, D)
            dbig = torch.stack([g02[0], g13[0], g02[1], g13[1]], 0)  # (4, RN, D), direction order
            dbb = None
            if x_proj_bias is not None:
                b02, b13 = dbias02.view(2, RN), dbias13.view(2, RN)
                dbb = torch.stack([b02[0], b13[0], b02[1], b13[1]], 0)
        else:
            dys = ops.cross_scan([dm] * 4, D, H, W)
            du, ddelta, dA, dB, dC, dD, dbias = ops.selective_scan_bwd(
                xs.view(B, 4 * D, L), dts.view(B, 4 * D, L), A, bc[:, :, :N], bc[:, :, N:], Df, dtb, dys.view(B, 4 * D, L), ckpt, softplus)
            ddbl = torch.empty((B, 4, RN, L), dtype=dt_, device=dev)
            dxc4 = ops.cross_scan_multi([([du.view(B, 4, D, L)[:, k] for k in range(4)], D, None),
                                         ([ddelta.view(B, 4, D, L)[:, k] for k in range(4)], D, ddbl[:, :, :D]),
                                         ([dB[:, k] for k in range(4)], N, ddbl[:, :, D:D + N]),
                                         ([dC[:, k] for k in range(4)], N, ddbl[:, :, D + N:])], W, H)[0]  # inverse orders
            ddbl = ddbl.view(B, 4 * RN, L)
            dx = ops.sum4_add(dxc4, ops.pixlin(ddbl, _wT(big.reshape(4 * RN, D), dt_)))
            dbb = torch.zeros(4 * RN, dtype=torch.float32, device=dev) if x_proj_bias is not None else None
            dbig = ops.pixlin_wgrad(ddbl, xc, dbias=dbb).view(4, RN, D)
            dbb = dbb.view(4, RN) if dbb is not None else None
        # unfold big_k = [W_dt,k W_x,k[:R] ; W_x,k[R:]] and bias_k = [W_dt,k b_k[:R] ; b_k[R:]]
        xw, dtw = x_proj_weight.detach().float(), dt_projs_weight.detach().float()
        d_xproj = torch.cat([torch.bmm(dtw.transpose(1, 2), dbig[:, :D]), dbig[:, D:]], 1)
        d_dtw = torch.bmm(dbig[:, :D], xw[:, :R].transpose(1, 2))
        d_xb = None
        if x_proj_bias is not None:
            xb = x_proj_bias.detach().float()
            d_xb = torch.cat([torch.bmm(dtw.transpose(1, 2), dbb[:, :D, None])[..., 0], dbb[:, D:]], 1)
            d_dtw = d_dtw + dbb[:, :D, None] * xb[:, None, :R]
        dA_logs = dA * A  # A = -exp(A_logs)
        shp = ctx.param_meta
        cast = lambda g, k: None if g is None else g.to(shp[k][1]).view(shp[k][0])
        return (dx.view(B, D, H, W).to(dt_), cast(d_xproj, "xw"), cast(d_xb, "xb"), cast(d_dtw, "dtw"), cast(dbias, "dtb"),
                cast(dA_logs, "A_logs"), cast(dD, "Ds"), None)


class CrossScan(torch.autograd.Function):
    """x (B,C,H,W) -> xs (B,4,C,H*W): row-major, column-major and both reversed (reference :325-343).  Forward: vmb_cross_scan
    (bit-exact gather).  Backward: the inverse gathers and their sum, i.e. CrossMerge's forward (vmb_merge_sum, fp32 accumulation,
    any H, W)."""

    @staticmethod
    def forward(ctx, x):
        _check_cuda(x)
        B, C, H, W = x.shape
        ctx.shape = (B, C, H, W)
        xc = x.contiguous().view(B, C, H * W)
        return ops.cross_scan([xc] * 4, C, H, W)

    @staticmethod
    def backward(ctx, ys):
        B, C, H, W = ctx.shape
        return ops.merge_sum(ys.contiguous(), C, H, W).to(ys.dtype).view(B, C, H, W)


class CrossMerge(torch.autograd.Function):
    """ys (B,4,D,H,W) in scan order -> y (B,D,H*W): the four directions summed in pixel order (reference :346-368).  Forward:
    vmb_merge_sum (fp32 accumulation, result in the input dtype).  Backward: vmb_cross_scan of the gradient (the four gathers)."""

    @staticmethod
    def forward(ctx, ys):
        _check_cuda(ys)
        B, K, D, H, W = ys.shape
        ctx.shape = (H, W)
        y = ops.merge_sum(ys.contiguous().view(B, K, D, H * W), D, H, W)
        return y.to(ys.dtype)

    @staticmethod
    def backward(ctx, dy):
        H, W = ctx.shape
        B, D, L = dy.shape
        dy = dy.contiguous()
        return ops.cross_scan([dy] * 4, D, H, W).view(B, 4, D, H, W)


def cross_selective_scan(x: torch.Tensor = None, x_proj_weight: torch.Tensor = None, x_proj_bias: torch.Tensor = None,
                         dt_projs_weight: torch.Tensor = None, dt_projs_bias: torch.Tensor = None, A_logs: torch.Tensor = None,
                         Ds: torch.Tensor = None, out_norm: torch.nn.Module = None, softmax_version=False, nrows=-1,
                         delta_softplus=True, to_dtype=True):
    """Drop-in for the reference's cross_selective_scan (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:371-434): same signature, shapes
    and result.  x (B,D,H,W); x_proj_weight (4, R+2N, D); x_proj_bias (4, R+2N) or None; dt_projs_weight (4, D, R); dt_projs_bias (4, D);
    A_logs (4D, N); Ds (4D); out_norm: the module applied to the merged (B,D,H,W) fp32 output.  -> out_norm(y), cast to x.dtype when
    to_dtype.  Differentiable w.r.t. x and every parameter.

    dtype rule (deviation from the reference): the scan operands stay in x's dtype -- fp32 in parity mode, 16-bit I/O with fp32 state
    and accumulation otherwise -- while the reference casts them to fp32; as for selective_scan_fn, 16-bit results therefore match the
    reference within bf16 / fp16 rounding of u, delta, B and C.  x_proj and dt_proj are applied as one folded matrix W_dt W_x[:R]
    (fp32 product, cast to x's dtype), so even fp32 results differ from the reference's two einsums in rounding only.
    softmax_version=True raises NotImplementedError (as SS2D_1 does); nrows is accepted and ignored (the kernels pick their own
    rows per warp, as selective_scan_cuda_core does).
    Under torch.use_deterministic_algorithms(True) the scan backward and the x_proj / dt_proj weight gradients (vmb_pixlin_wgrad) run
    the library's deterministic kernels, so the gradients are bitwise reproducible; the weight unfold's torch matmuls then need
    CUBLAS_WORKSPACE_CONFIG=:4096:8 (or :16:8), as torch requires for cuBLAS under that flag."""
    if softmax_version:
        raise NotImplementedError("cross_selective_scan: softmax_version is not supported")
    _check_cuda(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds)
    if x.dtype not in _DTYPES:
        raise RuntimeError(f"cross_selective_scan: x dtype must be float32/float16/bfloat16, got {x.dtype}")
    B, D, H, W = x.shape
    K, D2, R = dt_projs_weight.shape
    N = A_logs.shape[1]
    if K != 4 or D2 != D or tuple(x_proj_weight.shape) != (4, R + 2 * N, D) or tuple(A_logs.shape) != (4 * D, N) \
            or Ds.numel() != 4 * D or dt_projs_bias.numel() != 4 * D or (x_proj_bias is not None and x_proj_bias.numel() != 4 * (R + 2 * N)):
        raise RuntimeError("cross_selective_scan: expected x (B,D,H,W), x_proj_weight (4,R+2N,D), dt_projs_weight (4,D,R), "
                           "dt_projs_bias (4,D), A_logs (4D,N), Ds (4D)")
    with torch.autocast("cuda", enabled=False):
        y = _CrossSelectiveScan.apply(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, bool(delta_softplus))
    y = out_norm(y)
    if to_dtype:
        y = y.to(x.dtype)
    return y


# ----------------------------------------------------------------------------- the two-direction channel scan
# Reference: RealSR/VmambaIR/archs/MambaRealSR11_arch.py:438-534 (CrossScanC, CrossMergeC, cross_selective_scanC), called by
# SS2D_1.cforward_corev2 (:806-817) on the pooled (B, 1, C) descriptor.
#
#   forward   vmb_cross_selective_scan_c_fwd: one CTA per image loads x once and runs both projections, softplus, both scan
#             directions and the merge in fp32 shared memory -> y (B, L, 1, D) fp32
#   backward  vmb_cross_selective_scan_c_bwd: one CTA per image recomputes the forward, walks the recurrence backwards and writes dx
#             and its own parameter gradients; a second kernel sums those over the batch in a fixed order (bitwise reproducible)
#
# Shapes the kernels reject (cross_scan_c_supported: d_state > 16, D > 16, or a state history beyond one CTA's shared memory) take
# the composed path inside the same Function: fp32 torch einsums around the flat vmb_selective_scan_fwd / _bwd.


class CrossScanC(torch.autograd.Function):
    """x (B,D,L) -> xs (B,2,D,L) = [x, flip_L x] (reference :438-456).  Backward: ys[:,0] + flip_L ys[:,1], i.e. CrossMergeC's
    forward.  Plain torch indexing: the fused operator does not use it."""

    @staticmethod
    def forward(ctx, x):
        B, D, L = x.shape
        xs = x.new_empty((B, 2, D, L))
        xs[:, 0] = x
        xs[:, 1] = torch.flip(x, dims=[-1])
        return xs

    @staticmethod
    def backward(ctx, ys):
        return ys[:, 0] + ys[:, 1].flip(dims=[-1])


class CrossMergeC(torch.autograd.Function):
    """ys (B,2,D,L) -> ys[:,0] + flip_L ys[:,1] (reference :459-475).  Backward: [g, flip_L g], i.e. CrossScanC's forward."""

    @staticmethod
    def forward(ctx, ys):
        return ys[:, 0] + ys[:, 1].flip(dims=[-1])

    @staticmethod
    def backward(ctx, g):
        B, D, L = g.shape
        xs = g.new_empty((B, 2, D, L))
        xs[:, 0] = g
        xs[:, 1] = torch.flip(g, dims=[-1])
        return xs


def _csc_composed_fwd(x, xw, xb, dtw, dtb, A, Df, softplus):
    """fp32 composition for shapes the kernels reject -> (y (B, L, D), saved tensors)"""
    B, D, L = x.shape
    N = A.shape[1]
    R = xw.shape[1] - 2 * N
    xf = x.float()
    xs = torch.stack([xf, xf.flip(-1)], 1)  # (B, 2, D, L)
    dbl = torch.einsum("bkdl,kcd->bkcl", xs, xw)
    if xb is not None:
        dbl = dbl + xb.view(1, 2, -1, 1)
    dtr, Bs, Cs = dbl[:, :, :R], dbl[:, :, R:R + N].contiguous(), dbl[:, :, R + N:].contiguous()
    dts = torch.einsum("bkrl,kdr->bkdl", dtr, dtw).reshape(B, 2 * D, L).contiguous()
    u = xs.view(B, 2 * D, L)
    ys, ckpt = ops.selective_scan_fwd(u, dts, A, Bs, Cs, Df, dtb, softplus, need_ckpt=True)
    ys = ys.view(B, 2, D, L)
    y = (ys[:, 0] + ys[:, 1].flip(-1)).transpose(1, 2).contiguous()
    return y, (u, dtr.contiguous(), dts, Bs, Cs, ckpt)


def _csc_composed_bwd(saved, dy, xw, dtw, A, Df, dtb, softplus, has_bias):
    u, dtr, dts, Bs, Cs, ckpt = saved
    B, D2, L = u.shape
    D = D2 // 2
    dm = dy.transpose(1, 2)  # (B, D, L)
    dys = torch.stack([dm, dm.flip(-1)], 1).reshape(B, 2 * D, L).contiguous()
    du, ddelta, dA, dB, dC, dD, dbias = ops.selective_scan_bwd(u, dts, A, Bs, Cs, Df, dtb, dys, ckpt, softplus)
    dd = ddelta.view(B, 2, D, L)
    d_dtw = torch.einsum("bkdl,bkrl->kdr", dd, dtr)
    ddbl = torch.cat([torch.einsum("bkdl,kdr->bkrl", dd, dtw), dB, dC], 2)  # (B, 2, R+2N, L)
    xs = u.view(B, 2, D, L)
    d_xw = torch.einsum("bkcl,bkdl->kcd", ddbl, xs)
    d_xb = ddbl.sum((0, 3)) if has_bias else None
    dxs = du.view(B, 2, D, L) + torch.einsum("bkcl,kcd->bkdl", ddbl, xw)
    dx = dxs[:, 0] + dxs[:, 1].flip(-1)
    g = {"x_proj_weight": d_xw, "dt_projs_weight": d_dtw, "dt_projs_bias": dbias, "A_logs": dA * A, "Ds": dD}
    if has_bias:
        g["x_proj_bias"] = d_xb
    return dx, g


class _CrossSelectiveScanC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, delta_softplus):
        B, D, L = x.shape
        N = A_logs.shape[1]
        R = x_proj_weight.shape[1] - 2 * N
        f32 = lambda t: None if t is None else t.detach().float().contiguous()
        xw, dtw, A_logs32 = f32(x_proj_weight), f32(dt_projs_weight), f32(A_logs)
        xb = f32(x_proj_bias).view(2, -1) if x_proj_bias is not None else None
        dtb, Df = f32(dt_projs_bias).view(-1), f32(Ds).view(-1)
        fused = ops.cross_scan_c_supported(D, L, R, N)
        xd = x.detach()
        if xd.stride(-1) != 1:
            xd = xd.contiguous()
        if fused:
            y = ops.cross_selective_scan_c_fwd(xd, xw, xb, dtw, dtb, A_logs32, Df, delta_softplus)
            ctx.save_for_backward(xd, xw, xb, dtw, dtb, A_logs32, Df)
        else:
            A = (-torch.exp(A_logs32)).contiguous()
            y, saved = _csc_composed_fwd(xd, xw, xb, dtw, dtb, A, Df, delta_softplus)
            ctx.save_for_backward(xw, dtw, dtb, A, Df, *saved)
        ctx.geom = (B, D, L, fused, bool(delta_softplus), x.dtype, x_proj_bias is not None)
        ctx.param_meta = {k: (t.shape, t.dtype) for k, t in (("x_proj_weight", x_proj_weight), ("x_proj_bias", x_proj_bias),
                                                             ("dt_projs_weight", dt_projs_weight), ("dt_projs_bias", dt_projs_bias),
                                                             ("A_logs", A_logs), ("Ds", Ds)) if t is not None}
        return y.view(B, L, 1, D)

    @staticmethod
    def backward(ctx, dy):
        B, D, L, fused, softplus, x_dtype, has_bias = ctx.geom
        dy = dy.float().contiguous().view(B, L, D)
        if fused:
            xd, xw, xb, dtw, dtb, A_logs32, Df = ctx.saved_tensors
            dx, g = ops.cross_selective_scan_c_bwd(xd, xw, xb, dtw, dtb, A_logs32, Df, dy, softplus)
        else:
            xw, dtw, dtb, A, Df, *saved = ctx.saved_tensors
            dx, g = _csc_composed_bwd(saved, dy, xw, dtw, A, Df, dtb, softplus, has_bias)
        meta = ctx.param_meta
        cast = lambda k: g[k].to(meta[k][1]).view(meta[k][0]) if k in meta else None
        return (dx.to(x_dtype), cast("x_proj_weight"), cast("x_proj_bias"), cast("dt_projs_weight"), cast("dt_projs_bias"),
                cast("A_logs"), cast("Ds"), None)


def cross_selective_scanC(x: torch.Tensor = None, x_proj_weight: torch.Tensor = None, x_proj_bias: torch.Tensor = None,
                          dt_projs_weight: torch.Tensor = None, dt_projs_bias: torch.Tensor = None, A_logs: torch.Tensor = None,
                          Ds: torch.Tensor = None, out_norm: torch.nn.Module = None, softmax_version=False, nrows=-1,
                          delta_softplus=True, to_dtype=True):
    """Drop-in for the reference's cross_selective_scanC (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:478-534): same signature, shapes
    and result.  x (B,D,L) fp32 / bf16 / fp16 (SS2D_1 passes the pooled (B, 1, C) descriptor: D = 1, L = C); x_proj_weight
    (2, R+2N, D); x_proj_bias (2, R+2N) or None; dt_projs_weight (2, D, R); dt_projs_bias (2, D); A_logs (2D, N); Ds (2D); out_norm:
    the module applied to the merged y (B, L, 1, D) fp32.  -> out_norm(y), cast to x.dtype when to_dtype.  Differentiable w.r.t. x
    and every parameter; gradients come back in each parameter's dtype, and are bitwise reproducible on the fused path.

    dtype rule: every operand is cast to fp32 and the scan runs in fp32, as the reference's SelectiveScan (custom_fwd with
    cast_inputs=float32) does.  The one difference: x_proj and dt_proj also run in fp32 here, where an autocast caller of the
    reference would run those two einsums in bf16.  softmax_version=True raises NotImplementedError; nrows is accepted and ignored."""
    if softmax_version:
        raise NotImplementedError("cross_selective_scanC: softmax_version is not supported")
    _check_cuda(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds)
    if x.dtype not in _DTYPES:
        raise RuntimeError(f"cross_selective_scanC: x dtype must be float32/float16/bfloat16, got {x.dtype}")
    if x.dim() != 3 or dt_projs_weight.dim() != 3 or A_logs.dim() != 2:
        raise RuntimeError("cross_selective_scanC: expected x (B,D,L), dt_projs_weight (2,D,R), A_logs (2D,N)")
    B, D, L = x.shape
    K, D2, R = dt_projs_weight.shape
    N = A_logs.shape[1]
    if K != 2 or D2 != D or tuple(x_proj_weight.shape) != (2, R + 2 * N, D) or tuple(A_logs.shape) != (2 * D, N) \
            or Ds.numel() != 2 * D or dt_projs_bias.numel() != 2 * D or (x_proj_bias is not None and x_proj_bias.numel() != 2 * (R + 2 * N)):
        raise RuntimeError("cross_selective_scanC: expected x (B,D,L), x_proj_weight (2,R+2N,D), x_proj_bias (2,R+2N), "
                           "dt_projs_weight (2,D,R), dt_projs_bias (2,D), A_logs (2D,N), Ds (2D)")
    with torch.autocast("cuda", enabled=False):
        y = _CrossSelectiveScanC.apply(x, x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds, bool(delta_softplus))
    y = out_norm(y)
    if to_dtype:
        y = y.to(x.dtype)
    return y
