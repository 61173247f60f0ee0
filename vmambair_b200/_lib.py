"""ctypes loader of the C-ABI library (include/vmambair_b200.h).

There is NO fallback: if the CUDA library is missing or a call fails, a RuntimeError is raised.

Each Structure mirrors the header typedef its `_c_name_` names, field for field; tests/test_abi_cpu.py compiles the header and checks
sizes, offsets and names against these mirrors.  Build them with keyword arguments only (that test rejects positional ones), so a
value can never land in the wrong field.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VMB_LIB_PATH") or os.path.join(_HERE, "lib", "libvmambair_b200.so")
_lib = None

DT_F32, DT_BF16, DT_F16 = 0, 1, 2

i64 = C.c_int64
vp = C.c_void_p


class ScanFwdArgs(C.Structure):
    _c_name_ = "vmb_scan_fwd_args"
    _fields_ = [
        ("u", vp), ("delta", vp), ("A", vp), ("Bm", vp), ("Cm", vp), ("D", vp), ("delta_bias", vp),
        ("out", vp), ("ckpt", vp),
        ("batch", C.c_int), ("dim", C.c_int), ("seqlen", C.c_int), ("dstate", C.c_int), ("ngroups", C.c_int),
        ("u_bs", i64), ("u_ds", i64), ("delta_bs", i64), ("delta_ds", i64), ("out_bs", i64), ("out_ds", i64),
        ("B_bs", i64), ("B_gs", i64), ("B_ns", i64), ("C_bs", i64), ("C_gs", i64), ("C_ns", i64),
        ("delta_softplus", C.c_int), ("dtype", C.c_int), ("out_f32", C.c_int),
        ("z", vp), ("out_z", vp), ("z_bs", i64), ("z_ds", i64), ("out_z_bs", i64), ("out_z_ds", i64), ("ckpt_pairs", C.c_int),
    ]


class ScanGateArgs(C.Structure):
    _c_name_ = "vmb_scan_gate_args"
    _fields_ = [
        ("dout", vp), ("out", vp), ("z", vp), ("dout_eff", vp), ("dz", vp), ("out_z", vp),
        ("batch", C.c_int), ("dim", C.c_int), ("seqlen", C.c_int),
        ("dout_bs", i64), ("dout_ds", i64), ("out_bs", i64), ("out_ds", i64), ("z_bs", i64), ("z_ds", i64),
        ("dz_bs", i64), ("dz_ds", i64), ("out_z_bs", i64), ("out_z_ds", i64), ("dtype", C.c_int),
    ]


class ScanBwdArgs(C.Structure):
    _c_name_ = "vmb_scan_bwd_args"
    _fields_ = [
        ("u", vp), ("delta", vp), ("A", vp), ("Bm", vp), ("Cm", vp), ("D", vp), ("delta_bias", vp),
        ("dout", vp), ("ckpt", vp),
        ("du", vp), ("ddelta", vp), ("dA", vp), ("dB", vp), ("dC", vp), ("dD", vp), ("ddelta_bias", vp), ("workspace", vp),
        ("batch", C.c_int), ("dim", C.c_int), ("seqlen", C.c_int), ("dstate", C.c_int), ("ngroups", C.c_int),
        ("u_bs", i64), ("u_ds", i64), ("delta_bs", i64), ("delta_ds", i64), ("dout_bs", i64), ("dout_ds", i64),
        ("du_bs", i64), ("du_ds", i64), ("ddelta_bs", i64), ("ddelta_ds", i64),
        ("B_bs", i64), ("B_gs", i64), ("B_ns", i64), ("C_bs", i64), ("C_gs", i64), ("C_ns", i64),
        ("delta_softplus", C.c_int), ("dtype", C.c_int), ("dout_f32", C.c_int), ("deterministic", C.c_int),
    ]


class PixlinArgs(C.Structure):
    _c_name_ = "vmb_pixlin_args"
    _fields_ = [
        ("x", vp), ("w", vp), ("bias", vp), ("residual", vp), ("out", vp), ("ln_w", vp), ("ln_b", vp), ("gate", vp),
        ("ln_mode", C.c_int), ("gate_mode", C.c_int), ("act_from", C.c_int), ("act_to", C.c_int),
        ("batch", C.c_int), ("K", C.c_int), ("M", C.c_int), ("P", C.c_int),
        ("x_bs", i64), ("x_cs", i64), ("r_bs", i64), ("r_cs", i64), ("o_bs", i64), ("o_cs", i64), ("g_bs", i64), ("w_ld", i64),
        ("dtype", C.c_int), ("out_dtype", C.c_int),
    ]


class DwconvArgs(C.Structure):
    _c_name_ = "vmb_dwconv_args"
    _fields_ = [
        ("x", vp), ("w", vp), ("bias", vp), ("out", vp),
        ("batch", C.c_int), ("c_out", C.c_int), ("H", C.c_int), ("W", C.c_int), ("mode", C.c_int),
        ("x_bs", i64), ("x_cs", i64), ("o_bs", i64), ("o_cs", i64), ("dtype", C.c_int),
    ]


class CrossScanArgs(C.Structure):
    _c_name_ = "vmb_cross_scan_args"
    _fields_ = [
        ("src", vp * 4), ("out", vp),
        ("batch", C.c_int), ("rows", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("src_bs", i64), ("src_rs", i64), ("out_bs", i64), ("dtype", C.c_int), ("out_ks", i64),
    ]


class MergeArgs(C.Structure):
    _c_name_ = "vmb_merge_args"
    _fields_ = [
        ("ys", vp), ("z", vp), ("ln_w", vp), ("ln_b", vp), ("y2", vp), ("pooled", vp),
        ("batch", C.c_int), ("C", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("z_bs", i64), ("z_cs", i64), ("dtype", C.c_int), ("workspace", vp), ("in_place_order", C.c_int),
        ("z_preact", C.c_int), ("save_ws", C.c_int),
    ]


class TransposeArgs(C.Structure):
    _c_name_ = "vmb_transpose_args"
    _fields_ = [("x", vp), ("out", vp), ("planes", C.c_int), ("H", C.c_int), ("W", C.c_int), ("dtype", C.c_int)]


class PixelShuffleArgs(C.Structure):
    _c_name_ = "vmb_pixel_shuffle_args"
    _fields_ = [("x", vp), ("out", vp), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("C", C.c_int), ("dtype", C.c_int)]


class Conv3x3Args(C.Structure):
    _c_name_ = "vmb_conv3x3_args"
    _fields_ = [
        ("x", vp), ("w", vp), ("bias", vp), ("out", vp), ("add", vp),
        ("batch", C.c_int), ("Cin", C.c_int), ("Cout", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("in_nhwc", C.c_int), ("mode", C.c_int), ("add_scale", C.c_int),
        ("x_bs", i64), ("x_cs", i64), ("o_bs", i64), ("o_cs", i64), ("add_bs", i64), ("add_cs", i64),
        ("dtype", C.c_int),
    ]


class ScanGroupedArgs(C.Structure):
    _c_name_ = "vmb_scan_grouped_args"
    _fields_ = [
        ("u", vp * 4), ("delta", vp * 4), ("Bm", vp * 4), ("Cm", vp * 4), ("out", vp * 4), ("rev", C.c_int * 4),
        ("A", vp), ("D", vp), ("delta_bias", vp),
        ("batch", C.c_int), ("dim", C.c_int), ("seqlen", C.c_int), ("dstate", C.c_int), ("ngroups", C.c_int),
        ("u_bs", i64), ("u_ds", i64), ("delta_bs", i64), ("delta_ds", i64), ("out_bs", i64), ("out_ds", i64),
        ("B_bs", i64), ("B_ns", i64), ("C_bs", i64), ("C_ns", i64),
        ("delta_softplus", C.c_int), ("dtype", C.c_int), ("ckpt", vp),
    ]


class ScanGroupedBwdArgs(C.Structure):
    _c_name_ = "vmb_scan_grouped_bwd_args"
    _fields_ = [
        ("u", vp * 4), ("delta", vp * 4), ("Bm", vp * 4), ("Cm", vp * 4), ("dout", vp * 4),
        ("du", vp * 4), ("ddelta", vp * 4), ("dB", vp * 4), ("dC", vp * 4), ("rev", C.c_int * 4),
        ("A", vp), ("D", vp), ("delta_bias", vp), ("ckpt", vp),
        ("dA", vp), ("dD", vp), ("ddelta_bias", vp), ("workspace", vp),
        ("batch", C.c_int), ("dim", C.c_int), ("seqlen", C.c_int), ("dstate", C.c_int), ("ngroups", C.c_int),
        ("u_bs", i64), ("u_ds", i64), ("delta_bs", i64), ("delta_ds", i64), ("dout_bs", i64), ("dout_ds", i64),
        ("du_bs", i64), ("du_ds", i64), ("ddelta_bs", i64), ("ddelta_ds", i64),
        ("B_bs", i64), ("B_ns", i64), ("C_bs", i64), ("C_ns", i64), ("dB_bs", i64), ("dB_ns", i64), ("dC_bs", i64), ("dC_ns", i64),
        ("delta_softplus", C.c_int), ("dtype", C.c_int), ("deterministic", C.c_int),
    ]


class ChannelArgs(C.Structure):
    _c_name_ = "vmb_channel_args"
    _fields_ = [
        ("pooled", vp), ("inv_count", C.c_float),
        ("cin_w", vp), ("cin_b", vp), ("xc_proj", vp), ("dtc_w", vp), ("dtc_b", vp), ("Ac_logs", vp), ("Dsc", vp),
        ("cout_w", vp), ("cout_b", vp), ("cn_w", vp), ("cn_b", vp), ("c_out", vp),
        ("batch", C.c_int), ("C", C.c_int), ("dc", C.c_int), ("Rc", C.c_int), ("N", C.c_int),
    ]


class LnFwdArgs(C.Structure):
    _c_name_ = "vmb_ln_fwd_args"
    _fields_ = [("x", vp), ("w", vp), ("b", vp), ("y", vp), ("stats", vp),
                ("batch", C.c_int), ("C", C.c_int), ("L", C.c_int), ("mode", C.c_int),
                ("x_bs", i64), ("x_cs", i64), ("y_bs", i64), ("y_cs", i64), ("dtype", C.c_int)]


class LnBwdArgs(C.Structure):
    _c_name_ = "vmb_ln_bwd_args"
    _fields_ = [("x", vp), ("g", vp), ("add", vp), ("w", vp), ("dx", vp), ("dw", vp), ("db", vp), ("stats", vp),
                ("batch", C.c_int), ("C", C.c_int), ("L", C.c_int), ("mode", C.c_int),
                ("x_bs", i64), ("x_cs", i64), ("g_bs", i64), ("g_cs", i64), ("a_bs", i64), ("a_cs", i64),
                ("dx_bs", i64), ("dx_cs", i64), ("dtype", C.c_int)]


class MergeBwdArgs(C.Structure):
    _c_name_ = "vmb_merge_bwd_args"
    _fields_ = [("merged", vp), ("stats", vp), ("z", vp), ("dy2", vp), ("dpooled", vp), ("w", vp), ("b", vp),
                ("dm", vp), ("dz", vp), ("dw", vp), ("db", vp),
                ("batch", C.c_int), ("C", C.c_int), ("L", C.c_int),
                ("z_bs", i64), ("z_cs", i64), ("dz_bs", i64), ("dz_cs", i64), ("dtype", C.c_int)]


class DwconvBwdArgs(C.Structure):
    _c_name_ = "vmb_dwconv_bwd_args"
    _fields_ = [("x", vp), ("w", vp), ("bias", vp), ("g", vp), ("dv", vp), ("dw", vp), ("dbias", vp),
                ("batch", C.c_int), ("c_out", C.c_int), ("H", C.c_int), ("W", C.c_int), ("mode", C.c_int),
                ("x_bs", i64), ("x_cs", i64), ("g_bs", i64), ("g_cs", i64), ("dv_bs", i64), ("dv_cs", i64), ("dtype", C.c_int)]


class GateBwdArgs(C.Structure):
    _c_name_ = "vmb_gate_bwd_args"
    _fields_ = [("dyg", vp), ("y2", vp), ("gate", vp), ("dy2", vp), ("dgate", vp),
                ("batch", C.c_int), ("C", C.c_int), ("L", C.c_int), ("mode", C.c_int), ("dtype", C.c_int)]


class WgradArgs(C.Structure):
    _c_name_ = "vmb_wgrad_args"
    _fields_ = [("dy", vp), ("x", vp), ("out", vp), ("batch", C.c_int), ("M", C.c_int), ("K", C.c_int), ("L", C.c_int),
                ("dy_bs", i64), ("dy_cs", i64), ("x_bs", i64), ("x_cs", i64), ("per_batch", C.c_int), ("dtype", C.c_int),
                ("dbias", vp), ("workspace", vp), ("deterministic", C.c_int)]


class ChannelBwdArgs(C.Structure):
    _c_name_ = "vmb_channel_bwd_args"
    _fields_ = [("fwd", ChannelArgs), ("dc_out", vp), ("d_pooled", vp),
                ("d_cin_w", vp), ("d_cin_b", vp), ("d_xc_proj", vp), ("d_dtc_w", vp), ("d_dtc_b", vp), ("d_Ac_logs", vp), ("d_Dsc", vp),
                ("d_cout_w", vp), ("d_cout_b", vp), ("d_cn_w", vp), ("d_cn_b", vp), ("scratch", vp)]


class CrossScanCArgs(C.Structure):
    _c_name_ = "vmb_cross_scan_c_args"
    _fields_ = [("x", vp), ("x_proj_weight", vp), ("x_proj_bias", vp), ("dt_projs_weight", vp), ("dt_projs_bias", vp),
                ("A_logs", vp), ("Ds", vp), ("y", vp),
                ("batch", C.c_int), ("D", C.c_int), ("L", C.c_int), ("R", C.c_int), ("N", C.c_int),
                ("x_bs", i64), ("x_ds", i64), ("delta_softplus", C.c_int), ("dtype", C.c_int)]


class CrossScanCBwdArgs(C.Structure):
    _c_name_ = "vmb_cross_scan_c_bwd_args"
    _fields_ = [("fwd", CrossScanCArgs), ("dy", vp), ("dx", vp), ("d_params", vp), ("workspace", vp)]


class PrepJob(C.Structure):
    _c_name_ = "vmb_prep_job"
    _fields_ = [("src", vp), ("src2", vp), ("dst", vp), ("dst2", vp), ("type", C.c_int), ("M", C.c_int), ("K", C.c_int),
                ("N2", C.c_int), ("ld", C.c_int), ("ld2", C.c_int)]


class PrepArgs(C.Structure):
    _c_name_ = "vmb_prep_args"
    _fields_ = [("jobs", PrepJob * 16), ("njobs", C.c_int), ("dtype", C.c_int)]


class AdamArgs(C.Structure):
    _c_name_ = "vmb_adam_args"
    _fields_ = [("param", vp), ("grad", vp), ("exp_avg", vp), ("exp_avg_sq", vp), ("ema", vp), ("state", vp),
                ("n", C.c_long), ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float), ("decoupled_weight_decay", C.c_int),
                ("grad_scale", C.c_float), ("max_grad_norm", C.c_float), ("ema_decay", C.c_float), ("zero_grad", C.c_int),
                ("lr_dev", vp)]


class ImageMaxArgs(C.Structure):
    _c_name_ = "vmb_image_max_args"
    _fields_ = [("img", vp), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int), ("u16", C.c_int),
                ("row_stride", i64), ("pixel_stride", i64), ("channel_stride", i64), ("max_out", vp)]


class ImageToPlanesArgs(C.Structure):
    _c_name_ = "vmb_image_to_planes_args"
    _fields_ = [("img", vp), ("out", vp), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int), ("u16", C.c_int),
                ("row_stride", i64), ("pixel_stride", i64), ("channel_stride", i64), ("max_range", C.c_float),
                ("pad_h", C.c_int * 3), ("pad_w", C.c_int * 3), ("alpha_plane", C.c_int), ("dtype", C.c_int)]


class PlanesToImageArgs(C.Structure):
    _c_name_ = "vmb_planes_to_image_args"
    _fields_ = [("planes", vp), ("out", vp), ("alpha_src", vp), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int), ("u16", C.c_int),
                ("p_bs", i64), ("p_cs", i64), ("p_rs", i64), ("out_rs", i64), ("out_ps", i64),
                ("alpha_mode", C.c_int), ("alpha_H", C.c_int), ("alpha_W", C.c_int), ("alpha_u16", C.c_int),
                ("alpha_rs", i64), ("alpha_ps", i64), ("max_range", C.c_float), ("dtype", C.c_int)]


class ResizeLanczos4Args(C.Structure):
    _c_name_ = "vmb_resize_lanczos4_args"
    _fields_ = [("src", vp), ("dst", vp), ("sH", C.c_int), ("sW", C.c_int), ("dH", C.c_int), ("dW", C.c_int),
                ("channels", C.c_int), ("u16", C.c_int), ("src_rs", i64), ("src_ps", i64), ("dst_rs", i64), ("dst_ps", i64)]


class MetricSrc(C.Structure):
    _c_name_ = "vmb_metric_src"
    _fields_ = [("img", vp), ("dtype", C.c_int), ("batch_stride", i64), ("row_stride", i64), ("pixel_stride", i64),
                ("channel_stride", i64)]


class ToYArgs(C.Structure):
    _c_name_ = "vmb_to_y_args"
    _fields_ = [("src", MetricSrc), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int), ("out", vp)]


class PsnrArgs(C.Structure):
    _c_name_ = "vmb_psnr_args"
    _fields_ = [("img1", MetricSrc), ("img2", MetricSrc), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int),
                ("y_channel", C.c_int), ("mse", vp), ("max_value", vp), ("psnr", vp), ("workspace", vp)]


class SsimArgs(C.Structure):
    _c_name_ = "vmb_ssim_args"
    _fields_ = [("img1", MetricSrc), ("img2", MetricSrc), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int),
                ("y_channel", C.c_int), ("mode", C.c_int), ("taps", C.c_double * 11), ("mix", C.c_double * 9), ("max_value", vp),
                ("ssim", vp), ("workspace", vp)]


NIQE_BLOCK, NIQE_TABLE, NIQE_FEATURES = 96, 9801, 36  # VMB_NIQE_BLOCK / _TABLE / _FEATURES
NIQE_Y, NIQE_GRAY, NIQE_PLANE = 0, 1, 2  # VMB_NIQE_Y / _GRAY / _PLANE


class NiqePrepArgs(C.Structure):
    _c_name_ = "vmb_niqe_prep_args"
    _fields_ = [("src", MetricSrc), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int), ("channels", C.c_int), ("convert", C.c_int),
                ("plane", vp), ("half", vp)]


class NiqeFeaturesArgs(C.Structure):
    _c_name_ = "vmb_niqe_features_args"
    _fields_ = [("plane", vp), ("half", vp), ("table", vp), ("features", vp), ("mscn", vp), ("mscn_half", vp),
                ("window", C.c_double * 49), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class NiqeScoreArgs(C.Structure):
    _c_name_ = "vmb_niqe_score_args"
    _fields_ = [("features", vp), ("mu_pris", vp), ("cov_pris", vp), ("score", vp), ("batch", C.c_int), ("blocks", C.c_int)]


class Filter2dArgs(C.Structure):
    _c_name_ = "vmb_filter2d_args"
    _fields_ = [("img", vp), ("out", vp), ("kernel", vp), ("batch", C.c_int), ("channels", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("k", C.c_int), ("per_image", C.c_int), ("quantize_out", C.c_int)]


class UsmSharpArgs(C.Structure):
    _c_name_ = "vmb_usm_sharp_args"
    _fields_ = [("img", vp), ("out", vp), ("workspace", vp), ("batch", C.c_int), ("channels", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("k", C.c_int), ("taps", C.c_float * 51), ("weight", C.c_float), ("threshold", C.c_float)]


class JpegArgs(C.Structure):
    _c_name_ = "vmb_jpeg_args"
    _fields_ = [("img", vp), ("out", vp), ("quality", vp), ("factor", C.c_float), ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("clamp_in", C.c_int), ("quantize_out", C.c_int)]


class NoiseLevelsArgs(C.Structure):
    _c_name_ = "vmb_noise_levels_args"
    _fields_ = [("img", vp), ("rates", vp), ("rates_gray", vp), ("vals", vp), ("vals_gray", vp), ("workspace", vp),
                ("batch", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class NoiseApplyArgs(C.Structure):
    _c_name_ = "vmb_noise_apply_args"
    _fields_ = [("img", vp), ("out", vp), ("noise", vp), ("noise_gray", vp), ("u_param", vp), ("u_gray", vp),
                ("param_lo", C.c_float), ("param_span", C.c_float), ("gray_prob", C.c_float), ("vals", vp), ("vals_gray", vp),
                ("kind", C.c_int), ("batch", C.c_int), ("channels", C.c_int), ("H", C.c_int), ("W", C.c_int), ("clip", C.c_int),
                ("rounds", C.c_int)]


SN_MAX_LAYERS = 8  # VMB_SN_MAX_LAYERS


class SnFwdArgs(C.Structure):
    _c_name_ = "vmb_sn_fwd_args"
    _fields_ = [("w", vp * SN_MAX_LAYERS), ("wn", vp * SN_MAX_LAYERS), ("u", vp * SN_MAX_LAYERS), ("v", vp * SN_MAX_LAYERS),
                ("u_save", vp * SN_MAX_LAYERS), ("v_save", vp * SN_MAX_LAYERS), ("rows", C.c_int * SN_MAX_LAYERS),
                ("cols", C.c_int * SN_MAX_LAYERS), ("sigma", vp), ("workspace", vp), ("layers", C.c_int), ("train", C.c_int),
                ("dtype", C.c_int), ("eps", C.c_float)]


class SnBwdArgs(C.Structure):
    _c_name_ = "vmb_sn_bwd_args"
    _fields_ = [("g", vp * SN_MAX_LAYERS), ("w", vp * SN_MAX_LAYERS), ("u", vp * SN_MAX_LAYERS), ("v", vp * SN_MAX_LAYERS),
                ("grad", vp * SN_MAX_LAYERS), ("rows", C.c_int * SN_MAX_LAYERS), ("cols", C.c_int * SN_MAX_LAYERS),
                ("accumulate", C.c_int * SN_MAX_LAYERS), ("sigma", vp), ("workspace", vp), ("layers", C.c_int), ("dtype", C.c_int)]


class GanUpArgs(C.Structure):
    _c_name_ = "vmb_gan_up_args"
    _fields_ = [("pre", vp), ("skip", vp), ("out", vp), ("planes", C.c_int), ("H", C.c_int), ("W", C.c_int), ("dtype", C.c_int)]


class GanUpBwdArgs(C.Structure):
    _c_name_ = "vmb_gan_up_bwd_args"
    _fields_ = [("dout", vp), ("pre", vp), ("dpre", vp), ("dskip", vp), ("planes", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("dtype", C.c_int)]


class GanActArgs(C.Structure):
    _c_name_ = "vmb_gan_act_args"
    _fields_ = [("x", vp), ("skip", vp), ("out", vp), ("n", i64), ("dtype", C.c_int)]


class GanActBwdArgs(C.Structure):
    _c_name_ = "vmb_gan_act_bwd_args"
    _fields_ = [("g", vp), ("g2", vp), ("ref", vp), ("dx", vp), ("n", i64), ("dtype", C.c_int)]


class BceLogitsArgs(C.Structure):
    _c_name_ = "vmb_bce_logits_args"
    _fields_ = [("x", vp), ("loss", vp), ("workspace", vp), ("n", i64), ("target", C.c_float), ("weight", C.c_float),
                ("dtype", C.c_int)]


class BceLogitsBwdArgs(C.Structure):
    _c_name_ = "vmb_bce_logits_bwd_args"
    _fields_ = [("x", vp), ("grad_loss", vp), ("grad_x", vp), ("n", i64), ("target", C.c_float), ("weight", C.c_float),
                ("dtype", C.c_int)]


class MeanLossArgs(C.Structure):
    _c_name_ = "vmb_mean_loss_args"
    _fields_ = [("x", vp), ("y", vp), ("out", vp), ("workspace", vp), ("n", i64), ("weight", C.c_float), ("dtype", C.c_int)]


class GanOutGradArgs(C.Structure):
    _c_name_ = "vmb_gan_out_grad_args"
    _fields_ = [("out", vp), ("gt", vp), ("g_percep", vp), ("g_gan", vp), ("dout", vp), ("n", i64), ("w_pix", C.c_float),
                ("in_dtype", C.c_int), ("out_dtype", C.c_int)]


LR_MAX_MILESTONES = 8  # VMB_LR_MAX_MILESTONES
LR_MAX_PERIODS = 8  # VMB_LR_MAX_PERIODS


class LrRule(C.Structure):
    _c_name_ = "vmb_lr_rule"
    _fields_ = [("base", C.c_double), ("step_gamma", C.c_double), ("milestone_gamma", C.c_double), ("step_size", i64),
                ("milestones", i64 * LR_MAX_MILESTONES), ("n_milestones", C.c_int), ("n_periods", C.c_int),
                ("periods", i64 * LR_MAX_PERIODS), ("restart_weights", C.c_double * LR_MAX_PERIODS),
                ("eta_mins", C.c_double * LR_MAX_PERIODS)]


class LrScheduleArgs(C.Structure):
    _c_name_ = "vmb_lr_schedule_args"
    _fields_ = [("iter", vp), ("lr", vp), ("rule", LrRule * 2), ("n_rules", C.c_int)]


CROP_MIX_MAX_IMAGES = 64  # VMB_CROP_MIX_MAX_IMAGES


class CropMixTensor(C.Structure):
    _c_name_ = "vmb_crop_mix_tensor"
    _fields_ = [("src", vp), ("dst", vp), ("stride_n", i64), ("stride_c", i64), ("stride_h", i64), ("stride_w", i64),
                ("c", C.c_int), ("h", C.c_int), ("w", C.c_int), ("row0", C.c_int), ("col0", C.c_int)]


class BatchCropMixArgs(C.Structure):
    _c_name_ = "vmb_batch_crop_mix_args"
    _fields_ = [("t", CropMixTensor * 2), ("n_tensors", C.c_int), ("batch", C.c_int), ("idx", C.c_int * CROP_MIX_MAX_IMAGES),
                ("perm", C.c_int * CROP_MIX_MAX_IMAGES), ("lam", C.c_float), ("one_minus_lam", C.c_float), ("mix", C.c_int)]


PERCEP_L1, PERCEP_L2, PERCEP_FRO = 0, 1, 2  # VMB_PERCEP_L1 / _L2 / _FRO
PERCEP_MAX_FEATS = 37  # VMB_PERCEP_MAX_FEATS


class PercepNormArgs(C.Structure):
    _c_name_ = "vmb_percep_norm_args"
    _fields_ = [("x", vp), ("gt", vp), ("x_stride", i64 * 4), ("gt_stride", i64 * 4), ("mean", vp), ("std", vp), ("out", vp),
                ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("range_norm", C.c_int), ("dtype", C.c_int)]


class PercepNormBwdArgs(C.Structure):
    _c_name_ = "vmb_percep_norm_bwd_args"
    _fields_ = [("g", vp), ("dx", vp), ("std", vp), ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("range_norm", C.c_int),
                ("dtype", C.c_int)]


class PercepStageArgs(C.Structure):
    _c_name_ = "vmb_percep_stage_args"
    _fields_ = [("y", vp), ("pooled", vp), ("code", vp), ("save", vp * 3), ("partial", vp * 3), ("feat", C.c_int * 3),
                ("B", C.c_int), ("C", C.c_int), ("H", C.c_int), ("W", C.c_int), ("relu", C.c_int), ("pool", C.c_int),
                ("crit", C.c_int), ("dtype", C.c_int)]


class PercepLossArgs(C.Structure):
    _c_name_ = "vmb_percep_loss_args"
    _fields_ = [("partial", vp), ("loss", vp), ("value", vp), ("offset", C.c_int * (PERCEP_MAX_FEATS + 1)),
                ("numel", i64 * PERCEP_MAX_FEATS), ("weight", C.c_float * PERCEP_MAX_FEATS), ("feats", C.c_int), ("crit", C.c_int),
                ("perceptual_weight", C.c_float)]


class PercepStageBwdArgs(C.Structure):
    _c_name_ = "vmb_percep_stage_bwd_args"
    _fields_ = [("g_in", vp), ("g_out", vp), ("code", vp), ("save", vp * 3), ("grad_loss", vp), ("value", vp),
                ("feat", C.c_int * 3), ("feat_index", C.c_int * 3), ("scale", C.c_float * 3), ("B", C.c_int), ("C", C.c_int),
                ("H", C.c_int), ("W", C.c_int), ("relu", C.c_int), ("pool", C.c_int), ("crit", C.c_int), ("dtype", C.c_int)]


PMETRIC_LPIPS, PMETRIC_DISTS = 0, 1  # VMB_PMETRIC_LPIPS / _DISTS
PMETRIC_MAX_LAYERS = 6  # VMB_PMETRIC_MAX_LAYERS


class PmetricSrc(C.Structure):
    _c_name_ = "vmb_pmetric_src"
    _fields_ = [("data", vp), ("stride", i64 * 4), ("u8", C.c_int)]


class PmetricPrepArgs(C.Structure):
    _c_name_ = "vmb_pmetric_prep_args"
    _fields_ = [("src", PmetricSrc * 2), ("shift", vp), ("scale", vp), ("out", vp), ("stats", vp), ("B", C.c_int), ("H", C.c_int),
                ("W", C.c_int), ("metric", C.c_int), ("normalize", C.c_int)]


class LpipsLayerArgs(C.Structure):
    _c_name_ = "vmb_lpips_layer_args"
    _fields_ = [("y", vp), ("w", vp), ("partial", vp), ("B", C.c_int), ("C", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class LpipsFinalArgs(C.Structure):
    _c_name_ = "vmb_lpips_final_args"
    _fields_ = [("partial", vp), ("layer", vp), ("out", vp), ("offset", C.c_int * PMETRIC_MAX_LAYERS),
                ("ctas", C.c_int * PMETRIC_MAX_LAYERS), ("hw", i64 * PMETRIC_MAX_LAYERS), ("B", C.c_int), ("layers", C.c_int)]


class DistsLayerArgs(C.Structure):
    _c_name_ = "vmb_dists_layer_args"
    _fields_ = [("y", vp), ("pooled", vp), ("stats", vp), ("B", C.c_int), ("C", C.c_int), ("H", C.c_int), ("W", C.c_int)]


class DistsFinalArgs(C.Structure):
    _c_name_ = "vmb_dists_final_args"
    _fields_ = [("stats", vp), ("alpha", vp), ("beta", vp), ("score", vp), ("mean", vp), ("offset", i64 * PMETRIC_MAX_LAYERS),
                ("n", i64 * PMETRIC_MAX_LAYERS), ("C", C.c_int * PMETRIC_MAX_LAYERS), ("tiles", C.c_int * PMETRIC_MAX_LAYERS),
                ("B", C.c_int), ("layers", C.c_int)]


# every symbol include/vmambair_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "vmb_last_error": (C.c_char_p, []),
    "vmb_version": (C.c_char_p, []),
    "vmb_scan_ckpt_interval": (C.c_int, []),
    "vmb_selective_scan_fwd": (C.c_int, [C.POINTER(ScanFwdArgs), vp]),
    "vmb_selective_scan_bwd": (C.c_int, [C.POINTER(ScanBwdArgs), vp]),
    "vmb_scan_gate_bwd": (C.c_int, [C.POINTER(ScanGateArgs), vp]),
    "vmb_scan_bwd_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "vmb_scan_bwd_det_workspace_bytes": (C.c_int64, [C.POINTER(ScanBwdArgs)]),
    "vmb_pixlin": (C.c_int, [C.POINTER(PixlinArgs), vp]),
    "vmb_dwconv3x3": (C.c_int, [C.POINTER(DwconvArgs), vp]),
    "vmb_cross_scan": (C.c_int, [C.POINTER(CrossScanArgs), vp]),
    "vmb_merge_norm_gate": (C.c_int, [C.POINTER(MergeArgs), vp]),
    "vmb_merge_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "vmb_transpose_hw": (C.c_int, [C.POINTER(TransposeArgs), vp]),
    "vmb_pixel_shuffle2_nhwc": (C.c_int, [C.POINTER(PixelShuffleArgs), vp]),
    "vmb_pixel_shuffle2_nhwc_bias": (C.c_int, [C.POINTER(PixelShuffleArgs), vp, vp]),
    "vmb_conv3x3": (C.c_int, [C.POINTER(Conv3x3Args), vp]),
    "vmb_cross_scan_multi": (C.c_int, [C.POINTER(CrossScanArgs), C.c_int, vp]),
    "vmb_dwconv3x3_t": (C.c_int, [C.POINTER(DwconvArgs), vp, vp]),
    "vmb_selective_scan_fwd_grouped": (C.c_int, [C.POINTER(ScanGroupedArgs), vp]),
    "vmb_selective_scan_bwd_grouped": (C.c_int, [C.POINTER(ScanGroupedBwdArgs), vp]),
    "vmb_scan_grouped_bwd_det_workspace_bytes": (C.c_int64, [C.POINTER(ScanGroupedBwdArgs)]),
    "vmb_merge_sum": (C.c_int, [C.POINTER(MergeArgs), vp, vp]),
    "vmb_channel_branch": (C.c_int, [C.POINTER(ChannelArgs), vp]),
    "vmb_layernorm_fwd": (C.c_int, [C.POINTER(LnFwdArgs), vp]),
    "vmb_layernorm_bwd": (C.c_int, [C.POINTER(LnBwdArgs), vp]),
    "vmb_merge_norm_gate_bwd": (C.c_int, [C.POINTER(MergeBwdArgs), vp]),
    "vmb_dwconv3x3_bwd": (C.c_int, [C.POINTER(DwconvBwdArgs), vp]),
    "vmb_channel_gate_bwd": (C.c_int, [C.POINTER(GateBwdArgs), vp]),
    "vmb_fused_adam": (C.c_int, [C.POINTER(AdamArgs), vp]),
    "vmb_pixlin_wgrad": (C.c_int, [C.POINTER(WgradArgs), vp]),
    "vmb_pixlin_wgrad_workspace_bytes": (C.c_int64, [C.POINTER(WgradArgs)]),
    "vmb_channel_branch_bwd": (C.c_int, [C.POINTER(ChannelBwdArgs), vp]),
    "vmb_channel_branch_bwd_smem_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "vmb_channel_branch_bwd_scratch_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int]),
    "vmb_cross_selective_scan_c_fwd": (C.c_int, [C.POINTER(CrossScanCArgs), vp]),
    "vmb_cross_selective_scan_c_bwd": (C.c_int, [C.POINTER(CrossScanCBwdArgs), vp]),
    "vmb_cross_selective_scan_c_smem_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "vmb_cross_selective_scan_c_workspace_bytes": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "vmb_prep_block_weights": (C.c_int, [C.POINTER(PrepArgs), vp]),
    "vmb_sum4_add": (C.c_int, [vp, vp, vp, C.c_int, C.c_long, C.c_int, vp]),
    "vmb_image_max": (C.c_int, [C.POINTER(ImageMaxArgs), vp]),
    "vmb_image_to_planes": (C.c_int, [C.POINTER(ImageToPlanesArgs), vp]),
    "vmb_planes_to_image": (C.c_int, [C.POINTER(PlanesToImageArgs), vp]),
    "vmb_resize_lanczos4": (C.c_int, [C.POINTER(ResizeLanczos4Args), vp]),
    "vmb_to_y_channel": (C.c_int, [C.POINTER(ToYArgs), vp]),
    "vmb_psnr": (C.c_int, [C.POINTER(PsnrArgs), vp]),
    "vmb_psnr_workspace_bytes": (C.c_int64, [C.POINTER(PsnrArgs)]),
    "vmb_ssim": (C.c_int, [C.POINTER(SsimArgs), vp]),
    "vmb_ssim_workspace_bytes": (C.c_int64, [C.POINTER(SsimArgs)]),
    "vmb_niqe_table": (C.c_int, [vp, vp]),
    "vmb_niqe_prep": (C.c_int, [C.POINTER(NiqePrepArgs), vp]),
    "vmb_niqe_features": (C.c_int, [C.POINTER(NiqeFeaturesArgs), vp]),
    "vmb_niqe_score": (C.c_int, [C.POINTER(NiqeScoreArgs), vp]),
    "vmb_filter2d": (C.c_int, [C.POINTER(Filter2dArgs), vp]),
    "vmb_usm_sharp": (C.c_int, [C.POINTER(UsmSharpArgs), vp]),
    "vmb_jpeg": (C.c_int, [C.POINTER(JpegArgs), vp]),
    "vmb_noise_levels": (C.c_int, [C.POINTER(NoiseLevelsArgs), vp]),
    "vmb_noise_apply": (C.c_int, [C.POINTER(NoiseApplyArgs), vp]),
    "vmb_sn_fwd": (C.c_int, [C.POINTER(SnFwdArgs), vp]),
    "vmb_sn_workspace_bytes": (C.c_int64, [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vmb_sn_bwd": (C.c_int, [C.POINTER(SnBwdArgs), vp]),
    "vmb_sn_bwd_workspace_bytes": (C.c_int64, [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vmb_gan_up": (C.c_int, [C.POINTER(GanUpArgs), vp]),
    "vmb_gan_up_bwd": (C.c_int, [C.POINTER(GanUpBwdArgs), vp]),
    "vmb_gan_act": (C.c_int, [C.POINTER(GanActArgs), vp]),
    "vmb_gan_act_bwd": (C.c_int, [C.POINTER(GanActBwdArgs), vp]),
    "vmb_bce_logits": (C.c_int, [C.POINTER(BceLogitsArgs), vp]),
    "vmb_bce_logits_workspace_bytes": (C.c_int64, [C.c_int64]),
    "vmb_bce_logits_bwd": (C.c_int, [C.POINTER(BceLogitsBwdArgs), vp]),
    "vmb_mean_loss": (C.c_int, [C.POINTER(MeanLossArgs), vp]),
    "vmb_mean_loss_workspace_bytes": (C.c_int64, [C.c_int64]),
    "vmb_gan_out_grad": (C.c_int, [C.POINTER(GanOutGradArgs), vp]),
    "vmb_lr_schedule": (C.c_int, [C.POINTER(LrScheduleArgs), vp]),
    "vmb_ema_update": (C.c_int, [vp, vp, C.c_int64, C.c_float, vp]),
    "vmb_batch_crop_mix": (C.c_int, [C.POINTER(BatchCropMixArgs), vp]),
    "vmb_percep_norm": (C.c_int, [C.POINTER(PercepNormArgs), vp]),
    "vmb_percep_norm_bwd": (C.c_int, [C.POINTER(PercepNormBwdArgs), vp]),
    "vmb_percep_stage": (C.c_int, [C.POINTER(PercepStageArgs), vp]),
    "vmb_percep_stage_ctas": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "vmb_percep_loss": (C.c_int, [C.POINTER(PercepLossArgs), vp]),
    "vmb_percep_stage_bwd": (C.c_int, [C.POINTER(PercepStageBwdArgs), vp]),
    "vmb_pmetric_prep": (C.c_int, [C.POINTER(PmetricPrepArgs), vp]),
    "vmb_pmetric_tiles": (C.c_int, [C.c_int, C.c_int64]),
    "vmb_lpips_layer": (C.c_int, [C.POINTER(LpipsLayerArgs), vp]),
    "vmb_lpips_layer_ctas": (C.c_int, [C.c_int, C.c_int, C.c_int]),
    "vmb_lpips_final": (C.c_int, [C.POINTER(LpipsFinalArgs), vp]),
    "vmb_dists_layer": (C.c_int, [C.POINTER(DistsLayerArgs), vp]),
    "vmb_dists_final": (C.c_int, [C.POINTER(DistsFinalArgs), vp]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"vmambair_b200: CUDA library not built ({LIB_PATH}); run `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C vmambair_b200/csrc`. There is no CPU fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(l, name)  # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(status: int, what: str):
    if status != 0:
        msg = lib().vmb_last_error().decode()
        raise RuntimeError(f"{what}: {msg} (status {status})")
