// Decoding of a vmb_metric_src element and the reference's to_y_channel, shared by the metric kernels (metrics.cu, niqe.cu).
// The Y chain spells out every rounding (__fdiv_rn, __dmul_rn, __dadd_rn, ...) so nvcc cannot contract it: it equals the reference's
// numpy arithmetic bit for bit.
#pragma once
#include <math.h>

#include "common.cuh"

namespace vmb {

// the reference's float64 value of element (b, y, x, c)
__device__ __forceinline__ double load_val(const vmb_metric_src& s, int b, int y, int x, int c) {
    const int64_t i = b * s.batch_stride + y * s.row_stride + x * s.pixel_stride + c * s.channel_stride;
    if (s.dtype == VMB_MSRC_U8) return (double)reinterpret_cast<const uint8_t*>(s.img)[i];
    if (s.dtype == VMB_MSRC_U16) return (double)reinterpret_cast<const uint16_t*>(s.img)[i];
    if (s.dtype == VMB_MSRC_F32) return (double)reinterpret_cast<const float*>(s.img)[i];
    if (s.dtype == VMB_MSRC_F64) return reinterpret_cast<const double*>(s.img)[i];
    const float q = s.dtype == VMB_MSRC_Q_F32    ? reinterpret_cast<const float*>(s.img)[i]
                    : s.dtype == VMB_MSRC_Q_BF16 ? to_f32(reinterpret_cast<const __nv_bfloat16*>(s.img)[i])
                                                 : to_f32(reinterpret_cast<const __half*>(s.img)[i]);
    // tensor2img: clamp_(0, 1), (x * 255.0).round() in float32 (half to even), uint8; fminf / fmaxf map a NaN to 0 as the cast does
    return (double)rintf(__fmul_rn(fminf(fmaxf(q, 0.f), 1.f), 255.f));
}

// to_y_channel of one BGR pixel: img.astype(float32) / 255., np.dot(img, [24.966, 128.553, 65.481]) + 16.0 in float64 (left to
// right), / 255. and .astype(float32) (_convert_output_type_range), then * 255. in float32
__device__ __forceinline__ float y_bgr(double b, double g, double r) {
    const double xb = __fdiv_rn(__double2float_rn(b), 255.f), xg = __fdiv_rn(__double2float_rn(g), 255.f),
                 xr = __fdiv_rn(__double2float_rn(r), 255.f);
    const double d = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(xb, 24.966), __dmul_rn(xg, 128.553)), __dmul_rn(xr, 65.481)), 16.0);
    return __fmul_rn(__double2float_rn(__ddiv_rn(d, 255.0)), 255.f);
}

// to_y_channel of a one-channel image: the float32 round trip / 255. * 255.
__device__ __forceinline__ float y_gray(double v) { return __fmul_rn(__fdiv_rn(__double2float_rn(v), 255.f), 255.f); }

inline bool metric_src_ok(const vmb_metric_src& s) { return s.img != nullptr && s.dtype >= VMB_MSRC_U8 && s.dtype <= VMB_MSRC_Q_F16; }

}  // namespace vmb
