// Backward stages of the fused OSS block (training path; SURVEY.md 8 a15): the autograd of
//   LayerNorm (norm1 / norm2; reference SRGAN/VmambaIR/archs/MambaSISR6_arch.py:166-195),
//   out_norm + SiLU(z) gate + AdaptiveAvgPool2d sums (:433-441,493),
//   depthwise 3x3 + SiLU (:490-491) and depthwise 3x3 + exact-GELU gate (FeedForward :215-216),
//   the channel gate y*(1+c) / y+c in front of out_conv (:494-496)
// as hand-written kernels.  Activations are NCHW, pixel-contiguous (B, C, L) views addressed by (batch, channel) strides.
// Per-pixel reductions over channels run one thread per pixel (coalesced along L); per-channel reductions over pixels (the
// parameter gradients) run one CTA per (channel, image) with a block reduction and ONE fp32 atomicAdd per CTA.
// The 1x1-conv data gradients reuse vmb_pixlin with the transposed weight; the scan gradient is vmb_selective_scan_bwd.
#include "common.cuh"
#include "train_params.h"
#include "dwconv_common.cuh"

namespace vmb {

__device__ __forceinline__ float sigmoid_t(float v) { return rcp_approx(1.f + ex2(-v * kLog2e)); }
__device__ __forceinline__ float silu_t(float v) { return v * sigmoid_t(v); }
__device__ __forceinline__ float dsilu_t(float v) {  // d/dv v*sigmoid(v)
    const float s = sigmoid_t(v);
    return s * fmaf(v, 1.f - s, 1.f);
}
__device__ __forceinline__ float erf_t(float x) {  // Abramowitz-Stegun 7.1.26, |err| <= 1.5e-7 (same as the forward kernel)
    const float ax = fabsf(x);
    const float t = rcp_approx(fmaf(0.3275911f, ax, 1.f));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float r = 1.f - poly * t * ex2(-ax * ax * kLog2e);
    return copysignf(r, x);
}
__device__ __forceinline__ float gelu_t(float v) { return 0.5f * v * (1.f + erf_t(v * 0.70710678118654752f)); }
__device__ __forceinline__ float dgelu_t(float v) {  // Phi(v) + v*phi(v)
    const float cdf = 0.5f * (1.f + erf_t(v * 0.70710678118654752f));
    return fmaf(v * 0.3989422804014327f, ex2(-0.5f * v * v * kLog2e), cdf);
}

template <typename in_t> struct Pair;
template <> struct Pair<float> {
    static __device__ __forceinline__ float2 ld(const float* p) { return *reinterpret_cast<const float2*>(p); }
    static __device__ __forceinline__ void st(float* p, float2 v) { *reinterpret_cast<float2*>(p) = v; }
};
template <> struct Pair<__nv_bfloat16> {
    static __device__ __forceinline__ float2 ld(const __nv_bfloat16* p) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p)); }
    static __device__ __forceinline__ void st(__nv_bfloat16* p, float2 v) { *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v.x, v.y); }
};
template <> struct Pair<__half> {
    static __device__ __forceinline__ float2 ld(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }
    static __device__ __forceinline__ void st(__half* p, float2 v) { *reinterpret_cast<__half2*>(p) = __floats2half2_rn(v.x, v.y); }
};


__device__ __forceinline__ float block_sum_256(float v, float* sred) {  // 256 threads; result valid in thread 0
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sred[i];
    }
    __syncthreads();
    return t;
}

// ------------------------------------------------------------------------------------------ LayerNorm forward (materialised)
// y = (x - mu) * rstd * w + b  (mode 1, WithBias)   or   x * rstd * w  (mode 2, BiasFree; variance about the mean), two-pass.
template <typename in_t>
__global__ void __launch_bounds__(128) ln_fwd_kernel(const LnFwdParams p) {
    pdl_trigger();
    pdl_wait();
    const int l = blockIdx.x * 128 + threadIdx.x, b = blockIdx.y;
    if (l >= p.L) return;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs + l;
    float s = 0.f;
    for (int c = 0; c < p.C; ++c) s += to_f32<in_t>(x[(int64_t)c * p.x_cs]);
    const float mu = s / p.C;
    float v = 0.f;
    for (int c = 0; c < p.C; ++c) {
        const float d = to_f32<in_t>(x[(int64_t)c * p.x_cs]) - mu;
        v = fmaf(d, d, v);
    }
    const float rstd = rsqrtf(v / p.C + 1e-5f);
    if (p.stats) {
        p.stats[((int64_t)b * p.L + l) * 2] = mu;
        p.stats[((int64_t)b * p.L + l) * 2 + 1] = rstd;
    }
    if (!p.y) return;
    in_t* __restrict__ y = reinterpret_cast<in_t*>(p.y) + (int64_t)b * p.y_bs + l;
    for (int c = 0; c < p.C; ++c) {
        const float xv = to_f32<in_t>(x[(int64_t)c * p.x_cs]);
        const float o = p.mode == 1 ? fmaf((xv - mu) * rstd, p.w[c], p.b[c]) : xv * rstd * p.w[c];
        y[(int64_t)c * p.y_cs] = from_f32<in_t>(o);
    }
}

// ------------------------------------------------------------------------------------------ LayerNorm backward
// dx kernel: one thread per pixel.  mode 1: dx = rstd (gw - mean(gw) - xh mean(gw xh));  mode 2 (y = x rstd w):
// dx = rstd gw - rstd^3 (x - mu) mean(gw x).   gw = g*w, xh = (x - mu) rstd.   `add` (optional) is summed into dx
// (the residual branch's gradient).  Also writes (mu, rstd) per pixel for the parameter-gradient kernel.
template <typename in_t>
__global__ void __launch_bounds__(128) ln_bwd_dx_kernel(const LnBwdParams p) {
    pdl_trigger();
    pdl_wait();
    const int l = blockIdx.x * 128 + threadIdx.x, b = blockIdx.y;
    if (l >= p.L) return;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs + l;
    const in_t* __restrict__ g = reinterpret_cast<const in_t*>(p.g) + (int64_t)b * p.g_bs + l;
    float s = 0.f;
    for (int c = 0; c < p.C; ++c) s += to_f32<in_t>(x[(int64_t)c * p.x_cs]);
    const float mu = s / p.C;
    float v = 0.f, s1 = 0.f, s2 = 0.f;
    for (int c = 0; c < p.C; ++c) {
        const float xv = to_f32<in_t>(x[(int64_t)c * p.x_cs]);
        const float d = xv - mu;
        v = fmaf(d, d, v);
        const float gw = to_f32<in_t>(g[(int64_t)c * p.g_cs]) * p.w[c];
        s1 += gw;
        s2 = fmaf(gw, p.mode == 1 ? d : xv, s2);
    }
    const float rstd = rsqrtf(v / p.C + 1e-5f);
    p.stats[((int64_t)b * p.L + l) * 2] = mu;
    p.stats[((int64_t)b * p.L + l) * 2 + 1] = rstd;
    const float invC = 1.f / p.C;
    // mode 1: s2 = sum gw (x-mu) -> mean(gw xh) = s2 rstd / C ; term = xh * that = (x-mu) rstd^2 s2 / C
    const float k1 = s1 * invC, k2 = s2 * invC * rstd * rstd;
    const in_t* __restrict__ a = p.add ? reinterpret_cast<const in_t*>(p.add) + (int64_t)b * p.a_bs + l : nullptr;
    in_t* __restrict__ dx = reinterpret_cast<in_t*>(p.dx) + (int64_t)b * p.dx_bs + l;
    for (int c = 0; c < p.C; ++c) {
        const float xv = to_f32<in_t>(x[(int64_t)c * p.x_cs]);
        const float gw = to_f32<in_t>(g[(int64_t)c * p.g_cs]) * p.w[c];
        float o = p.mode == 1 ? rstd * (gw - k1 - (xv - mu) * k2) : rstd * (gw - (xv - mu) * k2);
        if (a) o += to_f32<in_t>(a[(int64_t)c * p.a_cs]);
        dx[(int64_t)c * p.dx_cs] = from_f32<in_t>(o);
    }
}

// parameter gradients: grid (C, B); dw[c] += sum_l g xh (mode 1) or g x rstd (mode 2); db[c] += sum_l g
template <typename in_t>
__global__ void __launch_bounds__(256) ln_bwd_dwdb_kernel(const LnBwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sred[8];
    const int c = blockIdx.x, b = blockIdx.y;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs + (int64_t)c * p.x_cs;
    const in_t* __restrict__ g = reinterpret_cast<const in_t*>(p.g) + (int64_t)b * p.g_bs + (int64_t)c * p.g_cs;
    const float2* __restrict__ st = reinterpret_cast<const float2*>(p.stats) + (int64_t)b * p.L;
    float aw = 0.f, ab = 0.f;
    if ((p.L & 1) == 0 && ((p.x_bs | p.x_cs | p.g_bs | p.g_cs) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.x) & 7) == 0 &&
        (reinterpret_cast<uintptr_t>(p.g) & 7) == 0) {
#pragma unroll 4
        for (int l = threadIdx.x * 2; l < p.L; l += 512) {
            const float4 s = *reinterpret_cast<const float4*>(st + l);
            const float2 gv = Pair<in_t>::ld(g + l), xv = Pair<in_t>::ld(x + l);
            aw = fmaf(gv.x, (p.mode == 1 ? xv.x - s.x : xv.x) * s.y, aw);
            aw = fmaf(gv.y, (p.mode == 1 ? xv.y - s.z : xv.y) * s.w, aw);
            ab += gv.x + gv.y;
        }
    } else
    for (int l = threadIdx.x; l < p.L; l += 256) {
        const float2 s = st[l];
        const float gv = to_f32<in_t>(g[l]), xv = to_f32<in_t>(x[l]);
        aw = fmaf(gv, (p.mode == 1 ? xv - s.x : xv) * s.y, aw);
        ab += gv;
    }
    const float tw = block_sum_256(aw, sred), tb = block_sum_256(ab, sred);
    if (threadIdx.x == 0) {
        atomicAdd(p.dw + c, tw);
        if (p.db) atomicAdd(p.db + c, tb);
    }
}

// ------------------------------------------------------------------------------------------ out_norm + gate backward
// forward (merge kernels): m = merged scan output (fp32), n = (m - mu) rstd w + b, y2 = n * silu(z), pooled[b,c] = sum_l y2.
// given dy2 and dpooled:  t = dy2 + dpooled[b,c];  dn = t silu(z);  dz = t n silu'(z);  dm = LayerNorm backward of dn.
template <typename in_t>
__global__ void __launch_bounds__(128) merge_bwd_dx_kernel(const MergeBwdParams p) {
    pdl_trigger();
    pdl_wait();
    const int l = blockIdx.x * 128 + threadIdx.x, b = blockIdx.y;
    if (l >= p.L) return;
    const int C = p.C;
    const float* __restrict__ m = p.merged + (int64_t)b * C * p.L + l;
    const float2 st = reinterpret_cast<const float2*>(p.stats)[(int64_t)b * p.L + l];
    const float invC = 1.f / C;
    const float mu = st.x * invC;
    const float rstd = rsqrtf(fmaxf(st.y * invC - mu * mu, 0.f) + 1e-5f);
    const in_t* __restrict__ z = reinterpret_cast<const in_t*>(p.z) + (int64_t)b * p.z_bs + l;
    const in_t* __restrict__ dy2 = reinterpret_cast<const in_t*>(p.dy2) + (int64_t)b * C * p.L + l;
    const float* __restrict__ dpool = p.dpooled ? p.dpooled + (int64_t)b * C : nullptr;
    float s1 = 0.f, s2 = 0.f;
    for (int c = 0; c < C; ++c) {
        const float t = to_f32<in_t>(dy2[(int64_t)c * p.L]) + (dpool ? dpool[c] : 0.f);
        const float gw = t * silu_t(to_f32<in_t>(z[(int64_t)c * p.z_cs])) * p.w[c];
        s1 += gw;
        s2 = fmaf(gw, m[(int64_t)c * p.L] - mu, s2);
    }
    const float k1 = s1 * invC, k2 = s2 * invC * rstd * rstd;
    in_t* __restrict__ dm = reinterpret_cast<in_t*>(p.dm) + (int64_t)b * C * p.L + l;
    in_t* __restrict__ dz = reinterpret_cast<in_t*>(p.dz) + (int64_t)b * p.dz_bs + l;
    for (int c = 0; c < C; ++c) {
        const float t = to_f32<in_t>(dy2[(int64_t)c * p.L]) + (dpool ? dpool[c] : 0.f);
        const float zv = to_f32<in_t>(z[(int64_t)c * p.z_cs]);
        const float d = m[(int64_t)c * p.L] - mu;
        const float gw = t * silu_t(zv) * p.w[c];
        dm[(int64_t)c * p.L] = from_f32<in_t>(rstd * (gw - k1 - d * k2));
        const float n = fmaf(d * rstd, p.w[c], p.b[c]);
        dz[(int64_t)c * p.dz_cs] = from_f32<in_t>(t * n * dsilu_t(zv));
    }
}

template <typename in_t>
__global__ void __launch_bounds__(256) merge_bwd_dwdb_kernel(const MergeBwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sred[8];
    const int c = blockIdx.x, b = blockIdx.y, C = p.C;
    const float* __restrict__ m = p.merged + ((int64_t)b * C + c) * p.L;
    const float2* __restrict__ st = reinterpret_cast<const float2*>(p.stats) + (int64_t)b * p.L;
    const in_t* __restrict__ z = reinterpret_cast<const in_t*>(p.z) + (int64_t)b * p.z_bs + (int64_t)c * p.z_cs;
    const in_t* __restrict__ dy2 = reinterpret_cast<const in_t*>(p.dy2) + ((int64_t)b * C + c) * p.L;
    const float dp = p.dpooled ? p.dpooled[(int64_t)b * C + c] : 0.f;
    const float invC = 1.f / C;
    float aw = 0.f, ab = 0.f;
    for (int l = threadIdx.x; l < p.L; l += 256) {
        const float2 s = st[l];
        const float mu = s.x * invC;
        const float rstd = rsqrtf(fmaxf(s.y * invC - mu * mu, 0.f) + 1e-5f);
        const float dn = (to_f32<in_t>(dy2[l]) + dp) * silu_t(to_f32<in_t>(z[l]));
        aw = fmaf(dn, (m[l] - mu) * rstd, aw);
        ab += dn;
    }
    const float tw = block_sum_256(aw, sred), tb = block_sum_256(ab, sred);
    if (threadIdx.x == 0) {
        atomicAdd(p.dw + c, tw);
        atomicAdd(p.db + c, tb);
    }
}


// ------------------------------------------------------------------------------------------ channel-split pixel kernels (fast path)
// The per-pixel LayerNorm kernels above walk all C channels in one thread (3 dependent passes, 16 K threads at 4 x 64x64: latency
// bound).  Fast path for even L and 4-byte aligned rows: a CTA of 256 threads owns 64 pixels (32 pairs, one 32-bit / 64-bit load
// per channel) x 8 channel slices; the per-pixel sums of the slices meet in shared memory.
constexpr int PX_PAIRS = 32, PX_Q = 8;

// sum of `v` over the PX_Q channel slices of one pixel pair; every thread of the pair gets the total
__device__ __forceinline__ float2 slice_sum(float2 v, float2 (*sm)[PX_PAIRS], int pp, int q) {
    __syncthreads();
    sm[q][pp] = v;
    __syncthreads();
    float2 t = make_float2(0.f, 0.f);
#pragma unroll
    for (int i = 0; i < PX_Q; ++i) {
        t.x += sm[i][pp].x;
        t.y += sm[i][pp].y;
    }
    return t;
}

template <typename in_t>
__global__ void __launch_bounds__(256) ln_fwd_px_kernel(const LnFwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float2 sm[PX_Q][PX_PAIRS];
    const int pp = threadIdx.x % PX_PAIRS, q = threadIdx.x / PX_PAIRS, b = blockIdx.y;
    const int l = min((blockIdx.x * PX_PAIRS + pp) * 2, p.L - 2);  // tail CTAs redo the last pair (idempotent)
    const int c0 = q * p.C / PX_Q, c1 = (q + 1) * p.C / PX_Q;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs + l;
    float2 s = make_float2(0.f, 0.f);
    for (int c = c0; c < c1; ++c) {
        const float2 v = Pair<in_t>::ld(x + (int64_t)c * p.x_cs);
        s.x += v.x; s.y += v.y;
    }
    s = slice_sum(s, sm, pp, q);
    const float2 mu = make_float2(s.x / p.C, s.y / p.C);
    float2 v2 = make_float2(0.f, 0.f);
    for (int c = c0; c < c1; ++c) {
        const float2 v = Pair<in_t>::ld(x + (int64_t)c * p.x_cs);
        v2.x = fmaf(v.x - mu.x, v.x - mu.x, v2.x);
        v2.y = fmaf(v.y - mu.y, v.y - mu.y, v2.y);
    }
    v2 = slice_sum(v2, sm, pp, q);
    const float2 rstd = make_float2(rsqrtf(v2.x / p.C + 1e-5f), rsqrtf(v2.y / p.C + 1e-5f));
    if (p.stats && q == 0) {
        float* st = p.stats + ((int64_t)b * p.L + l) * 2;
        *reinterpret_cast<float4*>(st) = make_float4(mu.x, rstd.x, mu.y, rstd.y);
    }
    if (!p.y) return;
    in_t* __restrict__ y = reinterpret_cast<in_t*>(p.y) + (int64_t)b * p.y_bs + l;
    for (int c = c0; c < c1; ++c) {
        const float2 v = Pair<in_t>::ld(x + (int64_t)c * p.x_cs);
        const float w = p.w[c];
        float2 o;
        if (p.mode == 1) {
            const float bb = p.b[c];
            o = make_float2(fmaf((v.x - mu.x) * rstd.x, w, bb), fmaf((v.y - mu.y) * rstd.y, w, bb));
        } else {
            o = make_float2(v.x * rstd.x * w, v.y * rstd.y * w);
        }
        Pair<in_t>::st(y + (int64_t)c * p.y_cs, o);
    }
}

template <typename in_t>
__global__ void __launch_bounds__(256) ln_bwd_dx_px_kernel(const LnBwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float2 sm[PX_Q][PX_PAIRS];
    const int pp = threadIdx.x % PX_PAIRS, q = threadIdx.x / PX_PAIRS, b = blockIdx.y;
    const int l = min((blockIdx.x * PX_PAIRS + pp) * 2, p.L - 2);
    const int c0 = q * p.C / PX_Q, c1 = (q + 1) * p.C / PX_Q;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs + l;
    const in_t* __restrict__ g = reinterpret_cast<const in_t*>(p.g) + (int64_t)b * p.g_bs + l;
    float2 s = make_float2(0.f, 0.f);
    for (int c = c0; c < c1; ++c) {
        const float2 v = Pair<in_t>::ld(x + (int64_t)c * p.x_cs);
        s.x += v.x; s.y += v.y;
    }
    s = slice_sum(s, sm, pp, q);
    const float2 mu = make_float2(s.x / p.C, s.y / p.C);
    float2 vv = make_float2(0.f, 0.f), s1 = vv, s2 = vv;
    for (int c = c0; c < c1; ++c) {
        const float2 v = Pair<in_t>::ld(x + (int64_t)c * p.x_cs);
        const float2 gv = Pair<in_t>::ld(g + (int64_t)c * p.g_cs);
        const float w = p.w[c];
        const float dx_ = v.x - mu.x, dy_ = v.y - mu.y;
        vv.x = fmaf(dx_, dx_, vv.x); vv.y = fmaf(dy_, dy_, vv.y);
        s1.x = fmaf(gv.x, w, s1.x); s1.y = fmaf(gv.y, w, s1.y);
        s2.x = fmaf(gv.x * w, p.mode == 1 ? dx_ : v.x, s2.x);
        s2.y = fmaf(gv.y * w, p.mode == 1 ? dy_ : v.y, s2.y);
    }
    vv = slice_sum(vv, sm, pp, q);
    s1 = slice_sum(s1, sm, pp, q);
    s2 = slice_sum(s2, sm, pp, q);
    const float2 rstd = make_float2(rsqrtf(vv.x / p.C + 1e-5f), rsqrtf(vv.y / p.C + 1e-5f));
    if (q == 0) {
        float* st = p.stats + ((int64_t)b * p.L + l) * 2;
        *reinterpret_cast<float4*>(st) = make_float4(mu.x, rstd.x, mu.y, rstd.y);
    }
    const float invC = 1.f / p.C;
    const float2 k1 = make_float2(s1.x * invC, s1.y * invC);
    const float2 k2 = make_float2(s2.x * invC * rstd.x * rstd.x, s2.y * invC * rstd.y * rstd.y);
    const in_t* __restrict__ a = p.add ? reinterpret_cast<const in_t*>(p.add) + (int64_t)b * p.a_bs + l : nullptr;
    in_t* __restrict__ dx = reinterpret_cast<in_t*>(p.dx) + (int64_t)b * p.dx_bs + l;
    for (int c = c0; c < c1; ++c) {
        const float2 v = Pair<in_t>::ld(x + (int64_t)c * p.x_cs);
        const float2 gv = Pair<in_t>::ld(g + (int64_t)c * p.g_cs);
        const float w = p.w[c];
        float2 o;
        if (p.mode == 1) {
            o.x = rstd.x * (gv.x * w - k1.x - (v.x - mu.x) * k2.x);
            o.y = rstd.y * (gv.y * w - k1.y - (v.y - mu.y) * k2.y);
        } else {
            o.x = rstd.x * (gv.x * w - (v.x - mu.x) * k2.x);
            o.y = rstd.y * (gv.y * w - (v.y - mu.y) * k2.y);
        }
        if (a) {
            const float2 av = Pair<in_t>::ld(a + (int64_t)c * p.a_cs);
            o.x += av.x; o.y += av.y;
        }
        Pair<in_t>::st(dx + (int64_t)c * p.dx_cs, o);
    }
}

template <typename in_t>
__global__ void __launch_bounds__(256) merge_bwd_dx_px_kernel(const MergeBwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float2 sm[PX_Q][PX_PAIRS];
    const int pp = threadIdx.x % PX_PAIRS, q = threadIdx.x / PX_PAIRS, b = blockIdx.y, C = p.C;
    const int l = min((blockIdx.x * PX_PAIRS + pp) * 2, p.L - 2);
    const int c0 = q * C / PX_Q, c1 = (q + 1) * C / PX_Q;
    const float* __restrict__ m = p.merged + (int64_t)b * C * p.L + l;
    const float4 st = *reinterpret_cast<const float4*>(p.stats + ((int64_t)b * p.L + l) * 2);  // (sum, sumsq) of two pixels
    const float invC = 1.f / C;
    const float2 mu = make_float2(st.x * invC, st.z * invC);
    const float2 rstd = make_float2(rsqrtf(fmaxf(st.y * invC - mu.x * mu.x, 0.f) + 1e-5f), rsqrtf(fmaxf(st.w * invC - mu.y * mu.y, 0.f) + 1e-5f));
    const in_t* __restrict__ z = reinterpret_cast<const in_t*>(p.z) + (int64_t)b * p.z_bs + l;
    const in_t* __restrict__ dy2 = reinterpret_cast<const in_t*>(p.dy2) + (int64_t)b * C * p.L + l;
    const float* __restrict__ dpool = p.dpooled ? p.dpooled + (int64_t)b * C : nullptr;
    float2 s1 = make_float2(0.f, 0.f), s2 = s1;
    for (int c = c0; c < c1; ++c) {
        const float2 t = Pair<in_t>::ld(dy2 + (int64_t)c * p.L);
        const float2 zv = Pair<in_t>::ld(z + (int64_t)c * p.z_cs);
        const float2 mv = *reinterpret_cast<const float2*>(m + (int64_t)c * p.L);
        const float dp = dpool ? dpool[c] : 0.f, w = p.w[c];
        const float gx = (t.x + dp) * silu_t(zv.x) * w, gy = (t.y + dp) * silu_t(zv.y) * w;
        s1.x += gx; s1.y += gy;
        s2.x = fmaf(gx, mv.x - mu.x, s2.x); s2.y = fmaf(gy, mv.y - mu.y, s2.y);
    }
    s1 = slice_sum(s1, sm, pp, q);
    s2 = slice_sum(s2, sm, pp, q);
    const float2 k1 = make_float2(s1.x * invC, s1.y * invC);
    const float2 k2 = make_float2(s2.x * invC * rstd.x * rstd.x, s2.y * invC * rstd.y * rstd.y);
    in_t* __restrict__ dm = reinterpret_cast<in_t*>(p.dm) + (int64_t)b * C * p.L + l;
    in_t* __restrict__ dz = reinterpret_cast<in_t*>(p.dz) + (int64_t)b * p.dz_bs + l;
    for (int c = c0; c < c1; ++c) {
        const float2 t0 = Pair<in_t>::ld(dy2 + (int64_t)c * p.L);
        const float2 zv = Pair<in_t>::ld(z + (int64_t)c * p.z_cs);
        const float2 mv = *reinterpret_cast<const float2*>(m + (int64_t)c * p.L);
        const float dp = dpool ? dpool[c] : 0.f, w = p.w[c], bb = p.b[c];
        const float2 t = make_float2(t0.x + dp, t0.y + dp);
        const float2 d = make_float2(mv.x - mu.x, mv.y - mu.y);
        const float gx = t.x * silu_t(zv.x) * w, gy = t.y * silu_t(zv.y) * w;
        Pair<in_t>::st(dm + (int64_t)c * p.L, make_float2(rstd.x * (gx - k1.x - d.x * k2.x), rstd.y * (gy - k1.y - d.y * k2.y)));
        const float nx = fmaf(d.x * rstd.x, w, bb), ny = fmaf(d.y * rstd.y, w, bb);
        Pair<in_t>::st(dz + (int64_t)c * p.dz_cs, make_float2(t.x * nx * dsilu_t(zv.x), t.y * ny * dsilu_t(zv.y)));
    }
}

// ------------------------------------------------------------------------------------------ depthwise 3x3 backward
// gradient w.r.t. the conv OUTPUT before the activation (the conv is recomputed, nothing but its input was saved):
//   mode 0: v = dw(x[c]) + b;  dv = g * silu'(v)
//   mode 1: v1 = dw(x[c]) + b[c], v2 = dw(x[c+Co]) + b[c+Co];  dv[c] = g * v2 * gelu'(v1),  dv[c+Co] = g * gelu(v1)
template <typename in_t>
__global__ void __launch_bounds__(256) dwconv_bwd_pre_kernel(const DwBwdParams p) {
    pdl_trigger();
    pdl_wait();
    const int c = blockIdx.y % p.Cout, b = blockIdx.y / p.Cout;
    const int L = p.H * p.W;
    const in_t* __restrict__ xb = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;
    const in_t* __restrict__ g = reinterpret_cast<const in_t*>(p.g) + (int64_t)b * p.g_bs + (int64_t)c * p.g_cs;
    in_t* __restrict__ dv = reinterpret_cast<in_t*>(p.dv) + (int64_t)b * p.dv_bs;
    float w0[9], w1[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        w0[i] = p.w[c * 9 + i];
        w1[i] = p.mode ? p.w[(c + p.Cout) * 9 + i] : 0.f;
    }
    const float b0 = p.bias ? p.bias[c] : 0.f, b1 = (p.bias && p.mode) ? p.bias[c + p.Cout] : 0.f;
    if (p.vec_ok) {  // 8-pixel strips, 16 B loads / stores
        constexpr int V = Vec<in_t>::N;
        for (int i = (blockIdx.x * 256 + threadIdx.x) * 8; i < L; i += gridDim.x * 256 * 8) {
            const int h = i / p.W, w = i % p.W;
            float a0[8], a1[8], gv[8], o0[8], o1[8];
            dw_strip<in_t>(xb + (int64_t)c * p.x_cs, w0, h, w, p.H, p.W, b0, a0);
#pragma unroll
            for (int j = 0; j < 8 / V; ++j) load_vec<in_t>(g + i + j * V, gv + j * V, V, true);
            if (p.mode == 0) {
#pragma unroll
                for (int j = 0; j < 8; ++j) o0[j] = gv[j] * dsilu_t(a0[j]);
            } else {
                dw_strip<in_t>(xb + (int64_t)(c + p.Cout) * p.x_cs, w1, h, w, p.H, p.W, b1, a1);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o0[j] = gv[j] * a1[j] * dgelu_t(a0[j]);
                    o1[j] = gv[j] * gelu_t(a0[j]);
                }
#pragma unroll
                for (int j = 0; j < 8 / V; ++j) store_vec<in_t>(dv + (int64_t)(c + p.Cout) * p.dv_cs + i + j * V, o1 + j * V, V, true);
            }
#pragma unroll
            for (int j = 0; j < 8 / V; ++j) store_vec<in_t>(dv + (int64_t)c * p.dv_cs + i + j * V, o0 + j * V, V, true);
        }
        return;
    }
    for (int i = blockIdx.x * 256 + threadIdx.x; i < L; i += gridDim.x * 256) {
        const int h = i / p.W, w = i % p.W;
        const float v = dw_at<in_t>(xb + (int64_t)c * p.x_cs, w0, h, w, p.H, p.W) + b0;
        const float gv = to_f32<in_t>(g[i]);
        if (p.mode == 0) {
            dv[(int64_t)c * p.dv_cs + i] = from_f32<in_t>(gv * dsilu_t(v));
        } else {
            const float v2 = dw_at<in_t>(xb + (int64_t)(c + p.Cout) * p.x_cs, w1, h, w, p.H, p.W) + b1;
            dv[(int64_t)c * p.dv_cs + i] = from_f32<in_t>(gv * v2 * dgelu_t(v));
            dv[(int64_t)(c + p.Cout) * p.dv_cs + i] = from_f32<in_t>(gv * gelu_t(v));
        }
    }
}

// weight / bias gradient of the depthwise conv: grid (channels, B);  dw[c][j] += sum_pix dv[pix] * x[pix + tap_j];  db[c] += sum dv
template <typename in_t>
__global__ void __launch_bounds__(256) dwconv_wgrad_kernel(const DwBwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sred[8];
    const int c = blockIdx.x, b = blockIdx.y;
    const int L = p.H * p.W;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs + (int64_t)c * p.x_cs;
    const in_t* __restrict__ dv = reinterpret_cast<const in_t*>(p.dv) + (int64_t)b * p.dv_bs + (int64_t)c * p.dv_cs;
    float acc[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) acc[j] = 0.f;
    if (p.vec_ok) {  // 8-pixel strips: three 16 B row loads of x (+2 halo scalars each) against one 16 B load of dv
        constexpr int V = Vec<in_t>::N;
        for (int i = threadIdx.x * 8; i < L; i += 256 * 8) {
            const int h = i / p.W, w0 = i % p.W;
            float d[8];
#pragma unroll
            for (int j = 0; j < 8 / V; ++j) load_vec<in_t>(dv + i + j * V, d + j * V, V, true);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[9] += d[j];
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy) {
                const int hh = h + dy;
                if (hh < 0 || hh >= p.H) continue;
                const in_t* __restrict__ row = x + (int64_t)hh * p.W;
                float v[10];
                v[0] = w0 > 0 ? to_f32<in_t>(row[w0 - 1]) : 0.f;
                v[9] = w0 + 8 < p.W ? to_f32<in_t>(row[w0 + 8]) : 0.f;
#pragma unroll
                for (int j = 0; j < 8 / V; ++j) load_vec<in_t>(row + w0 + j * V, v + 1 + j * V, V, true);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    acc[(dy + 1) * 3 + 0] = fmaf(d[j], v[j], acc[(dy + 1) * 3 + 0]);
                    acc[(dy + 1) * 3 + 1] = fmaf(d[j], v[j + 1], acc[(dy + 1) * 3 + 1]);
                    acc[(dy + 1) * 3 + 2] = fmaf(d[j], v[j + 2], acc[(dy + 1) * 3 + 2]);
                }
            }
        }
    } else
    for (int i = threadIdx.x; i < L; i += 256) {
        const int h = i / p.W, w = i % p.W;
        const float d = to_f32<in_t>(dv[i]);
        acc[9] += d;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int hh = h + dy;
            if (hh < 0 || hh >= p.H) continue;
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int ww = w + dx;
                if (ww < 0 || ww >= p.W) continue;
                acc[(dy + 1) * 3 + dx + 1] = fmaf(d, to_f32<in_t>(x[hh * p.W + ww]), acc[(dy + 1) * 3 + dx + 1]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 10; ++j) {
        const float t = block_sum_256(acc[j], sred);
        if (threadIdx.x == 0) {
            if (j < 9) atomicAdd(p.dwgt + c * 9 + j, t);
            else if (p.dbias) atomicAdd(p.dbias + c, t);
        }
    }
}

// ------------------------------------------------------------------------------------------ channel gate backward
// forward (prologue of out_conv): yg = y2 * (1 + c[b,k]) (mode 1) or y2 + c[b,k] (mode 2).  grid (C, B).
template <typename in_t>
__global__ void __launch_bounds__(256) gate_bwd_kernel(const GateBwdParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sred[8];
    const int c = blockIdx.x, b = blockIdx.y;
    const in_t* __restrict__ dyg = reinterpret_cast<const in_t*>(p.dyg) + ((int64_t)b * p.C + c) * p.L;
    const in_t* __restrict__ y2 = reinterpret_cast<const in_t*>(p.y2) + ((int64_t)b * p.C + c) * p.L;
    in_t* __restrict__ dy2 = reinterpret_cast<in_t*>(p.dy2) + ((int64_t)b * p.C + c) * p.L;
    const float gate = p.gate[(int64_t)b * p.C + c];
    float acc = 0.f;
    for (int l = threadIdx.x; l < p.L; l += 256) {
        const float d = to_f32<in_t>(dyg[l]);
        if (p.mode == 1) {
            acc = fmaf(d, to_f32<in_t>(y2[l]), acc);
            dy2[l] = from_f32<in_t>(d * (1.f + gate));
        } else {
            acc += d;
            dy2[l] = dyg[l];
        }
    }
    const float t = block_sum_256(acc, sred);
    if (threadIdx.x == 0) p.dgate[(int64_t)b * p.C + c] = t;
}

// ------------------------------------------------------------------------------------------ fused Adam(W) + clip + EMA
// One pass over the flat fp32 parameter / gradient / moment buffers (reference: optimizer_g.step() + model_ema() +
// clip_grad_norm_, SRGAN/VmambaIR/models/MambaSISR_model.py:141-147, Deraining/basicsr/models/image_restoration_model.py:165-173,
// Deraining/basicsr/models/base_model.py:54-62) instead of ~1 500 per-tensor launches.  `state` (device, 4 floats):
// [0] step count (incremented by the trailing 1-thread kernel: graph replays advance it), [1] sum of squared gradients.
__global__ void __launch_bounds__(256) sqsum_kernel(const float* __restrict__ g, long n, float* __restrict__ state) {
    __shared__ float sred[8];
    float acc = 0.f;
    for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long)gridDim.x * 256) acc = fmaf(g[i], g[i], acc);
    const float t = block_sum_256(acc, sred);
    if (threadIdx.x == 0) atomicAdd(state + 1, t);
}

__global__ void __launch_bounds__(256) fused_adam_kernel(const AdamParams p) {
    const float step = p.state[0] + 1.f;
    const float bc1 = 1.f - powf(p.beta1, step), bc2 = 1.f - powf(p.beta2, step);
    float gs = p.grad_scale;
    if (p.max_norm > 0.f) {  // clip_grad_norm_: scale by max_norm / (total_norm + 1e-6), clamped to 1
        const float total = sqrtf(p.state[1]) * p.grad_scale;
        gs *= fminf(p.max_norm / (total + 1e-6f), 1.f);
    }
    const float step_size = p.lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
    for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < p.n; i += (long)gridDim.x * 256) {
        float w = p.param[i];
        float g = p.grad[i] * gs;
        if (p.weight_decay != 0.f) {
            if (p.decoupled) w -= p.lr * p.weight_decay * w;  // AdamW
            else g = fmaf(p.weight_decay, w, g);                // Adam (L2)
        }
        const float m = fmaf(p.beta1, p.m[i], (1.f - p.beta1) * g);
        const float v = fmaf(p.beta2, p.v[i], (1.f - p.beta2) * g * g);
        p.m[i] = m;
        p.v[i] = v;
        w -= step_size * m / (sqrtf(v) * inv_sqrt_bc2 + p.eps);
        p.param[i] = w;
        if (p.ema) p.ema[i] = fmaf(p.ema_decay, p.ema[i], (1.f - p.ema_decay) * w);
        if (p.zero_grad) p.grad[i] = 0.f;
    }
}

__global__ void adam_step_inc_kernel(float* state) {
    state[0] += 1.f;
    state[1] = 0.f;
}

int fused_adam_launch(const AdamParams& p, cudaStream_t stream) {
    const int blocks = (int)((p.n + 255) / 256 < num_sms() * 8 ? (p.n + 255) / 256 : num_sms() * 8);
    if (p.max_norm > 0.f) sqsum_kernel<<<blocks, 256, 0, stream>>>(p.grad, p.n, p.state);
    fused_adam_kernel<<<blocks, 256, 0, stream>>>(p);
    adam_step_inc_kernel<<<1, 1, 0, stream>>>(p.state);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------ per-step weight preparation
// One launch per OSS block and step instead of ~35 small torch kernels: every 1x1-conv weight of the block in kernel layout
// (compute dtype, rows zero-padded to 16 elements) together with its transpose (the data-gradient GEMMs), the folded
// x_proj / dt_proj matrix  big[k] = [W_dt,k W_x,k[:R] ; W_x,k[R:]]  (MambaSISR6_arch.py:409-414 as ONE contraction on the
// un-permuted x), A = -exp(A_logs) and the spatially flipped depthwise taps (transposed conv of the backward pass).
// job types: 0 convert (M x K -> M x ld), 1 convert + transpose (M x K -> K x ld), 2 fold (writes big and its transpose),
//            3 A = -exp(src) fp32, 4 flip the 9 taps fp32
template <typename out_t>
__global__ void __launch_bounds__(256) prep_weights_kernel(const PrepParams p) {
    const PrepJob j = p.jobs[blockIdx.y];
    const long stride = (long)gridDim.x * 256;
    const long i0 = (long)blockIdx.x * 256 + threadIdx.x;
    if (j.type == 0 || j.type == 1) {
        out_t* dst = reinterpret_cast<out_t*>(j.dst);
        const int rows = j.type == 0 ? j.M : j.K, cols = j.type == 0 ? j.K : j.M;
        for (long i = i0; i < (long)rows * j.ld; i += stride) {
            const int r = (int)(i / j.ld), c = (int)(i % j.ld);
            float v = 0.f;
            if (c < cols) v = j.type == 0 ? j.src[(long)r * j.K + c] : j.src[(long)c * j.K + r];
            dst[i] = from_f32<out_t>(v);
        }
    } else if (j.type == 2) {  // src = x_proj (4, R+2N, C), src2 = dt_w (4, C, R): M = C, K = R, N2 = 2N
        out_t* big = reinterpret_cast<out_t*>(j.dst);
        out_t* bigT = reinterpret_cast<out_t*>(j.dst2);
        const int C = j.M, R = j.K, N2 = j.N2, RN = R + N2, rows = 4 * (C + N2);
        for (long i = i0; i < (long)rows * C; i += stride) {
            const int row = (int)(i / C), c = (int)(i % C);
            const int k = row / (C + N2), d = row % (C + N2);
            float v;
            if (d < C) {
                v = 0.f;
                for (int r = 0; r < R; ++r) v = fmaf(j.src2[((long)k * C + d) * R + r], j.src[((long)k * RN + r) * C + c], v);
            } else {
                v = j.src[((long)k * RN + R + (d - C)) * C + c];
            }
            big[(long)row * j.ld + c] = from_f32<out_t>(v);
            bigT[(long)c * j.ld2 + row] = from_f32<out_t>(v);
        }
        // zero the padding columns
        for (long i = i0; i < (long)rows * (j.ld - C); i += stride) big[(i / (j.ld - C)) * j.ld + C + i % (j.ld - C)] = from_f32<out_t>(0.f);
        for (long i = i0; i < (long)C * (j.ld2 - rows); i += stride) bigT[(i / (j.ld2 - rows)) * j.ld2 + rows + i % (j.ld2 - rows)] = from_f32<out_t>(0.f);
    } else if (j.type == 3) {
        float* dst = reinterpret_cast<float*>(j.dst);
        for (long i = i0; i < (long)j.M * j.K; i += stride) dst[i] = -expf(j.src[i]);
    } else {
        float* dst = reinterpret_cast<float*>(j.dst);
        for (long i = i0; i < (long)j.M * 9; i += stride) dst[i] = j.src[(i / 9) * 9 + (8 - i % 9)];
    }
}

int prep_weights_launch(const PrepParams& p, int dtype, cudaStream_t stream) {
    dim3 grid(64, p.njobs);
    switch (dtype) {
        case VMB_F32: prep_weights_kernel<float><<<grid, 256, 0, stream>>>(p); break;
        case VMB_BF16: prep_weights_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(p); break;
        case VMB_F16: prep_weights_kernel<__half><<<grid, 256, 0, stream>>>(p); break;
        default: set_error("prep_weights: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// out = add + sum_k x4[:, k]   (the four un-permuted direction gradients of u joined with the x_proj data gradient)
template <typename in_t>
__global__ void __launch_bounds__(256) sum4_add_kernel(const in_t* __restrict__ x4, const in_t* __restrict__ add, in_t* __restrict__ out,
                                                       long per_dir, long per_batch, long total) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = Vec<in_t>::N;
    for (long i = ((long)blockIdx.x * 256 + threadIdx.x) * V; i < total; i += (long)gridDim.x * 256 * V) {
        const long b = i / per_dir, o = i % per_dir;
        float acc[V], t[V];
        load_vec<in_t>(add + i, acc, V, true);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            load_vec<in_t>(x4 + b * per_batch + k * per_dir + o, t, V, true);
#pragma unroll
            for (int e = 0; e < V; ++e) acc[e] += t[e];
        }
        store_vec<in_t>(out + i, acc, V, true);
    }
}

// ---------------------------------------------------------------------------------------------------- launchers
#define VMB_DISPATCH(dtype, KERN, grid, block, ...)                                                    \
    switch (dtype) {                                                                                   \
        case VMB_F32: VMB_CUDA(launch_pdl(KERN<float>, grid, block, 0, stream, __VA_ARGS__)); break;    \
        case VMB_BF16: VMB_CUDA(launch_pdl(KERN<__nv_bfloat16>, grid, block, 0, stream, __VA_ARGS__)); break; \
        case VMB_F16: VMB_CUDA(launch_pdl(KERN<__half>, grid, block, 0, stream, __VA_ARGS__)); break;   \
        default: set_error("unsupported dtype %d", dtype); return VMB_ERR_INVALID;                     \
    }

static inline bool even(int64_t v) { return (v & 1) == 0; }
static inline bool al8(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 7) == 0; }

int ln_fwd_launch(const LnFwdParams& p, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.B <= 65535, "layernorm_fwd: batch > 65535");
    if (p.L >= 2 && even(p.L) && even(p.x_bs) && even(p.x_cs) && even(p.y_bs) && even(p.y_cs) && al8(p.x) && (!p.y || al8(p.y)) && p.C >= PX_Q) {
        VMB_DISPATCH(dtype, ln_fwd_px_kernel, dim3((p.L / 2 + PX_PAIRS - 1) / PX_PAIRS, p.B), dim3(256), p);
        VMB_CUDA(cudaGetLastError());
        return VMB_OK;
    }
    VMB_DISPATCH(dtype, ln_fwd_kernel, dim3((p.L + 127) / 128, p.B), dim3(128), p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int ln_bwd_launch(const LnBwdParams& p, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.B <= 65535 && p.C <= 65535, "layernorm_bwd: batch / channels > 65535");
    if (!p.dx) {  // parameter gradients only (the statistics of an earlier data-gradient call)
        VMB_DISPATCH(dtype, ln_bwd_dwdb_kernel, dim3(p.C, p.B), dim3(256), p);
        VMB_CUDA(cudaGetLastError());
        return VMB_OK;
    }
    if (p.L >= 2 && even(p.L) && even(p.x_bs) && even(p.x_cs) && even(p.g_bs) && even(p.g_cs) && even(p.a_bs) && even(p.a_cs) && even(p.dx_bs) &&
        even(p.dx_cs) && al8(p.x) && al8(p.g) && al8(p.dx) && (!p.add || al8(p.add)) && p.C >= PX_Q) {
        VMB_DISPATCH(dtype, ln_bwd_dx_px_kernel, dim3((p.L / 2 + PX_PAIRS - 1) / PX_PAIRS, p.B), dim3(256), p);
    } else
    VMB_DISPATCH(dtype, ln_bwd_dx_kernel, dim3((p.L + 127) / 128, p.B), dim3(128), p);
    if (p.dw) VMB_DISPATCH(dtype, ln_bwd_dwdb_kernel, dim3(p.C, p.B), dim3(256), p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int merge_bwd_launch(const MergeBwdParams& p, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.B <= 65535 && p.C <= 65535, "merge_bwd: batch / channels > 65535");
    if (!p.dm) {  // parameter gradients only
        VMB_DISPATCH(dtype, merge_bwd_dwdb_kernel, dim3(p.C, p.B), dim3(256), p);
        VMB_CUDA(cudaGetLastError());
        return VMB_OK;
    }
    if (p.L >= 2 && even(p.L) && even(p.z_bs) && even(p.z_cs) && even(p.dz_bs) && even(p.dz_cs) && al8(p.z) && al8(p.dz) && al8(p.dy2) &&
        al8(p.dm) && (reinterpret_cast<uintptr_t>(p.stats) & 15) == 0 && p.C >= PX_Q) {
        VMB_DISPATCH(dtype, merge_bwd_dx_px_kernel, dim3((p.L / 2 + PX_PAIRS - 1) / PX_PAIRS, p.B), dim3(256), p);
    } else
    VMB_DISPATCH(dtype, merge_bwd_dx_kernel, dim3((p.L + 127) / 128, p.B), dim3(128), p);
    if (p.dw) VMB_DISPATCH(dtype, merge_bwd_dwdb_kernel, dim3(p.C, p.B), dim3(256), p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int dwconv_bwd_launch(const DwBwdParams& p, int dtype, cudaStream_t stream) {
    const int L = p.H * p.W;
    const int chans = p.mode ? 2 * p.Cout : p.Cout;
    VMB_CHECK((long)p.B * chans <= 65535, "dwconv_bwd: batch * channels > 65535");
    const int per = p.vec_ok ? 8 : 1;
    VMB_DISPATCH(dtype, dwconv_bwd_pre_kernel, dim3((L / per + 255) / 256 > 0 ? (L / per + 255) / 256 : 1, p.B * p.Cout), dim3(256), p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int dwconv_wgrad_launch(const DwBwdParams& p, int dtype, cudaStream_t stream) {
    const int chans = p.mode ? 2 * p.Cout : p.Cout;
    VMB_CHECK(chans <= 65535 && p.B <= 65535, "dwconv_wgrad: grid too large");
    VMB_DISPATCH(dtype, dwconv_wgrad_kernel, dim3(chans, p.B), dim3(256), p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int gate_bwd_launch(const GateBwdParams& p, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.B <= 65535 && p.C <= 65535, "gate_bwd: grid too large");
    VMB_DISPATCH(dtype, gate_bwd_kernel, dim3(p.C, p.B), dim3(256), p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb

// ---------------------------------------------------------------------------------------------------- C ABI
using namespace vmb;
static inline bool tdt_ok(int d) { return d == VMB_F32 || d == VMB_BF16 || d == VMB_F16; }

extern "C" int vmb_layernorm_fwd(const vmb_ln_fwd_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->w && (a->y || a->stats), "layernorm_fwd: null pointer");
    VMB_CHECK(tdt_ok(a->dtype) && (a->mode == 1 || a->mode == 2) && (a->mode == 2 || a->b), "layernorm_fwd: bad dtype / mode / bias");
    VMB_CHECK(a->batch > 0 && a->C > 0 && a->L > 0, "layernorm_fwd: bad sizes");
    LnFwdParams p{a->x, a->w, a->b, a->y, a->stats, a->batch, a->C, a->L, a->mode, a->x_bs, a->x_cs, a->y_bs, a->y_cs};
    return ln_fwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_layernorm_bwd(const vmb_ln_bwd_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->g && a->w && (a->dx || a->dw) && a->stats, "layernorm_bwd: null pointer");
    VMB_CHECK(tdt_ok(a->dtype) && (a->mode == 1 || a->mode == 2), "layernorm_bwd: bad dtype / mode");
    VMB_CHECK(a->batch > 0 && a->C > 0 && a->L > 0, "layernorm_bwd: bad sizes");
    LnBwdParams p{a->x, a->g, a->add, a->w, a->dx, a->dw, a->db, a->stats, a->batch, a->C, a->L, a->mode,
                  a->x_bs, a->x_cs, a->g_bs, a->g_cs, a->a_bs, a->a_cs, a->dx_bs, a->dx_cs};
    return ln_bwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_merge_norm_gate_bwd(const vmb_merge_bwd_args* a, void* stream) {
    VMB_CHECK(a && a->merged && a->stats && a->z && a->dy2 && a->w && a->b, "merge_bwd: null pointer");
    VMB_CHECK((a->dm && a->dz) || (!a->dm && !a->dz && a->dw), "merge_bwd: dm and dz together (data gradients), or neither (parameter gradients only)");
    VMB_CHECK((a->dw == nullptr) == (a->db == nullptr), "merge_bwd: dw and db together");
    VMB_CHECK(tdt_ok(a->dtype) && a->batch > 0 && a->C > 0 && a->L > 0, "merge_bwd: bad arguments");
    MergeBwdParams p{a->merged, a->stats, a->z, a->dy2, a->dpooled, a->w, a->b, a->dm, a->dz, a->dw, a->db,
                     a->batch, a->C, a->L, a->z_bs, a->z_cs, a->dz_bs, a->dz_cs};
    return merge_bwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_dwconv3x3_bwd(const vmb_dwconv_bwd_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->w && a->dv && (a->g || a->dw), "dwconv_bwd: null pointer");
    VMB_CHECK(tdt_ok(a->dtype) && (a->mode == 0 || a->mode == 1) && a->batch > 0 && a->c_out > 0 && a->H > 0 && a->W > 0, "dwconv_bwd: bad arguments");
    DwBwdParams p{a->x, a->w, a->bias, a->g, a->dv, a->dw, a->dbias, a->batch, a->c_out, a->H, a->W, a->mode,
                  a->x_bs, a->x_cs, a->g_bs, a->g_cs, a->dv_bs, a->dv_cs, false};
    {
        auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
        p.vec_ok = a->W % 8 == 0 && al16(a->x) && (!a->g || al16(a->g)) && al16(a->dv) && a->x_bs % 8 == 0 && a->x_cs % 8 == 0 &&
                   (!a->g || (a->g_bs % 8 == 0 && a->g_cs % 8 == 0)) && a->dv_bs % 8 == 0 && a->dv_cs % 8 == 0;
    }
    int rc = VMB_OK;
    if (a->g) rc = dwconv_bwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream));  // g == NULL: dv is an input, weight gradients only
    if (rc != VMB_OK || !a->dw) return rc;
    return dwconv_wgrad_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_fused_adam(const vmb_adam_args* a, void* stream) {
    VMB_CHECK(a && a->param && a->grad && a->exp_avg && a->exp_avg_sq && a->state, "fused_adam: null pointer");
    VMB_CHECK(a->n > 0 && a->lr >= 0.f && a->beta1 >= 0.f && a->beta1 < 1.f && a->beta2 >= 0.f && a->beta2 < 1.f && a->eps > 0.f,
              "fused_adam: bad hyper-parameters");
    AdamParams p{a->param, a->grad, a->exp_avg, a->exp_avg_sq, a->ema, a->state, a->n, a->lr, a->beta1, a->beta2, a->eps,
                 a->weight_decay, a->decoupled_weight_decay, a->grad_scale, a->max_grad_norm, a->ema_decay, a->zero_grad};
    return fused_adam_launch(p, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_prep_block_weights(const vmb_prep_args* a, void* stream) {
    VMB_CHECK(a && a->njobs > 0 && a->njobs <= VMB_PREP_MAX_JOBS, "prep_block_weights: 1..%d jobs", VMB_PREP_MAX_JOBS);
    PrepParams p{};
    p.njobs = a->njobs;
    for (int i = 0; i < a->njobs; ++i) {
        const vmb_prep_job& j = a->jobs[i];
        VMB_CHECK(j.src && j.dst && j.type >= 0 && j.type <= 4 && j.M > 0 && (j.type == 4 || j.K > 0), "prep_block_weights: bad job %d", i);
        VMB_CHECK(j.type != 2 || (j.src2 && j.dst2), "prep_block_weights: fold job %d needs src2 / dst2", i);
        p.jobs[i] = PrepJob{j.src, j.src2, j.dst, j.dst2, j.type, j.M, j.K, j.N2, j.ld, j.ld2};
    }
    return prep_weights_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_sum4_add(const void* x4, const void* add, void* out, int batch, long per_dir, int dtype, void* stream) {
    VMB_CHECK(x4 && add && out && batch > 0 && per_dir > 0, "sum4_add: bad arguments");
    const int v = dtype == VMB_F32 ? 4 : 8;
    VMB_CHECK(per_dir % v == 0 && ((reinterpret_cast<uintptr_t>(x4) | reinterpret_cast<uintptr_t>(add) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
              "sum4_add: 16 B aligned contiguous tensors");
    const long total = (long)batch * per_dir;
    const int blocks = (int)((total / v + 255) / 256 < num_sms() * 8 ? (total / v + 255) / 256 : num_sms() * 8);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (dtype) {
        case VMB_F32: VMB_CUDA(launch_pdl(sum4_add_kernel<float>, dim3(blocks), dim3(256), 0, st, (const float*)x4, (const float*)add, (float*)out, per_dir, 4 * per_dir, total)); break;
        case VMB_BF16: VMB_CUDA(launch_pdl(sum4_add_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, st, (const __nv_bfloat16*)x4, (const __nv_bfloat16*)add, (__nv_bfloat16*)out, per_dir, 4 * per_dir, total)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(sum4_add_kernel<__half>, dim3(blocks), dim3(256), 0, st, (const __half*)x4, (const __half*)add, (__half*)out, per_dir, 4 * per_dir, total)); break;
        default: set_error("sum4_add: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_channel_gate_bwd(const vmb_gate_bwd_args* a, void* stream) {
    VMB_CHECK(a && a->dyg && a->y2 && a->gate && a->dy2 && a->dgate, "channel_gate_bwd: null pointer");
    VMB_CHECK(tdt_ok(a->dtype) && (a->mode == 1 || a->mode == 2) && a->batch > 0 && a->C > 0 && a->L > 0, "channel_gate_bwd: bad arguments");
    GateBwdParams p{a->dyg, a->y2, a->gate, a->dy2, a->dgate, a->batch, a->C, a->L, a->mode};
    return gate_bwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}
