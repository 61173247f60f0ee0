// Memory-bound stages of the fused OSS block (reference: SRGAN/VmambaIR/archs/MambaSISR6_arch.py):
//   dwconv3x3_kernel       depthwise 3x3 + bias + SiLU (SS2D_1.conv2d/act :286-294,490-491) or the EFFN's
//                          depthwise 3x3 + exact-GELU gate (FeedForward :215-216)
//   cross_scan_kernel      the four direction orders as index arithmetic (cross_scan_2d :401-404 / CrossScan):
//                          out[k][row][l] = src_k[row][pi_k(l)],  pi_0 = id, pi_1 = column-major, pi_2/3 = reversed
//   merge_norm_gate_kernel inverse orders + 4-way sum in the reference's fp32 order (:427-430), out_norm
//                          LayerNorm over C (:433), gate with SiLU(z) (:493) and the per-(b,c) pooled sums
//                          for the channel branch (AdaptiveAvgPool2d, :441)
//   channel_branch_kernel  the whole channel OSS (cforward_corev1 :438-483 and the 3 other variants) for one
//                          image in one CTA: conv_cin, xc_proj, dtc_proj, bidirectional scan over L=C,
//                          conv_cout, channel_norm -> c[b][C]
#include <stdlib.h>

#include "common.cuh"
#include "oss_params.h"
#include "dwconv_common.cuh"

namespace vmb {

__device__ __forceinline__ float silu2(float v) { return v * rcp_approx(1.f + ex2(-v * kLog2e)); }
// erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, branch-free, 2 MUFU): GELU stays the exact-erf form of F.gelu
__device__ __forceinline__ float erf_as(float x) {
    const float ax = fabsf(x);
    const float t = rcp_approx(fmaf(0.3275911f, ax, 1.f));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    const float r = 1.f - poly * t * ex2(-ax * ax * kLog2e);
    return copysignf(r, x);
}
__device__ __forceinline__ float gelu_exact(float v) { return 0.5f * v * (1.f + erf_as(v * 0.70710678118654752f)); }

// ------------------------------------------------------------------------------------------ depthwise 3x3

template <typename in_t>
__global__ void __launch_bounds__(256) dwconv3x3_kernel(const DwParams p) {
    pdl_trigger();
    pdl_wait();
    const int c = blockIdx.y % p.Cout, b = blockIdx.y / p.Cout;
    const int L = p.H * p.W;
    const in_t* __restrict__ xb = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;
    in_t* __restrict__ ob = reinterpret_cast<in_t*>(p.out) + (int64_t)b * p.o_bs + (int64_t)c * p.o_cs;
    float w0[9], w1[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        w0[i] = p.w[c * 9 + i];
        w1[i] = p.mode == 1 ? p.w[(c + p.Cout) * 9 + i] : 0.f;
    }
    const float b0 = p.bias ? p.bias[c] : 0.f, b1 = (p.bias && p.mode == 1) ? p.bias[c + p.Cout] : 0.f;
    if (p.vec_ok) {
        constexpr int V = Vec<in_t>::N;
        for (int i = (blockIdx.x * blockDim.x + threadIdx.x) * 8; i < L; i += gridDim.x * blockDim.x * 8) {
            const int h = i / p.W, w = i % p.W;
            float a0[8], a1[8];
            dw_strip<in_t>(xb + (int64_t)c * p.x_cs, w0, h, w, p.H, p.W, b0, a0);
            if (p.mode == 0) {
#pragma unroll
                for (int j = 0; j < 8; ++j) a0[j] = silu2(a0[j]);
            } else if (p.mode == 1) {
                dw_strip<in_t>(xb + (int64_t)(c + p.Cout) * p.x_cs, w1, h, w, p.H, p.W, b1, a1);
#pragma unroll
                for (int j = 0; j < 8; ++j) a0[j] = gelu_exact(a0[j]) * a1[j];
            }
#pragma unroll
            for (int j = 0; j < 8 / V; ++j) store_vec<in_t>(ob + i + j * V, a0 + j * V, V, true);
        }
        return;
    }
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x) {
        const int h = i / p.W, w = i % p.W;
        float v = dw_at<in_t>(xb + (int64_t)c * p.x_cs, w0, h, w, p.H, p.W) + b0;
        if (p.mode == 0) {
            v = silu2(v);
        } else if (p.mode == 1) {
            const float g = dw_at<in_t>(xb + (int64_t)(c + p.Cout) * p.x_cs, w1, h, w, p.H, p.W) + b1;
            v = gelu_exact(v) * g;
        }
        ob[i] = from_f32<in_t>(v);
    }
}

// Row-block version (W a power of two in [8, 256], H % 4 == 0, 16 B aligned rows): one thread = an 8-pixel strip of FOUR
// consecutive output rows, so six 16 B row loads feed four outputs (the strip kernel: three loads per output), and the left / right
// halo pixels come from the neighbouring lanes' vectors by shuffle instead of two scalar loads per row.  The loads are split from the
// arithmetic: all six row vectors (twelve in the gated mode: both channel sets) are requested before the first use, so one thread
// has 6-12 loads in flight instead of stalling on each row load in turn.  Same fmaf order as the strip kernel (dy ascending, dx
// ascending; out-of-image taps contribute fmaf(k, 0, acc) = acc), so the results are bit-identical.
template <typename in_t>
__device__ __forceinline__ void dw_rows4_load(const in_t* __restrict__ xc, int h0, int w0, int H, int W,
                                              uint4 (&raw)[6][8 / Vec<in_t>::N]) {
    constexpr int V = Vec<in_t>::N;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const int hh = h0 - 1 + r;
        const bool in = hh >= 0 && hh < H;
#pragma unroll
        for (int j = 0; j < 8 / V; ++j) raw[r][j] = in ? ldg128(xc + (int64_t)hh * W + w0 + j * V) : make_uint4(0u, 0u, 0u, 0u);
    }
}
template <typename in_t>
__device__ __forceinline__ void dw_rows4_compute(const uint4 (&raw)[6][8 / Vec<in_t>::N], const float* __restrict__ w9, int s, int S,
                                                 float bias, float (*acc)[8]) {
    constexpr int V = Vec<in_t>::N;
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[o][i] = bias;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        float v[10];
        if constexpr (sizeof(in_t) == 2) {
            unpack8<in_t>(raw[r][0], v + 1);
        } else {
#pragma unroll
            for (int j = 0; j < 8 / V; ++j) {
                v[1 + 4 * j] = __uint_as_float(raw[r][j].x); v[2 + 4 * j] = __uint_as_float(raw[r][j].y);
                v[3 + 4 * j] = __uint_as_float(raw[r][j].z); v[4 + 4 * j] = __uint_as_float(raw[r][j].w);
            }
        }
        const float left = __shfl_up_sync(0xffffffffu, v[8], 1, S), right = __shfl_down_sync(0xffffffffu, v[1], 1, S);
        v[0] = s > 0 ? left : 0.f;
        v[9] = s < S - 1 ? right : 0.f;
#pragma unroll
        for (int o = 0; o < 4; ++o) {
            const int dy = r - 1 - o;
            if (dy >= -1 && dy <= 1) {
                const float k0 = w9[(dy + 1) * 3], k1 = w9[(dy + 1) * 3 + 1], k2 = w9[(dy + 1) * 3 + 2];
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[o][i] = fmaf(k2, v[i + 2], fmaf(k1, v[i + 1], fmaf(k0, v[i], acc[o][i])));
            }
        }
    }
}

template <typename in_t>
__global__ void __launch_bounds__(256, 2) dwconv3x3_rows4_pre_kernel(const DwParams p, const int S, const int log2_tpp, const long total) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = Vec<in_t>::N;
    const long gt = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = gt < total;
    const long g = valid ? gt : total - 1;      // clamped: every lane takes part in the shuffles
    const int plane = (int)(g >> log2_tpp), t = (int)(g & ((1L << log2_tpp) - 1));
    const int c = plane % p.Cout, b = plane / p.Cout;
    const int s = t & (S - 1), h0 = (t / S) * 4, w0 = s * 8;
    const in_t* __restrict__ xb = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;
    in_t* __restrict__ ob = reinterpret_cast<in_t*>(p.out) + (int64_t)b * p.o_bs + (int64_t)c * p.o_cs;
    uint4 raw0[6][8 / V], raw1[6][8 / V];
    dw_rows4_load<in_t>(xb + (int64_t)c * p.x_cs, h0, w0, p.H, p.W, raw0);
    if (p.mode == 1) dw_rows4_load<in_t>(xb + (int64_t)(c + p.Cout) * p.x_cs, h0, w0, p.H, p.W, raw1);
    float w0k[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) w0k[i] = p.w[c * 9 + i];
    float a0[4][8];
    dw_rows4_compute<in_t>(raw0, w0k, s, S, p.bias ? p.bias[c] : 0.f, a0);
    if (p.mode == 0) {
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
            for (int i = 0; i < 8; ++i) a0[o][i] = silu2(a0[o][i]);
    } else if (p.mode == 1) {
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
            for (int i = 0; i < 8; ++i) a0[o][i] = gelu_exact(a0[o][i]);
        float w1k[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) w1k[i] = p.w[(c + p.Cout) * 9 + i];
        float a1[4][8];
        dw_rows4_compute<in_t>(raw1, w1k, s, S, p.bias ? p.bias[c + p.Cout] : 0.f, a1);
#pragma unroll
        for (int o = 0; o < 4; ++o)
#pragma unroll
            for (int i = 0; i < 8; ++i) a0[o][i] *= a1[o][i];
    }
    if (!valid) return;
#pragma unroll
    for (int o = 0; o < 4; ++o)
#pragma unroll
        for (int j = 0; j < 8 / V; ++j) store_vec<in_t>(ob + (int64_t)(h0 + o) * p.W + w0 + j * V, a0[o] + j * V, V, true);
    if (p.out_t != nullptr) {
        // transposed copy: this thread's 4 rows x 8 columns are 8 runs of 4 consecutive h in the (W, H) plane; the four row blocks
        // of a warp that share a strip fill whole 32 B sectors
        in_t* __restrict__ ot = reinterpret_cast<in_t*>(p.out_t) + ((int64_t)b * p.Cout + c) * ((int64_t)p.H * p.W);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            in_t* q = ot + (int64_t)(w0 + i) * p.H + h0;
            if constexpr (sizeof(in_t) == 2) {
                uint2 v;
                v.x = pack2<in_t>(a0[0][i], a0[1][i]);
                v.y = pack2<in_t>(a0[2][i], a0[3][i]);
                *reinterpret_cast<uint2*>(q) = v;
            } else {
                *reinterpret_cast<float4*>(q) = make_float4(a0[0][i], a0[1][i], a0[2][i], a0[3][i]);
            }
        }
    }
}

template <typename in_t>
static int dwconv_rows4_launch(const DwParams& p, cudaStream_t stream) {
    const int S = p.W / 8;
    const long tpp = (long)S * (p.H / 4);
    int lg = 0;
    while ((1L << lg) < tpp) ++lg;
    const long total = tpp * p.B * p.Cout;
    VMB_CUDA(launch_pdl(dwconv3x3_rows4_pre_kernel<in_t>, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream, p, S, lg, total));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int dwconv_launch(const DwParams& p, int dtype, cudaStream_t stream) {
    const int L = p.H * p.W;
    const int S = p.W / 8;
    const long tpp = (long)S * (p.H / 4);
    // row-block kernel where it applies: W and the threads per plane powers of two (plane index by shift, halo shuffles inside one
    // row of strips); every other geometry takes the strip kernel
    if (p.vec_ok && p.W >= 8 && p.W <= 256 && (p.W & (p.W - 1)) == 0 && p.H % 4 == 0 && (tpp & (tpp - 1)) == 0) {
        switch (dtype) {
            case VMB_F32: return dwconv_rows4_launch<float>(p, stream);
            case VMB_BF16: return dwconv_rows4_launch<__nv_bfloat16>(p, stream);
            case VMB_F16: return dwconv_rows4_launch<__half>(p, stream);
            default: set_error("dwconv: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
        }
    }
    const int per_thread = p.vec_ok ? 8 : 1;
    dim3 grid((L / per_thread + 255) / 256 > 0 ? (L / per_thread + 255) / 256 : 1, p.B * p.Cout);
    switch (dtype) {
        case VMB_F32: VMB_CUDA(launch_pdl(dwconv3x3_kernel<float>, grid, dim3(256), 0, stream, p)); break;
        case VMB_BF16: VMB_CUDA(launch_pdl(dwconv3x3_kernel<__nv_bfloat16>, grid, dim3(256), 0, stream, p)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(dwconv3x3_kernel<__half>, grid, dim3(256), 0, stream, p)); break;
        default: set_error("dwconv: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    if (p.out_t != nullptr) {  // geometries the row-block kernel does not take: the transposed copy as its own pass (same values)
        VMB_CHECK(p.o_cs == (int64_t)L && p.o_bs == (int64_t)L * p.Cout, "dwconv: the transposed copy needs a dense primary output");
        return transpose_launch(TransposeParams{p.out, p.out_t, p.B * p.Cout, p.H, p.W}, dtype, stream);
    }
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------ cross scan (4 orders)
// One CTA = one (b, row-set entry, 32x32 pixel tile).  src rows may differ per direction (x_proj outputs) or be
// shared (x).  Output row index = k*rows + row, sequence-contiguous.

template <typename in_t>
__global__ void __launch_bounds__(256) cross_scan_kernel(const CrossScanParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float tile[4][32][33];
    const int tiles_w = (p.W + 31) / 32;
    const int th = blockIdx.x / tiles_w, tw = blockIdx.x % tiles_w;
    const int row = blockIdx.y, b = blockIdx.z;
    const int L = p.H * p.W;
    const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;  // 32 x 8
    const int h0 = th * 32, w0 = tw * 32;
    bool same = p.src[0] == p.src[1] && p.src[0] == p.src[2] && p.src[0] == p.src[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (same && k > 0) break;
        const in_t* __restrict__ s = reinterpret_cast<const in_t*>(p.src[k]) + (int64_t)b * p.src_bs + (int64_t)row * p.src_rs;
        for (int j = ty; j < 32; j += 8) {
            const int h = h0 + j, w = w0 + tx;
            tile[k][j][tx] = (h < p.H && w < p.W) ? to_f32<in_t>(s[h * p.W + w]) : 0.f;
        }
    }
    __syncthreads();
    in_t* __restrict__ o = reinterpret_cast<in_t*>(p.out) + (int64_t)b * p.out_bs;
    const int64_t dir_stride = p.out_ks;
    for (int j = ty; j < 32; j += 8) {
        // row-major orders: l = h*W + w (k=0) and its reversal (k=2); threads along w
        int h = h0 + j, w = w0 + tx;
        if (h < p.H && w < p.W) {
            const int l = h * p.W + w;
            o[0 * dir_stride + (int64_t)row * L + l] = from_f32<in_t>(tile[0][j][tx]);
            o[2 * dir_stride + (int64_t)row * L + (L - 1 - l)] = from_f32<in_t>(tile[same ? 0 : 2][j][tx]);
        }
        // column-major orders: l = w*H + h (k=1) and its reversal (k=3); threads along h
        h = h0 + tx;
        w = w0 + j;
        if (h < p.H && w < p.W) {
            const int l = w * p.H + h;
            o[1 * dir_stride + (int64_t)row * L + l] = from_f32<in_t>(tile[same ? 0 : 1][tx][j]);
            o[3 * dir_stride + (int64_t)row * L + (L - 1 - l)] = from_f32<in_t>(tile[same ? 0 : 3][tx][j]);
        }
    }
}


// Vectorised variant (H % 8 == 0, W % 8 == 0, 16 B aligned rows; 16-bit and fp32 I/O): a CTA owns a 64 x 64 pixel tile of one row,
// loads it with 16 B vectors, and writes the four orders as 16 B vectors -- 8 consecutive w for the row-major orders (reversed
// in-register for k = 2), 8 consecutive h gathered from the fp32 smem tile for the column-major orders.  8x fewer load / store
// instructions than the per-element kernel above (which stays as the fallback for odd geometries).
template <typename in_t>
__device__ __forceinline__ void cross_scan_vec_body(const CrossScanParams& p, const int row, const int b, float* cs_tile) {
    constexpr int V = Vec<in_t>::N;           // 8 (16-bit) or 4 (fp32) elements per 16 B
    constexpr int TS = 64;
    const int tiles_w = (p.W + TS - 1) / TS;
    const int h0 = (blockIdx.x / tiles_w) * TS, w0 = (blockIdx.x % tiles_w) * TS;
    const int L = p.H * p.W;
    const bool same = p.src[0] == p.src[1] && p.src[0] == p.src[2] && p.src[0] == p.src[3];
    const int nsrc = same ? 1 : 4;
    for (int k = 0; k < nsrc; ++k) {
        const in_t* __restrict__ s = reinterpret_cast<const in_t*>(p.src[k]) + (int64_t)b * p.src_bs + (int64_t)row * p.src_rs;
        float* t = cs_tile + k * TS * (TS + 1);
        for (int it = threadIdx.x; it < TS * (TS / V); it += 256) {
            const int hh = it / (TS / V), wv = (it % (TS / V)) * V;
            const int h = h0 + hh, w = w0 + wv;
            float f[V];
            if (h < p.H && w < p.W) load_vec<in_t>(s + (int64_t)h * p.W + w, f, V, true);  // W % V == 0: whole vectors
            else {
#pragma unroll
                for (int i = 0; i < V; ++i) f[i] = 0.f;
            }
#pragma unroll
            for (int i = 0; i < V; ++i) t[hh * (TS + 1) + wv + i] = f[i];
        }
    }
    __syncthreads();
    in_t* __restrict__ o = reinterpret_cast<in_t*>(p.out) + (int64_t)b * p.out_bs + (int64_t)row * L;
    const float* t0 = cs_tile;
    const float* t1 = cs_tile + (same ? 0 : 1) * TS * (TS + 1);
    const float* t2 = cs_tile + (same ? 0 : 2) * TS * (TS + 1);
    const float* t3 = cs_tile + (same ? 0 : 3) * TS * (TS + 1);
    for (int it = threadIdx.x; it < TS * (TS / V); it += 256) {
        {  // row-major orders: V consecutive w of image row h
            const int hh = it / (TS / V), wv = (it % (TS / V)) * V;
            const int h = h0 + hh, w = w0 + wv;
            if (h < p.H && w < p.W) {
                const int l = h * p.W + w;
                float f[V], r[V];
#pragma unroll
                for (int i = 0; i < V; ++i) {
                    f[i] = t0[hh * (TS + 1) + wv + i];
                    r[V - 1 - i] = t2[hh * (TS + 1) + wv + i];
                }
                store_vec<in_t>(o + l, f, V, true);
                store_vec<in_t>(o + 2 * p.out_ks + (L - l - V), r, V, true);  // positions L-1-l ... L-1-(l+V-1), ascending in memory
            }
        }
        {  // column-major orders: V consecutive h of image column w
            const int ww = it / (TS / V), hv = (it % (TS / V)) * V;
            const int w = w0 + ww, h = h0 + hv;
            if (h < p.H && w < p.W) {
                const int l = w * p.H + h;
                float f[V], r[V];
#pragma unroll
                for (int i = 0; i < V; ++i) {
                    f[i] = t1[(hv + i) * (TS + 1) + ww];
                    r[V - 1 - i] = t3[(hv + i) * (TS + 1) + ww];
                }
                store_vec<in_t>(o + p.out_ks + l, f, V, true);
                store_vec<in_t>(o + 3 * p.out_ks + (L - l - V), r, V, true);
            }
        }
    }
}

template <typename in_t>
__global__ void __launch_bounds__(256) cross_scan_vec_kernel(const CrossScanParams p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float cs_tile[];        // [nsrc][64][65]
    cross_scan_vec_body<in_t>(p, blockIdx.y, blockIdx.z, cs_tile);
}

// Up to four cross-scans of one geometry in ONE launch (the training path gathers x, delta and B|C of a block into the four scan
// orders, and scatters du, ddelta, dB, dC back: 3 + 4 launches for a few MB -- launch / latency bound): blockIdx.y
// walks the rows of all segments.
template <typename in_t>
__global__ void __launch_bounds__(256) cross_scan_vec_multi_kernel(const CrossScanMulti m) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float cs_tile[];
    int row = blockIdx.y, s = 0;
    while (s + 1 < m.nseg && row >= m.row_end[s]) ++s;
    if (s > 0) row -= m.row_end[s - 1];
    cross_scan_vec_body<in_t>(m.seg[s], row, blockIdx.z, cs_tile);
}

static bool cross_scan_vec_ok(const CrossScanParams& p, int dtype) {
    const int v = dtype == VMB_F32 ? 4 : 8;
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    return p.H % v == 0 && p.W % v == 0 && al16(p.src[0]) && al16(p.src[1]) && al16(p.src[2]) && al16(p.src[3]) && al16(p.out) &&
           p.src_bs % v == 0 && p.src_rs % v == 0 && p.out_bs % v == 0 && p.out_ks % v == 0;
}

int cross_scan_multi_launch(const CrossScanMulti& m, int dtype, cudaStream_t stream) {
    bool vec = true, all_same = true;
    for (int i = 0; i < m.nseg; ++i) {
        const CrossScanParams& p = m.seg[i];
        vec = vec && cross_scan_vec_ok(p, dtype) && p.B == m.seg[0].B && p.H == m.seg[0].H && p.W == m.seg[0].W;
        all_same = all_same && p.src[0] == p.src[1] && p.src[0] == p.src[2] && p.src[0] == p.src[3];
    }
    if (!vec || m.nseg == 1 || m.row_end[m.nseg - 1] > 65535) {  // one launch per segment: same values
        for (int i = 0; i < m.nseg; ++i) {
            const int rc = cross_scan_launch(m.seg[i], dtype, stream);
            if (rc != VMB_OK) return rc;
        }
        return VMB_OK;
    }
    const CrossScanParams& p0 = m.seg[0];
    const size_t smem = sizeof(float) * (all_same ? 1 : 4) * 64 * 65;
    const dim3 grid(((p0.H + 63) / 64) * ((p0.W + 63) / 64), m.row_end[m.nseg - 1], p0.B);
#define VMB_CSM(T)                                                                                                              \
    {                                                                                                                           \
        if (smem > 48 * 1024)                                                                                                   \
            VMB_CUDA(cudaFuncSetAttribute(cross_scan_vec_multi_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        VMB_CUDA(launch_pdl(cross_scan_vec_multi_kernel<T>, grid, dim3(256), smem, stream, m));                                  \
    }
    switch (dtype) {
        case VMB_F32: VMB_CSM(float) break;
        case VMB_BF16: VMB_CSM(__nv_bfloat16) break;
        case VMB_F16: VMB_CSM(__half) break;
        default: set_error("cross_scan: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
#undef VMB_CSM
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int cross_scan_launch(const CrossScanParams& p, int dtype, cudaStream_t stream) {
    dim3 grid(((p.H + 31) / 32) * ((p.W + 31) / 32), p.rows, p.B);
    VMB_CHECK(p.rows <= 65535 && p.B <= 65535, "cross_scan: too many rows / batch");
    if (cross_scan_vec_ok(p, dtype)) {
        const bool same = p.src[0] == p.src[1] && p.src[0] == p.src[2] && p.src[0] == p.src[3];
        const size_t smem = sizeof(float) * (same ? 1 : 4) * 64 * 65;
        dim3 gv(((p.H + 63) / 64) * ((p.W + 63) / 64), p.rows, p.B);
#define VMB_CSV(T)                                                                                                        \
    {                                                                                                                     \
        if (smem > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(cross_scan_vec_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        VMB_CUDA(launch_pdl(cross_scan_vec_kernel<T>, gv, dim3(256), smem, stream, p));                                    \
    }
        switch (dtype) {
            case VMB_F32: VMB_CSV(float) break;
            case VMB_BF16: VMB_CSV(__nv_bfloat16) break;
            case VMB_F16: VMB_CSV(__half) break;
            default: set_error("cross_scan: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
        }
#undef VMB_CSV
        VMB_CUDA(cudaGetLastError());
        return VMB_OK;
    }
    // per-element kernel: H or W not a multiple of the vector width, or unaligned rows
    switch (dtype) {
        case VMB_F32: VMB_CUDA(launch_pdl(cross_scan_kernel<float>, grid, dim3(256), 0, stream, p)); break;
        case VMB_BF16: VMB_CUDA(launch_pdl(cross_scan_kernel<__nv_bfloat16>, grid, dim3(256), 0, stream, p)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(cross_scan_kernel<__half>, grid, dim3(256), 0, stream, p)); break;
        default: set_error("cross_scan: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------ plane transpose
template <typename in_t>
__global__ void __launch_bounds__(256) transpose_hw_kernel(const TransposeParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float tile[32][33];
    const int tiles_w = (p.W + 31) / 32;
    const int h0 = (blockIdx.x / tiles_w) * 32, w0 = (blockIdx.x % tiles_w) * 32;
    const int64_t plane = (int64_t)blockIdx.y * p.H * p.W;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + plane;
    in_t* __restrict__ o = reinterpret_cast<in_t*>(p.out) + plane;
    const int tx = threadIdx.x % 32, ty = threadIdx.x / 32;
#pragma unroll
    for (int j = ty; j < 32; j += 8)
        tile[j][tx] = (h0 + j < p.H && w0 + tx < p.W) ? to_f32<in_t>(x[(int64_t)(h0 + j) * p.W + w0 + tx]) : 0.f;
    __syncthreads();
#pragma unroll
    for (int j = ty; j < 32; j += 8)
        if (w0 + j < p.W && h0 + tx < p.H) o[(int64_t)(w0 + j) * p.H + h0 + tx] = from_f32<in_t>(tile[tx][j]);
}

int transpose_launch(const TransposeParams& p, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.planes <= 65535, "transpose: too many planes");
    dim3 grid(((p.H + 31) / 32) * ((p.W + 31) / 32), p.planes);
    switch (dtype) {
        case VMB_F32: VMB_CUDA(launch_pdl(transpose_hw_kernel<float>, grid, dim3(256), 0, stream, p)); break;
        case VMB_BF16: VMB_CUDA(launch_pdl(transpose_hw_kernel<__nv_bfloat16>, grid, dim3(256), 0, stream, p)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(transpose_hw_kernel<__half>, grid, dim3(256), 0, stream, p)); break;
        default: set_error("transpose: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------ PixelShuffle(2), NHWC
// One thread moves 16 B of an input pixel's channel vector: 16-bit: channels [8t, 8t+8) = output channels 2t, 2t+1 at the
// four sub-positions k = 2i + j -> one 32-bit word {c=2t, c=2t+1} to each of the four output pixels (2h+i, 2w+j);
// fp32: channels [4t, 4t+4) = output channel t at the four sub-positions.  Consecutive threads walk consecutive
// channels, so both the 16 B loads and the 4 B stores of a warp are contiguous.
template <typename T>
__global__ void __launch_bounds__(256) pixel_shuffle2_nhwc_kernel(const PixelShuffleParams p) {
    pdl_trigger();
    pdl_wait();
    constexpr int V = 16 / sizeof(T);        // input channels per thread
    const int vec_per_px = 4 * p.C / V;
    const int64_t total = (int64_t)p.B * p.H * p.W * vec_per_px;
    const uint4* __restrict__ in = reinterpret_cast<const uint4*>(p.x);
    uint32_t* __restrict__ out = reinterpret_cast<uint32_t*>(p.out);
    const int words_per_px = p.C * (int)sizeof(T) / 4;  // 32-bit words of one output pixel
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(i % vec_per_px);
        const int64_t px = i / vec_per_px;
        const int w = (int)(px % p.W);
        const int64_t bh = px / p.W;
        const int h = (int)(bh % p.H);
        const int64_t b = bh / p.H;
        uint4 v = __ldg(in + i);
        if (p.bias != nullptr) {  // the conv in front ran without its bias: input channel 16/sizeof(T) * t + e gets bias[...] here
            const float* __restrict__ bs = p.bias + t * V;
            if constexpr (sizeof(T) == 2) {
                float f[8];
                unpack8<T>(v, f);
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] += bs[e];
                v.x = pack2<T>(f[0], f[1]); v.y = pack2<T>(f[2], f[3]); v.z = pack2<T>(f[4], f[5]); v.w = pack2<T>(f[6], f[7]);
            } else {
                v.x = __float_as_uint(__uint_as_float(v.x) + bs[0]); v.y = __float_as_uint(__uint_as_float(v.y) + bs[1]);
                v.z = __float_as_uint(__uint_as_float(v.z) + bs[2]); v.w = __float_as_uint(__uint_as_float(v.w) + bs[3]);
            }
        }
        uint32_t wk[4];
        if (sizeof(T) == 2) {
            // halves e0..e7 of the 16 B: element e = (c - 2t) * 4 + k; word_k = {e_k, e_{4+k}}
            wk[0] = __byte_perm(v.x, v.z, 0x5410);
            wk[1] = __byte_perm(v.x, v.z, 0x7632);
            wk[2] = __byte_perm(v.y, v.w, 0x5410);
            wk[3] = __byte_perm(v.y, v.w, 0x7632);
        } else {
            wk[0] = v.x; wk[1] = v.y; wk[2] = v.z; wk[3] = v.w;
        }
        const int64_t row0 = (b * 2 * p.H + 2 * h) * (2 * (int64_t)p.W) + 2 * w;  // output pixel (2h, 2w)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t opx = row0 + (k >> 1) * (2 * (int64_t)p.W) + (k & 1);
            out[opx * words_per_px + t] = wk[k];
        }
    }
}

int pixel_shuffle_launch(const PixelShuffleParams& p, int dtype, cudaStream_t stream) {
    const int v = dtype == VMB_F32 ? 4 : 8;
    VMB_CHECK((4 * p.C) % v == 0, "pixel_shuffle: 4*C must be a multiple of %d", v);
    const int64_t total = (int64_t)p.B * p.H * p.W * (4 * p.C / v);
    int64_t blocks = (total + 255) / 256;
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
    dim3 grid((unsigned)blocks);
    switch (dtype) {
        case VMB_F32: VMB_CUDA(launch_pdl(pixel_shuffle2_nhwc_kernel<float>, grid, dim3(256), 0, stream, p)); break;
        case VMB_BF16: VMB_CUDA(launch_pdl(pixel_shuffle2_nhwc_kernel<__nv_bfloat16>, grid, dim3(256), 0, stream, p)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(pixel_shuffle2_nhwc_kernel<__half>, grid, dim3(256), 0, stream, p)); break;
        default: set_error("pixel_shuffle: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------ merge + out_norm + gate + pool
// CTA = (b, 8x8 pixel tile), all C channels.  Phase 1: sum the four directions in the reference's order,
// (y0 + flip(y2)) + T(y1) + T(flip(y3)), fp32, into smem [C][64].  Phase 2: LayerNorm over C per pixel,
// * z, store y2, accumulate the per-channel sum of y2 (for AdaptiveAvgPool2d).

// Two fully parallel kernels (a single kernel that owns all C channels of a pixel tile has too few CTAs at 64x64):
//  A  merge_sum_kernel    grid (16x16 pixel tiles, C/8 channel chunks, B): directions 0/2 read with threads along w
//                         (32 B row segments), directions 1/3 with threads along h (32 B column segments of the
//                         (W,H)-ordered arrays) and transposed through smem; writes the fp32 merged value
//                         ((y0 + flip y2) + T y1) + T flip y3 and accumulates per-pixel sum / sum of squares over C.
//  B  norm_gate_pool_kernel  grid (C, B): LayerNorm over C with the per-pixel statistics, * z, store, and the per-(b,c)
//                         sum for AdaptiveAvgPool2d by a block reduction (no atomics, no memset of `pooled`).
constexpr int MG_CH = 8;

template <typename in_t>
__global__ void __launch_bounds__(256) merge_sum_kernel(const MergeParams p, float* __restrict__ msum, float* __restrict__ stats) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sT[2 * MG_CH][16][17];
    const int C = p.C, L = p.H * p.W;
    const int tiles_w = (p.W + 15) / 16;
    const int h0 = (blockIdx.x / tiles_w) * 16, w0 = (blockIdx.x % tiles_w) * 16;
    const int c0 = blockIdx.y * MG_CH, b = blockIdx.z;
    const int th = threadIdx.x / 16, tw = threadIdx.x % 16;
    const int64_t CL = (int64_t)C * L;
    const in_t* __restrict__ ys = reinterpret_cast<const in_t*>(p.ys) + (int64_t)b * 4 * CL;
    const int ph = h0 + th, pw = w0 + tw;
    const bool ok = ph < p.H && pw < p.W;
    const int l_row = ph * p.W + pw;
    const int i2 = p.in_place_order ? l_row : L - 1 - l_row;
    const int qh = h0 + tw, qw = w0 + th;  // transposed loads: consecutive threads walk h
    const bool okq = qh < p.H && qw < p.W;
    const int l_col = qw * p.H + qh;
    const int i3 = p.in_place_order ? l_col : L - 1 - l_col;
    float nat[MG_CH];
#pragma unroll
    for (int j = 0; j < MG_CH; ++j) {
        const int c = c0 + j;
        nat[j] = 0.f;
        if (c < C) {
            const in_t* __restrict__ yc = ys + (int64_t)c * L;
            if (ok) nat[j] = to_f32<in_t>(yc[l_row]) + to_f32<in_t>(yc[2 * CL + i2]);
            if (okq) {
                sT[j][th][tw] = to_f32<in_t>(yc[CL + l_col]);
                sT[MG_CH + j][th][tw] = to_f32<in_t>(yc[3 * CL + i3]);
            }
        }
    }
    __syncthreads();
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < MG_CH; ++j) {
        const int c = c0 + j;
        if (c < C && ok) {
            const float v = (nat[j] + sT[j][tw][th]) + sT[MG_CH + j][tw][th];
            msum[((int64_t)b * C + c) * L + l_row] = v;
            s1 += v;
            s2 = fmaf(v, v, s2);
        }
    }
    if (ok) {
        atomicAdd(stats + ((int64_t)b * L + l_row) * 2, s1);
        atomicAdd(stats + ((int64_t)b * L + l_row) * 2 + 1, s2);
    }
}

template <typename in_t>
__global__ void __launch_bounds__(256) norm_gate_pool_kernel(const MergeParams p, const float* __restrict__ msum,
                                                             const float* __restrict__ stats) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sRed[8];
    const int C = p.C, L = p.H * p.W;
    const int c = blockIdx.x, b = blockIdx.y;
    const float* __restrict__ m = msum + ((int64_t)b * C + c) * L;
    const float2* __restrict__ st = reinterpret_cast<const float2*>(stats) + (int64_t)b * L;
    const in_t* __restrict__ z = reinterpret_cast<const in_t*>(p.z) + (int64_t)b * p.z_bs + (int64_t)c * p.z_cs;
    in_t* __restrict__ o = reinterpret_cast<in_t*>(p.y2) + ((int64_t)b * C + c) * L;
    const float lw = p.ln_w[c], lb = p.ln_b[c], invC = 1.f / C;
    float acc = 0.f;
    for (int l = threadIdx.x; l < L; l += 256) {
        const float2 s = st[l];
        const float mu = s.x * invC;
        // sum of squares in fp32: |mu| is O(sigma) for the merged scan outputs, the cancellation costs < 1e-6 relative
        const float rstd = rsqrtf(fmaxf(s.y * invC - mu * mu, 0.f) + 1e-5f);
        const float nrm = (m[l] - mu) * rstd * lw + lb;
        // the reference rounds y1 to the activation dtype before the gate (.to(x.dtype), :434)
        const float n_r = to_f32<in_t>(from_f32<in_t>(nrm));
        const float zv = to_f32<in_t>(z[l]);
        const in_t y = from_f32<in_t>(n_r * (p.z_preact ? silu2(zv) : zv));
        o[l] = y;
        acc += to_f32<in_t>(y);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sRed[i];
        p.pooled[(int64_t)b * C + c] = t;
    }
}


// ---- single-kernel variant (round 2): 16-bit I/O, H % 16 == 0, W % 16 == 0, C <= 96 ------------------------------------------------
// The judgement above ("too few CTAs") was about a CTA that also walks its channels serially with exposed load latency.  Here a CTA
// of 512 threads owns a 16 x 16 pixel tile and ALL channels, and the four direction tiles of 4 channels at a time arrive through a
// 4-deep cp.async ring in their MEMORY order (32 B row segments of the (H,W)-ordered directions 0 / 2, 32 B column segments of the
// (W,H)-ordered directions 1 / 3, mirrored segments for the reversed scan orders), so that phase 1 (thread = pixel: the reference's
// ((y0 + flip y2) + T y1) + T flip y3, fp32, into the smem tile [C][256], per-pixel sum / sum of squares in registers -- no
// atomics, no memset) never waits for a load.  Phase 2 (thread = 8-pixel vector x channel slice): LayerNorm with the per-pixel
// statistics, gate, 16 B stores, per-channel tile sums; the last CTA of an image (counter in the workspace) adds the tile sums in a
// fixed order into `pooled` -- deterministic, unlike a float atomicAdd.
constexpr int MF_CG = 4, MF_ST = 4, MF_PITCH = 24;
constexpr int MF_MAXPW = 6;                                           // channels per warp in phase 2 (16 warps: C <= 96)                    // channels per stage, ring depth, tile row pitch (elements)
constexpr int MF_STAGE = MF_CG * 4 * 16 * MF_PITCH;                   // elements of one ring stage
__host__ __device__ constexpr size_t merge_fused_smem(int C) {
    return sizeof(float) * ((size_t)C * 256 + 512) + 2 * (size_t)MF_ST * MF_STAGE + 16;
}

template <typename in_t>
__global__ void __launch_bounds__(512) merge_fused_kernel(const MergeParams p, float* __restrict__ msum, float* __restrict__ stats,
                                                          float* __restrict__ parts, unsigned* __restrict__ counters, const int save_ws) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char mf_raw[];
    const int C = p.C, H = p.H, W = p.W, L = H * W;
    float* sSum = reinterpret_cast<float*>(mf_raw);                    // [C][256]
    float* sMu = sSum + (size_t)C * 256;                               // [256]
    float* sRs = sMu + 256;                                            // [256]
    in_t* sRing = reinterpret_cast<in_t*>(sRs + 256);                  // [MF_ST][4 ch][4 dir][16][MF_PITCH]
    __shared__ int s_last;
    const int tid = threadIdx.x;
    const int tiles_w = W / 16, ntiles = (H / 16) * tiles_w;
    const int tile = blockIdx.x, b = blockIdx.y;
    const int h0 = (tile / tiles_w) * 16, w0 = (tile % tiles_w) * 16;
    const int64_t CL = (int64_t)C * L;
    const in_t* __restrict__ ys = reinterpret_cast<const in_t*>(p.ys) + (int64_t)b * 4 * CL;
    const int ngroups = (C + MF_CG - 1) / MF_CG;
    const bool inplace = p.in_place_order != 0;

    // 512 16-byte chunks per stage, one per thread: chunk -> (direction k, channel cl of the group, tile row r, half row); everything
    // but the channel group is loop-invariant, so the source pointer advances by 4 channels per stage and nothing else is recomputed
    const in_t* csrc;
    uint32_t cdst;
    int ccl;
    {
        const int k = tid >> 7, cl = (tid >> 5) & 3, r = (tid >> 1) & 15, half = tid & 1;
        int64_t idx;
        if ((k & 1) == 0) idx = (int64_t)(h0 + r) * W + w0;        // directions 0 / 2: row r of the tile, 16 consecutive w
        else idx = (int64_t)(w0 + r) * H + h0;                     // directions 1 / 3: column r of the tile, 16 consecutive h
        if (k >= 2 && !inplace) idx = (int64_t)L - 16 - idx;        // reversed scan order: the mirrored 16-element segment
        csrc = ys + (int64_t)k * CL + (int64_t)cl * L + idx + 8 * half;
        cdst = static_cast<uint32_t>(__cvta_generic_to_shared(sRing + ((cl * 4 + k) * 16 + r) * MF_PITCH + 8 * half));
        ccl = cl;
    }
    const int64_t gstep = (int64_t)MF_CG * L;
    auto issue = [&](int g) {
        const uint32_t soff = (uint32_t)((g % MF_ST) * MF_STAGE * (int)sizeof(in_t));
        const bool ok = g * MF_CG + ccl < C;
        const in_t* src = ok ? csrc + (int64_t)g * gstep : ys;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(cdst + soff), "l"(src), "r"(ok ? 16 : 0) : "memory");
    };
#pragma unroll
    for (int g = 0; g < MF_ST - 1; ++g) {
        if (g < ngroups) issue(g);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    // the gate operand of phase 2 (this lane's 8-pixel vector of every channel of its warp's slice) is fetched now: it lands while
    // phase 1 runs
    const int lane = tid & 31, warp = tid >> 5;
    const int vh = lane >> 1, vw = (lane & 1) * 8;
    const int l0 = (h0 + vh) * W + w0 + vw;
    uint4 zr[MF_MAXPW];
    {
        const in_t* __restrict__ zb = reinterpret_cast<const in_t*>(p.z) + (int64_t)b * p.z_bs + l0;
#pragma unroll
        for (int j = 0; j < MF_MAXPW; ++j) {
            const int c = warp + 16 * j;
            zr[j] = c < C ? ldg128(zb + (int64_t)c * p.z_cs) : make_uint4(0u, 0u, 0u, 0u);
        }
    }
    // phase 1: thread = (channel half of the group, pixel (th, tw))
    const int hsel = tid >> 8, pix = tid & 255;
    const int th = pix >> 4, tw = pix & 15;
    const int o2 = inplace ? tw : 15 - tw;   // position of this pixel inside the (possibly mirrored) row segment of direction 2
    const int o3 = inplace ? th : 15 - th;   // ... inside the column segment of direction 3
    const int r0 = (0 * 16 + th) * MF_PITCH + tw, r1 = (1 * 16 + tw) * MF_PITCH + th;
    const int r2 = (2 * 16 + th) * MF_PITCH + o2, r3 = (3 * 16 + tw) * MF_PITCH + o3;
    float s1 = 0.f, s2 = 0.f;
    float* sumcol = sSum + pix;
#pragma unroll 1
    for (int g = 0; g < ngroups; ++g) {
        asm volatile("cp.async.wait_group %0;" ::"n"(MF_ST - 2) : "memory");
        __syncthreads();  // stage g landed for every thread; stage g-1 is free again
        if (g + MF_ST - 1 < ngroups) issue(g + MF_ST - 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        const in_t* st = sRing + (size_t)(g % MF_ST) * MF_STAGE;
#pragma unroll
        for (int j = 0; j < MF_CG / 2; ++j) {
            const int cl = 2 * hsel + j;
            const int c = g * MF_CG + cl;
            if (c < C) {
                const in_t* t = st + cl * 4 * 16 * MF_PITCH;
                const float y0 = to_f32<in_t>(t[r0]);
                const float y1 = to_f32<in_t>(t[r1]);
                const float y2 = to_f32<in_t>(t[r2]);
                const float y3 = to_f32<in_t>(t[r3]);
                const float v = ((y0 + y2) + y1) + y3;
                sumcol[c * 256] = v;
                s1 += v;
                s2 = fmaf(v, v, s2);
            }
        }
    }
    // per-pixel statistics: the two channel halves meet in smem (sMu / sRs double as the exchange buffer)
    if (hsel == 1) {
        sMu[pix] = s1;
        sRs[pix] = s2;
    }
    __syncthreads();
    if (hsel == 0) {
        s1 += sMu[pix];
        s2 += sRs[pix];
        const float invC = 1.f / C;
        const float mu = s1 * invC;
        sMu[pix] = mu;
        sRs[pix] = rsqrtf(fmaxf(s2 * invC - mu * mu, 0.f) + 1e-5f);
        if (save_ws) {
            const int l = (h0 + th) * W + w0 + tw;
            *reinterpret_cast<float2*>(stats + ((int64_t)b * L + l) * 2) = make_float2(s1, s2);
        }
    }
    __syncthreads();
    // phase 2: lane = 8-pixel vector of the tile (row lane/2, half lane%2), warp = channel slice (z vectors prefetched above)
    float mu8[8], rs8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        mu8[i] = sMu[vh * 16 + vw + i];
        rs8[i] = sRs[vh * 16 + vw + i];
    }
    in_t* __restrict__ ob = reinterpret_cast<in_t*>(p.y2) + (int64_t)b * CL;
    const bool zact = p.z_preact != 0;
#pragma unroll
    for (int j = 0; j < MF_MAXPW; ++j) {
        const int c = warp + 16 * j;
        if (c < C) {
            float zv[8], m8[8], o8[8];
            unpack8<in_t>(zr[j], zv);
            *reinterpret_cast<float4*>(m8) = *reinterpret_cast<const float4*>(sSum + c * 256 + vh * 16 + vw);
            *reinterpret_cast<float4*>(m8 + 4) = *reinterpret_cast<const float4*>(sSum + c * 256 + vh * 16 + vw + 4);
            const float lw = p.ln_w[c], lb = p.ln_b[c];
            float acc = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float nrm = (m8[i] - mu8[i]) * rs8[i] * lw + lb;
                const float n_r = to_f32<in_t>(from_f32<in_t>(nrm));  // the reference rounds y1 to the activation dtype before the gate
                const in_t y = from_f32<in_t>(n_r * (zact ? silu2(zv[i]) : zv[i]));
                o8[i] = to_f32<in_t>(y);
                acc += o8[i];
            }
            store_vec<in_t>(ob + (int64_t)c * L + l0, o8, 8, true);
            if (save_ws) {
                float* mrow = msum + ((int64_t)b * C + c) * L + l0;
                *reinterpret_cast<float4*>(mrow) = *reinterpret_cast<const float4*>(m8);
                *reinterpret_cast<float4*>(mrow + 4) = *reinterpret_cast<const float4*>(m8 + 4);
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
            if (lane == 0) parts[((int64_t)b * ntiles + tile) * C + c] = acc;
        }
    }
    // the last tile of the image adds the tile sums, in tile order
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(counters + b, 1u) == (unsigned)(ntiles - 1);
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (int c = tid; c < C; c += 512) {
            float t = 0.f;
            for (int i = 0; i < ntiles; ++i) t += __ldcg(parts + ((int64_t)b * ntiles + i) * C + c);
            p.pooled[(int64_t)b * C + c] = t;
        }
        if (tid == 0) counters[b] = 0;  // ready for the next launch on this workspace
    }
}

// the workspace regions of the fused kernel sit behind the fp32 merged values and the statistics
static bool merge_fused_applicable(const MergeParams& p, int dtype) {
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    const bool legal = (dtype == VMB_BF16 || dtype == VMB_F16) && p.H % 16 == 0 && p.W % 16 == 0 && p.C <= 16 * MF_MAXPW &&
                       merge_fused_smem(p.C) <= 200 * 1024 && al16(p.ys) && al16(p.z) && al16(p.y2) && p.z_bs % 8 == 0 && p.z_cs % 8 == 0;
    // from 128 x 128 pixels per image up: the normalisation kernel of the two-kernel path walks all pixels of a channel in one CTA,
    // which dominates at large images; a CTA of the single kernel walks all channel groups of its tile at any size, which dominates
    // at small ones.  On the H100 the crossover lies between 32 x 32 and 64 x 64 (DESIGN §1.4: timings, and why it is kept here)
    return legal && (long)p.H * p.W >= 16384;
}

int merge_launch(const MergeParams& p, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.ws != nullptr, "merge: workspace missing");
    const int L = p.H * p.W;
    float* msum = reinterpret_cast<float*>(p.ws);
    float* stats = msum + (size_t)p.B * p.C * L;
    if (merge_fused_applicable(p, dtype)) {
        const int ntiles = (p.H / 16) * (p.W / 16);
        float* parts = stats + 2 * (size_t)p.B * L;
        unsigned* counters = reinterpret_cast<unsigned*>(parts + (size_t)p.B * ntiles * p.C);
        const size_t smem = merge_fused_smem(p.C);
        VMB_CHECK(p.B <= 65535, "merge: batch > 65535");
        VMB_CUDA(cudaMemsetAsync(counters, 0, sizeof(unsigned) * p.B, stream));  // (the kernel also leaves them at zero)
        dim3 grid(ntiles, p.B);
        if (dtype == VMB_BF16) {
            auto k = merge_fused_kernel<__nv_bfloat16>;
            VMB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k<<<grid, 512, smem, stream>>>(p, msum, stats, parts, counters, p.save_ws);
        } else {
            auto k = merge_fused_kernel<__half>;
            VMB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            k<<<grid, 512, smem, stream>>>(p, msum, stats, parts, counters, p.save_ws);
        }
        VMB_CUDA(cudaGetLastError());
        return VMB_OK;
    }
    VMB_CUDA(cudaMemsetAsync(stats, 0, sizeof(float) * 2 * (size_t)p.B * L, stream));
    dim3 gridA(((p.H + 15) / 16) * ((p.W + 15) / 16), (p.C + MG_CH - 1) / MG_CH, p.B);
    dim3 gridB(p.C, p.B);
    VMB_CHECK(gridA.y <= 65535 && p.B <= 65535 && p.C <= 65535, "merge: grid too large");
#define VMB_MERGE(T)                                                       \
    {                                                                      \
        merge_sum_kernel<T><<<gridA, 256, 0, stream>>>(p, msum, stats); /* follows a memset node: plain launch */ \
        VMB_CUDA(launch_pdl(norm_gate_pool_kernel<T>, gridB, dim3(256), 0, stream, p, (const float*)msum, (const float*)stats)); \
    }
    switch (dtype) {
        case VMB_F32: VMB_MERGE(float) break;
        case VMB_BF16: VMB_MERGE(__nv_bfloat16) break;
        case VMB_F16: VMB_MERGE(__half) break;
        default: set_error("merge: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
#undef VMB_MERGE
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// the four-way fp32 sum alone (merge_sum_kernel into `out`, its per-pixel statistics into the workspace): cross_selective_scan's merge
// (forward) and its adjoint of the direction-aware backward (du of every direction + the x_proj data gradients, in the groups' orders)
int merge_sum_launch(const MergeParams& p, float* out, int dtype, cudaStream_t stream) {
    VMB_CHECK(p.ws != nullptr && out != nullptr, "merge_sum: workspace / output missing");
    const int L = p.H * p.W;
    float* stats = reinterpret_cast<float*>(p.ws) + (size_t)p.B * p.C * L;
    VMB_CUDA(cudaMemsetAsync(stats, 0, sizeof(float) * 2 * (size_t)p.B * L, stream));
    dim3 gridA(((p.H + 15) / 16) * ((p.W + 15) / 16), (p.C + MG_CH - 1) / MG_CH, p.B);
    VMB_CHECK(gridA.y <= 65535 && p.B <= 65535, "merge_sum: grid too large");
    switch (dtype) {
        case VMB_F32: merge_sum_kernel<float><<<gridA, 256, 0, stream>>>(p, out, stats); break;
        case VMB_BF16: merge_sum_kernel<__nv_bfloat16><<<gridA, 256, 0, stream>>>(p, out, stats); break;
        case VMB_F16: merge_sum_kernel<__half><<<gridA, 256, 0, stream>>>(p, out, stats); break;
        default: set_error("merge_sum: unsupported dtype %d", dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// ------------------------------------------------------------------------------------------ channel branch
// One CTA (256 threads) per image.  Sequence = the C pooled channel means, dc rows, 2 directions, N states.

__global__ void __launch_bounds__(256) channel_branch_kernel(const ChannelParams p) {
    pdl_trigger();
    extern __shared__ float sm[];
    const int C = p.C, dc = p.dc, Rc = p.Rc, N = p.N, RN = Rc + 2 * N;
    const int CP = C | 1;                // odd row pitch of sDbl: the 16 state lanes of the scan read 16 different rows
    float* sSeq = sm;                    // [dc][C]     xc
    float* sDbl = sSeq + dc * C;         // [2][RN][C]  xc_dbl per direction (direction order)
    float* sDt = sDbl + 2 * RN * CP;     // [2][dc][C]  softplus'ed dt
    float* sY = sDt + 2 * dc * C;        // [2][dc][C]  scan outputs (direction order)
    float* sOut = sY + 2 * dc * C;       // [C]
    float* sRed = sOut + C;              // [64]
    // parameters staged once (one batch of independent loads instead of a dependent global load per phase)
    float* sXp = sRed + 64;              // [2][RN][dc]
    float* sDw = sXp + 2 * RN * dc;      // [2][dc][Rc]
    float* sDb = sDw + 2 * dc * Rc;      // [2][dc]
    float* sCio = sDb + 2 * dc;          // cin_w[dc] cin_b[dc] cout_w[dc] cout_b[1]
    const int b = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < 2 * RN * dc; i += 256) sXp[i] = p.xc_proj[i];
    for (int i = tid; i < 2 * dc * Rc; i += 256) sDw[i] = p.dtc_w[i];
    if (tid < 2 * dc) sDb[tid] = p.dtc_b[tid];
    if (tid < dc) {
        sCio[tid] = p.cin_w ? p.cin_w[tid] : 1.f;
        sCio[dc + tid] = p.cin_w ? p.cin_b[tid] : 0.f;
        sCio[2 * dc + tid] = p.cout_w ? p.cout_w[tid] : 1.f;
    }
    if (tid == 0) sCio[3 * dc] = p.cout_w ? p.cout_b[0] : 0.f;
    pdl_wait();  // the parameter staging above overlaps the tail of the merge kernels; `pooled` is read from here on
    __syncthreads();
    // xc = conv_cin(pool)  (per-channel affine of the pooled mean)
    for (int i = tid; i < dc * C; i += 256) {
        const int j = i / C, l = i % C;
        const float m = p.pooled[(int64_t)b * C + l] * p.inv_count;
        sSeq[i] = fmaf(m, sCio[j], sCio[dc + j]);
    }
    __syncthreads();
    // xc_dbl[k][c][l] = sum_j W[k][c][j] * xs[k][j][l],  xs[1] = flipped sequence
    for (int i = tid; i < 2 * RN * C; i += 256) {
        const int k = i / (RN * C), c = (i / C) % RN, l = i % C;
        const int ls = k ? C - 1 - l : l;
        float a = 0.f;
        for (int j = 0; j < dc; ++j) a = fmaf(sXp[(k * RN + c) * dc + j], sSeq[j * C + ls], a);
        sDbl[(k * RN + c) * CP + l] = a;
    }
    __syncthreads();
    // dt[k][j][l] = softplus(sum_r Wdt[k][j][r] * dbl[k][r][l] + bias)
    for (int i = tid; i < 2 * dc * C; i += 256) {
        const int k = i / (dc * C), j = (i / C) % dc, l = i % C;
        float a = sDb[k * dc + j];
        for (int r = 0; r < Rc; ++r) a = fmaf(sDw[(k * dc + j) * Rc + r], sDbl[(k * RN + r) * CP + l], a);
        sDt[i] = softplus_f(a);
    }
    __syncthreads();
    // sequential scan: one thread per (direction k, row j, state n); N <= 16 lanes reduce y with shuffles
    const int rows = 2 * dc;
    const int unit = tid / 16, n = tid % 16;  // 16 units of 16 lanes
    for (int row = unit; row < rows; row += 16) {
        const int k = row / dc, j = row % dc;
        const bool act = n < N;
        const float A = act ? -__expf(p.Ac_logs[row * N + n]) * kLog2e : 0.f;
        const float Dv = p.Dsc[row];
        const float* __restrict__ dtr = sDt + (k * dc + j) * C;
        const float* __restrict__ Br = sDbl + (k * RN + Rc + (act ? n : 0)) * CP;
        const float* __restrict__ Cr = sDbl + (k * RN + Rc + N + (act ? n : 0)) * CP;
        float* __restrict__ yr = sY + (k * dc + j) * C;
        float h = 0.f;
        int l = 0;
        // 4 positions per iteration: the recurrence is sequential, the four 16-lane reductions run interleaved
        for (; l + 4 <= C; l += 4) {
            float dt[4], u[4], a[4], y[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                dt[i] = dtr[l + i];
                u[i] = sSeq[j * C + (k ? C - 1 - (l + i) : l + i)];
                a[i] = ex2(dt[i] * A);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                h = fmaf(a[i], h, act ? dt[i] * u[i] * Br[l + i] : 0.f);
                y[i] = act ? h * Cr[l + i] : 0.f;
            }
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) {
#pragma unroll
                for (int i = 0; i < 4; ++i) y[i] += __shfl_xor_sync(0xffffffffu, y[i], o, 16);
            }
            if (n == 0) {
#pragma unroll
                for (int i = 0; i < 4; ++i) yr[l + i] = fmaf(Dv, u[i], y[i]);
            }
        }
        for (; l < C; ++l) {
            const float dt = dtr[l];
            const float u = sSeq[j * C + (k ? C - 1 - l : l)];
            h = fmaf(ex2(dt * A), h, act ? dt * u * Br[l] : 0.f);
            float y = act ? h * Cr[l] : 0.f;
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) y += __shfl_xor_sync(0xffffffffu, y, o, 16);
            if (n == 0) yr[l] = fmaf(Dv, u, y);
        }
    }
    __syncthreads();
    // merge directions, conv_cout, channel_norm over the C positions
    float part = 0.f;
    for (int l = tid; l < C; l += 256) {
        float acc = sCio[3 * dc];
        for (int j = 0; j < dc; ++j) {
            const float y = sY[(0 * dc + j) * C + l] + sY[(1 * dc + j) * C + (C - 1 - l)];
            acc = fmaf(y, sCio[2 * dc + j], acc);
        }
        sOut[l] = acc;
        part += acc;
    }
    // block mean / variance (two-pass)
    auto block_sum = [&](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        __syncthreads();
        if ((tid & 31) == 0) sRed[tid >> 5] = v;
        __syncthreads();
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += sRed[i];
        return t;
    };
    const float mu = block_sum(part) / C;
    float vp = 0.f;
    for (int l = tid; l < C; l += 256) {
        const float d = sOut[l] - mu;
        vp += d * d;
    }
    const float rstd = rsqrtf(block_sum(vp) / C + 1e-5f);
    for (int l = tid; l < C; l += 256) p.c_out[(int64_t)b * C + l] = (sOut[l] - mu) * rstd * p.cn_w[l] + p.cn_b[l];
}

// Second version (default): 512 threads, row-per-warp loops without integer division, and a scan whose serial loop
// carries only the h recurrence -- exp / dt*u*B are independent of h and are hoisted eight positions ahead, the
// per-position sum over the 16 states (a 4-stage shuffle chain per position in v1) becomes a store of h*C into
// shared memory and one parallel reduction afterwards.
constexpr int CH2_THREADS = 512;

__global__ void __launch_bounds__(CH2_THREADS) channel_branch_v2_kernel(const ChannelParams p) {
    pdl_trigger();
    extern __shared__ float sm[];
    const int C = p.C, dc = p.dc, Rc = p.Rc, N = p.N, RN = Rc + 2 * N;
    const int CP = C | 1;                 // odd row pitch: the 16 state lanes touch 16 different rows without bank conflicts
    const int rows = 2 * dc;              // (direction, row) scan rows
    float* sSeq = sm;                     // [dc][C]     xc
    float* sDbl = sSeq + dc * C;          // [2][RN][CP] xc_dbl per direction (direction order)
    float* sDt = sDbl + 2 * RN * CP;      // [2][dc][C]  softplus'ed dt
    float* sY = sDt + rows * C;           // [2][dc][C]  scan outputs (direction order)
    float* sOut = sY + rows * C;          // [C]
    float* sRed = sOut + C;               // [64]
    float* sXp = sRed + 64;               // [2][RN][dc]
    float* sDw = sXp + 2 * RN * dc;       // [2][dc][Rc]
    float* sDb = sDw + 2 * dc * Rc;       // [2][dc]
    float* sCio = sDb + 2 * dc;           // cin_w[dc] cin_b[dc] cout_w[dc] cout_b[1]
    float* sHC = sCio + 3 * dc + 1;       // [rows][16][CP]  h * C per state
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    constexpr int NW = CH2_THREADS / 32;
    for (int i = tid; i < 2 * RN * dc; i += CH2_THREADS) sXp[i] = p.xc_proj[i];
    for (int i = tid; i < 2 * dc * Rc; i += CH2_THREADS) sDw[i] = p.dtc_w[i];
    if (tid < 2 * dc) sDb[tid] = p.dtc_b[tid];
    if (tid < dc) {
        sCio[tid] = p.cin_w ? p.cin_w[tid] : 1.f;
        sCio[dc + tid] = p.cin_w ? p.cin_b[tid] : 0.f;
        sCio[2 * dc + tid] = p.cout_w ? p.cout_w[tid] : 1.f;
    }
    if (tid == 0) sCio[3 * dc] = p.cout_w ? p.cout_b[0] : 0.f;
    // scan parameters of this thread's (row, state): weights, loaded ahead of the wait
    const int srow = tid >> 4, n = tid & 15;
    const bool sact = srow < rows && n < N;
    const float A2 = sact ? -__expf(p.Ac_logs[srow * N + n]) * kLog2e : 0.f;
    pdl_wait();  // the parameter staging above overlaps the tail of the merge kernels; `pooled` is read from here on
    __syncthreads();
    // xc = conv_cin(pool)  (per-channel affine of the pooled mean): warp j-strided rows, lanes over the sequence
    for (int j = warp; j < dc; j += NW)
        for (int l = lane; l < C; l += 32) sSeq[j * C + l] = fmaf(p.pooled[(int64_t)b * C + l] * p.inv_count, sCio[j], sCio[dc + j]);
    __syncthreads();
    // xc_dbl[k][c][l] = sum_j W[k][c][j] * xs[k][j][l],  xs[1] = flipped sequence
    for (int kc = warp; kc < 2 * RN; kc += NW) {
        const int k = kc >= RN;
        const float* wrow = sXp + kc * dc;
        for (int l = lane; l < C; l += 32) {
            const int ls = k ? C - 1 - l : l;
            float a = 0.f;
            for (int j = 0; j < dc; ++j) a = fmaf(wrow[j], sSeq[j * C + ls], a);
            sDbl[kc * CP + l] = a;
        }
    }
    __syncthreads();
    // dt[k][j][l] = softplus(sum_r Wdt[k][j][r] * dbl[k][r][l] + bias)
    for (int kj = warp; kj < rows; kj += NW) {
        const int k = kj / dc;
        for (int l = lane; l < C; l += 32) {
            float a = sDb[kj];
            for (int r = 0; r < Rc; ++r) a = fmaf(sDw[kj * Rc + r], sDbl[(k * RN + r) * CP + l], a);
            sDt[kj * C + l] = softplus_f(a);
        }
    }
    __syncthreads();
    // sequential scan: thread = (row, state n)
    if (srow < rows) {
        const int k = srow / dc, j = srow - k * dc;
        const float* __restrict__ dtr = sDt + srow * C;
        const float* __restrict__ ur = sSeq + j * C;
        const float* __restrict__ Br = sDbl + (k * RN + Rc + (sact ? n : 0)) * CP;
        const float* __restrict__ Cr = sDbl + (k * RN + Rc + N + (sact ? n : 0)) * CP;
        float* __restrict__ hc = sHC + (srow * 16 + n) * CP;
        float h = 0.f;
        int l = 0;
        for (; l + 8 <= C; l += 8) {
            float a[8], bu[8], cv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float dt = dtr[l + i];
                const float u = ur[k ? C - 1 - (l + i) : l + i];
                a[i] = ex2(dt * A2);
                bu[i] = sact ? dt * u * Br[l + i] : 0.f;
                cv[i] = sact ? Cr[l + i] : 0.f;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                h = fmaf(a[i], h, bu[i]);
                hc[l + i] = h * cv[i];
            }
        }
        for (; l < C; ++l) {
            const float dt = dtr[l];
            const float u = ur[k ? C - 1 - l : l];
            h = fmaf(ex2(dt * A2), h, sact ? dt * u * Br[l] : 0.f);
            hc[l] = sact ? h * Cr[l] : 0.f;
        }
    }
    __syncthreads();
    // y[row][l] = D u + sum over the 16 state slots
    for (int row = warp; row < rows; row += NW) {
        const int k = row / dc, j = row - k * dc;
        const float Dv = p.Dsc[row];
        for (int l = lane; l < C; l += 32) {
            float y = 0.f;
#pragma unroll
            for (int s = 0; s < 16; ++s) y += sHC[(row * 16 + s) * CP + l];
            sY[row * C + l] = fmaf(Dv, sSeq[j * C + (k ? C - 1 - l : l)], y);
        }
    }
    __syncthreads();
    // merge directions, conv_cout, channel_norm over the C positions
    float part = 0.f;
    for (int l = tid; l < C; l += CH2_THREADS) {
        float acc = sCio[3 * dc];
        for (int j = 0; j < dc; ++j) {
            const float y = sY[(0 * dc + j) * C + l] + sY[(1 * dc + j) * C + (C - 1 - l)];
            acc = fmaf(y, sCio[2 * dc + j], acc);
        }
        sOut[l] = acc;
        part += acc;
    }
    auto block_sum = [&](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        __syncthreads();
        if (lane == 0) sRed[warp] = v;
        __syncthreads();
        float t = 0.f;
        for (int i = 0; i < NW; ++i) t += sRed[i];
        return t;
    };
    const float mu = block_sum(part) / C;
    float vp = 0.f;
    for (int l = tid; l < C; l += CH2_THREADS) {
        const float d = sOut[l] - mu;
        vp += d * d;
    }
    const float rstd = rsqrtf(block_sum(vp) / C + 1e-5f);
    for (int l = tid; l < C; l += CH2_THREADS) p.c_out[(int64_t)b * C + l] = (sOut[l] - mu) * rstd * p.cn_w[l] + p.cn_b[l];
}

int channel_launch(const ChannelParams& p, cudaStream_t stream) {
    VMB_CHECK(p.N <= 16, "channel branch: dstate <= 16 supported (got %d)", p.N);
    const int RN = p.Rc + 2 * p.N;
    const size_t base = sizeof(float) * ((size_t)p.dc * p.C + 2 * RN * (p.C | 1) + 4 * p.dc * p.C + p.C + 64 + 2 * RN * p.dc +
                                         2 * p.dc * p.Rc + 2 * p.dc + 3 * p.dc + 1);
    const size_t smem2 = base + sizeof(float) * (size_t)2 * p.dc * 16 * (p.C | 1);
    if (2 * p.dc * 16 <= CH2_THREADS && smem2 <= 227 * 1024) {
        if (smem2 > 48 * 1024)
            VMB_CUDA(cudaFuncSetAttribute(channel_branch_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        VMB_CUDA(launch_pdl(channel_branch_v2_kernel, dim3(p.B), dim3(CH2_THREADS), smem2, stream, p));
        VMB_CUDA(cudaGetLastError());
        return VMB_OK;
    }
    const size_t smem = base;
    VMB_CHECK(smem <= 227 * 1024, "channel branch: C=%d too large", p.C);
    if (smem > 48 * 1024)
        VMB_CUDA(cudaFuncSetAttribute(channel_branch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    VMB_CUDA(launch_pdl(channel_branch_kernel, dim3(p.B), dim3(256), smem, stream, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb
