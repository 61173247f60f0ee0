// Per-pixel linear layer on NCHW activations ("1x1 conv") with fused prologue / epilogue:
//     out[b, m, p] = epi( sum_k W[m,k] * pro(x)[b, k, p] )
// replaces, inside one OSS block (reference SRGAN/VmambaIR/archs/MambaSISR6_arch.py):
//   norm1 + in_conv (+SiLU on the z half)        :166-195, :487-489       (prologue LN, epilogue bias + SiLU range)
//   x_proj for the 4 directions as ONE GEMM        :409-410                 (fp32 output)
//   channel gate + out_conv + residual             :494-498, :512           (prologue per-(b,k) gate, epilogue residual)
//   norm2 + project_in                             :213-214, :513           (prologue LN)
//   project_out + residual                         :217, :513               (epilogue residual)
// bf16/fp16 I/O: tensor cores (mma.sync m16n8k16, fp32 accumulate) on smem tiles;  fp32 I/O: FFMA tiles
// (the fp32 mode exists for 1e-3 parity against the reference, not for speed).
// Tile: 64 pixels x 64 output channels per step, the whole K (<=512) of the pixel tile resident in smem so the
// LayerNorm statistics are computed once in the prologue; larger K streams in chunks of 512.
#include <stdlib.h>

#include "common.cuh"
#include "oss_params.h"

namespace vmb {

constexpr int PL_PT = 64;      // pixels per CTA
constexpr int PL_MT = 64;      // output channels per step
constexpr int PL_KC = 768;     // resident K chunk: PL_KC / 2 = 384 fp32 rows (the widest LayerNorm of the nets, dim*8; 221 KB of smem)
constexpr int PL_THREADS = 128;

template <typename T> struct MmaType;
template <> struct MmaType<__nv_bfloat16> {
    __device__ static void mma(float* c, const uint32_t* a, const uint32_t* b) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
};
template <> struct MmaType<__half> {
    __device__ static void mma(float* c, const uint32_t* a, const uint32_t* b) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
};

__device__ __forceinline__ float silu_f(float v) { return v * rcp_approx(1.f + ex2(-v * kLog2e)); }

// ---- staging of the activation tile [kc][64 px] (+ optional LN / gate prologue) --------------------------
template <typename in_t, typename st_t>
__device__ __forceinline__ void stage_x(st_t* __restrict__ sX, int XP, const PixlinParams& p, int b, int p0, int k0, int kc,
                                        int kpad) {
    constexpr int V = Vec<in_t>::N;
    const in_t* __restrict__ xb = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;
    const int groups = PL_PT / V;
    for (int it = threadIdx.x; it < kpad * groups; it += PL_THREADS) {
        const int k = it / groups, pg = (it % groups) * V;
        float f[V];
        if (k < kc) {
            load_vec<in_t>(xb + (int64_t)(k0 + k) * p.x_cs + p0 + pg, f, p.P - (p0 + pg), p.vec_ok);
        } else {
#pragma unroll
            for (int i = 0; i < V; ++i) f[i] = 0.f;
        }
#pragma unroll
        for (int i = 0; i < V; ++i) sX[k * XP + pg + i] = st_t(f[i]);
    }
}

template <typename st_t>
__device__ __forceinline__ void prologue(st_t* __restrict__ sX, int XP, const PixlinParams& p, int b, int K, float* sStat) {
    if (p.ln_mode) {
        __syncthreads();
        // per-pixel statistics over the K channels (two-pass, fp32) -- 2 threads per pixel
        const int px = threadIdx.x % PL_PT, half = threadIdx.x / PL_PT;
        float s = 0.f;
        for (int k = half; k < K; k += 2) s += float(sX[k * XP + px]);
        sStat[half * PL_PT + px] = s;
        __syncthreads();
        const float mu = (sStat[px] + sStat[PL_PT + px]) / K;
        __syncthreads();
        float v = 0.f;
        for (int k = half; k < K; k += 2) {
            const float dlt = float(sX[k * XP + px]) - mu;
            v += dlt * dlt;
        }
        sStat[half * PL_PT + px] = v;
        __syncthreads();
        const float rstd = rsqrtf((sStat[px] + sStat[PL_PT + px]) / K + 1e-5f);
        __syncthreads();
        sStat[px] = mu;
        sStat[PL_PT + px] = rstd;
        __syncthreads();
        for (int it = threadIdx.x; it < K * PL_PT; it += PL_THREADS) {
            const int k = it / PL_PT, q = it % PL_PT;
            float xv = float(sX[k * XP + q]);
            xv = p.ln_mode == 1 ? (xv - sStat[q]) * sStat[PL_PT + q] * p.ln_w[k] + p.ln_b[k] : xv * sStat[PL_PT + q] * p.ln_w[k];
            sX[k * XP + q] = st_t(xv);
        }
    }
    if (p.gate_mode) {
        __syncthreads();
        const float* __restrict__ g = p.gate + (int64_t)b * p.g_bs;
        for (int it = threadIdx.x; it < K * PL_PT; it += PL_THREADS) {
            const int k = it / PL_PT, q = it % PL_PT;
            const float xv = float(sX[k * XP + q]);
            sX[k * XP + q] = st_t(p.gate_mode == 1 ? fmaf(xv, g[k], xv) : xv + g[k]);
        }
    }
}

template <typename in_t, typename st_t>
__device__ __forceinline__ void stage_w(st_t* __restrict__ sW, int WP, const PixlinParams& p, int m0, int k0, int kc, int kpad) {
    constexpr int V = Vec<in_t>::N;
    const in_t* __restrict__ w = reinterpret_cast<const in_t*>(p.w);
    const int groups = kpad / V;  // kpad is a multiple of 16
    const bool vec = p.w_vec;     // rows 16 B aligned and padded (w_ld % V == 0, w_ld >= kpad_all)
    for (int it = threadIdx.x; it < PL_MT * groups; it += PL_THREADS) {
        const int m = it / groups, k = (it % groups) * V;
        float f[V];
        if (m0 + m < p.M) {
            load_vec<in_t>(w + (int64_t)(m0 + m) * p.w_ld + k0 + k, f, vec ? V : kc - k, vec);
            if (!vec) {
#pragma unroll
                for (int i = 0; i < V; ++i) f[i] = (k + i < kc) ? f[i] : 0.f;
            }
        } else {
#pragma unroll
            for (int i = 0; i < V; ++i) f[i] = 0.f;
        }
#pragma unroll
        for (int i = 0; i < V; ++i) sW[m * WP + k + i] = st_t(f[i]);
    }
}

// ---- epilogue from the fp32 smem tile: bias, SiLU range, residual, store ---------------------------------
template <typename in_t, typename out_t>
__device__ __forceinline__ void epilogue(const float* __restrict__ sOut, int OP, const PixlinParams& p, int b, int p0, int m0) {
    constexpr int G = 8;  // pixels per item
    const in_t* __restrict__ res = p.residual ? reinterpret_cast<const in_t*>(p.residual) + (int64_t)b * p.r_bs : nullptr;
    out_t* __restrict__ ob = reinterpret_cast<out_t*>(p.out) + (int64_t)b * p.o_bs;
    for (int it = threadIdx.x; it < PL_MT * (PL_PT / G); it += PL_THREADS) {
        const int m = it / (PL_PT / G), q = (it % (PL_PT / G)) * G;
        const int mg = m0 + m;
        if (mg >= p.M) continue;
        const int valid = p.P - (p0 + q);
        if (valid <= 0) continue;
        float v[G];
        const float bs = p.bias ? p.bias[mg] : 0.f;
        const bool act = mg >= p.act_from && mg < p.act_to;
#pragma unroll
        for (int i = 0; i < G; ++i) {
            float t = sOut[m * OP + q + i] + bs;
            v[i] = act ? silu_f(t) : t;
        }
        if (res) {
            float r[G];
            constexpr int VI = Vec<in_t>::N;
#pragma unroll
            for (int j = 0; j < G / VI; ++j) load_vec<in_t>(res + (int64_t)mg * p.r_cs + p0 + q + j * VI, r + j * VI, valid - j * VI, p.vec_ok);
#pragma unroll
            for (int i = 0; i < G; ++i) v[i] += r[i];
        }
        constexpr int VO = Vec<out_t>::N;
#pragma unroll
        for (int j = 0; j < G / VO; ++j) store_vec<out_t>(ob + (int64_t)mg * p.o_cs + p0 + q + j * VO, v + j * VO, valid - j * VO, p.vec_ok);
    }
}

// ---- tensor-core kernel (bf16 / fp16 I/O) ----------------------------------------------------------------
// 256 threads = 8 warps as 2 (M halves of 32) x 4 (pixel quarters of PT/4); the K x PT activation tile stays in
// smem for all output-channel tiles; weight tiles (64 x K) arrive by cp.async, double-buffered, one barrier per tile;
// each warp drains its accumulators through a private smem patch (no CTA barrier) into 64 B-contiguous row stores.
constexpr int PL2_THREADS = 256;
constexpr int PL2_KC = 384;  // resident K (LayerNorm prologue needs the whole K); larger K streams in chunks

__device__ __forceinline__ void cp_async16_pl(void* smem_dst, const void* gsrc, int src_bytes) {
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}

template <typename in_t, int PT>
__device__ __forceinline__ void stage_x2(in_t* __restrict__ sX, int XP, const PixlinParams& p, int b, int p0, int k0, int kc,
                                         int kpad) {
    constexpr int V = Vec<in_t>::N;
    const in_t* __restrict__ xb = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;
    constexpr int groups = PT / V;
    if (p.vec_ok) {  // asynchronous 16 B copies: every thread keeps all of its copies in flight (memory-level parallelism)
        for (int it = threadIdx.x; it < kpad * groups; it += PL2_THREADS) {
            const int k = it / groups, pg = (it % groups) * V;
            const bool ok = k < kc && p0 + pg < p.P;
            cp_async16_pl(sX + k * XP + pg, ok ? (const void*)(xb + (int64_t)(k0 + k) * p.x_cs + p0 + pg) : (const void*)xb,
                          ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        return;
    }
    for (int it = threadIdx.x; it < kpad * groups; it += PL2_THREADS) {
        const int k = it / groups, pg = (it % groups) * V;
        in_t tmp[V];
        const int valid = p.P - (p0 + pg);
#pragma unroll
        for (int i = 0; i < V; ++i)
            tmp[i] = (k < kc && i < valid) ? xb[(int64_t)(k0 + k) * p.x_cs + p0 + pg + i] : from_f32<in_t>(0.f);
        *reinterpret_cast<uint4*>(sX + k * XP + pg) = *reinterpret_cast<uint4*>(tmp);
    }
}

template <typename T> __device__ __forceinline__ float2 unpack2(uint32_t v);
template <> __device__ __forceinline__ float2 unpack2<__nv_bfloat16>(uint32_t v) {
    return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
}
template <> __device__ __forceinline__ float2 unpack2<__half>(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2*>(&v));
}

// LayerNorm / gate prologue on the resident tile, two adjacent pixels per thread (packed 32-bit smem accesses)
template <typename in_t, int PT>
__device__ __forceinline__ void prologue2(in_t* __restrict__ sX, int XP, const PixlinParams& p, int b, int K, float* sStat) {
    constexpr int PP = PT / 2;               // pixel pairs
    constexpr int SL = PL2_THREADS / PP;     // K slices (4 or 8)
    const int px = (threadIdx.x % PP) * 2, sl = threadIdx.x / PP;
    float2* st0 = reinterpret_cast<float2*>(sStat);   // [SL][PP]
    float2* st1 = st0 + SL * PP;                       // [SL][PP]
    if (p.ln_mode) {
        __syncthreads();
        float2 s = make_float2(0.f, 0.f);
        for (int k = sl; k < K; k += SL) {
            const float2 v = unpack2<in_t>(*reinterpret_cast<const uint32_t*>(sX + k * XP + px));
            s.x += v.x;
            s.y += v.y;
        }
        st0[sl * PP + px / 2] = s;
        __syncthreads();
        float2 mu = make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < SL; ++i) {
            const float2 t = st0[i * PP + px / 2];
            mu.x += t.x;
            mu.y += t.y;
        }
        mu.x /= K;
        mu.y /= K;
        float2 v2 = make_float2(0.f, 0.f);
        for (int k = sl; k < K; k += SL) {
            const float2 v = unpack2<in_t>(*reinterpret_cast<const uint32_t*>(sX + k * XP + px));
            v2.x = fmaf(v.x - mu.x, v.x - mu.x, v2.x);
            v2.y = fmaf(v.y - mu.y, v.y - mu.y, v2.y);
        }
        st1[sl * PP + px / 2] = v2;
        __syncthreads();
        float2 var = make_float2(0.f, 0.f);
#pragma unroll
        for (int i = 0; i < SL; ++i) {
            const float2 t = st1[i * PP + px / 2];
            var.x += t.x;
            var.y += t.y;
        }
        const float r0 = rsqrtf(var.x / K + 1e-5f), r1 = rsqrtf(var.y / K + 1e-5f);
        const bool wb = p.ln_mode == 1;
        const float m0 = wb ? mu.x : 0.f, m1 = wb ? mu.y : 0.f;
        for (int k = sl; k < K; k += SL) {
            uint32_t* ptr = reinterpret_cast<uint32_t*>(sX + k * XP + px);
            const float2 v = unpack2<in_t>(*ptr);
            const float w = p.ln_w[k] , bb = wb ? p.ln_b[k] : 0.f;
            *ptr = pack2<in_t>(fmaf((v.x - m0) * r0, w, bb), fmaf((v.y - m1) * r1, w, bb));
        }
    }
    if (p.gate_mode) {
        __syncthreads();
        const float* __restrict__ g = p.gate + (int64_t)b * p.g_bs;
        for (int k = sl; k < K; k += SL) {
            uint32_t* ptr = reinterpret_cast<uint32_t*>(sX + k * XP + px);
            const float2 v = unpack2<in_t>(*ptr);
            const float gk = g[k];
            *ptr = p.gate_mode == 1 ? pack2<in_t>(fmaf(v.x, gk, v.x), fmaf(v.y, gk, v.y)) : pack2<in_t>(v.x + gk, v.y + gk);
        }
    }
}

// weight tile [64][kpad] of output channels [m0, m0+64), K range [k0, k0+kc): cp.async when rows are padded/aligned
template <typename in_t>
__device__ __forceinline__ void stage_w2(in_t* __restrict__ sW, int WP, const PixlinParams& p, int m0, int k0, int kc, int kpad) {
    constexpr int V = Vec<in_t>::N;
    const in_t* __restrict__ w = reinterpret_cast<const in_t*>(p.w);
    const int groups = kpad / V;
    // 16 x 16 thread grid over (rows, 16-byte groups): no integer division in the loop
    const int tm = threadIdx.x >> 4, tk = threadIdx.x & 15;
    for (int m = tm; m < PL_MT; m += 16) {
        const bool row_ok = m0 + m < p.M;
        const in_t* __restrict__ wrow = w + (int64_t)(row_ok ? m0 + m : 0) * p.w_ld + k0;
        for (int kg = tk; kg < groups; kg += 16) {
            const int k = kg * V;
            in_t* dst = sW + m * WP + k;
            if (p.w_vec) {
                cp_async16_pl(dst, wrow + k, row_ok ? 16 : 0);
            } else {
                in_t tmp[V];
#pragma unroll
                for (int i = 0; i < V; ++i) tmp[i] = (row_ok && k + i < kc) ? wrow[k + i] : from_f32<in_t>(0.f);
                *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<uint4*>(tmp);
            }
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

template <typename in_t, typename out_t, int PT>
__global__ void __launch_bounds__(PL2_THREADS) pixlin_mma_kernel(const PixlinParams p) {
    pdl_trigger();
    pdl_wait();
    constexpr int WN = PT / 4;       // pixels per warp
    constexpr int NT8 = WN / 8;      // n8 tiles per warp
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int kpad_all = (p.K + 15) / 16 * 16;
    const int KC = min(kpad_all, PL2_KC);
    const int XP = PT + 8, WP = KC + 8;
    constexpr int OP = WN + 4;
    in_t* sX = reinterpret_cast<in_t*>(smem_raw);                    // [KC][XP]
    in_t* sW0 = sX + KC * XP;                                        // [2][64][WP]
    float* sOut = reinterpret_cast<float*>(sW0 + p.w_tiles * PL_MT * WP);  // [8 warps][16][OP]
    float* sStat = sOut + 8 * 16 * OP;                               // [1024]
    const int b = blockIdx.z, p0 = blockIdx.x * PT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wm = warp >> 2, wn = warp & 3;                         // 2 x 4 warp grid
    const int nkc = (kpad_all + KC - 1) / KC;
    const bool resident = nkc == 1;
    const int mtiles = (p.M + PL_MT - 1) / PL_MT;
    const int my_tiles = (mtiles - (int)blockIdx.y + (int)gridDim.y - 1) / (int)gridDim.y;
    const int steps = my_tiles * nkc;  // (m-tile, k-chunk) steps of this CTA

    auto step_m0 = [&](int s) { return ((int)blockIdx.y + (s / nkc) * (int)gridDim.y) * PL_MT; };
    auto step_k0 = [&](int s) { return (s % nkc) * KC; };
    const bool w_all = p.w_all;  // every weight tile of this CTA resident: one batch of copies, no per-tile wait / barrier
    if (w_all) {
        for (int s = 0; s < steps; ++s) stage_w2<in_t>(sW0 + s * PL_MT * WP, WP, p, step_m0(s), 0, p.K, kpad_all);
    } else if (steps > 0) {
        stage_w2<in_t>(sW0, WP, p, step_m0(0), step_k0(0), min(p.K - step_k0(0), KC), min(kpad_all - step_k0(0), KC));
    }
    if (resident) {
        stage_x2<in_t, PT>(sX, XP, p, b, p0, 0, p.K, KC);
        prologue2<in_t, PT>(sX, XP, p, b, p.K, sStat);
    }
    float acc[2][NT8][4];
    float* myOut = sOut + warp * 16 * OP;
    const in_t* __restrict__ res = p.residual ? reinterpret_cast<const in_t*>(p.residual) + (int64_t)b * p.r_bs : nullptr;
    out_t* __restrict__ ob = reinterpret_cast<out_t*>(p.out) + (int64_t)b * p.o_bs;

    for (int s = 0; s < steps; ++s) {
        const int m0 = step_m0(s), k0 = step_k0(s);
        const int kpad = min(kpad_all - k0, KC);
        in_t* sW = sW0 + (w_all ? s : (s & 1)) * PL_MT * WP;
        if (s % nkc == 0) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < NT8; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
        }
        if (!resident) {
            __syncthreads();  // previous chunk's X fully consumed
            stage_x2<in_t, PT>(sX, XP, p, b, p0, k0, min(p.K - k0, KC), kpad);
        }
        if (!w_all || s == 0) {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();  // W[s] (and X) visible to all; everyone is done reading the other W buffer
        }
        if (!w_all && s + 1 < steps)
            stage_w2<in_t>(sW0 + ((s + 1) & 1) * PL_MT * WP, WP, p, step_m0(s + 1), step_k0(s + 1),
                           min(p.K - step_k0(s + 1), KC), min(kpad_all - step_k0(s + 1), KC));
        for (int kk = 0; kk < kpad; kk += 16) {
            uint32_t af[2][4], bf[NT8][2];
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                const in_t* addr = sW + (wm * 32 + mi * 16 + (lane & 15)) * WP + kk + ((lane >> 4) << 3);
                const uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(addr));
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(af[mi][0]), "=r"(af[mi][1]), "=r"(af[mi][2]), "=r"(af[mi][3]) : "r"(sa));
            }
#pragma unroll
            for (int nj = 0; nj < NT8; nj += 2) {
                const in_t* addr = sX + (kk + (lane & 15)) * XP + wn * WN + nj * 8 + ((lane >> 4) << 3);
                const uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(addr));
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(bf[nj][0]), "=r"(bf[nj][1]), "=r"(bf[nj + 1][0]), "=r"(bf[nj + 1][1]) : "r"(sa));
            }
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int nj = 0; nj < NT8; ++nj) MmaType<in_t>::mma(acc[mi][nj], af[mi], bf[nj]);
        }
        if (s % nkc != nkc - 1) continue;
        // ---- epilogue of this output-channel tile ----
        if constexpr (sizeof(out_t) == 2) {
            if (p.vec_ok) {  // straight from the accumulators: each thread owns 2 adjacent pixels of 16 (row, n8) fragments
#pragma unroll
                for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf) {
                        const int mg = m0 + wm * 32 + mi * 16 + hf * 8 + (lane >> 2);
                        if (mg >= p.M) continue;
                        const float bs = p.bias ? p.bias[mg] : 0.f;
                        const bool act = mg >= p.act_from && mg < p.act_to;
#pragma unroll
                        for (int nj = 0; nj < NT8; ++nj) {
                            const int pg = p0 + wn * WN + nj * 8 + 2 * (lane & 3);
                            if (pg >= p.P) continue;
                            float v0 = acc[mi][nj][hf * 2] + bs, v1 = acc[mi][nj][hf * 2 + 1] + bs;
                            if (act) {
                                v0 = silu_f(v0);
                                v1 = silu_f(v1);
                            }
                            if (res) {
                                const float2 r2 = unpack2<in_t>(*reinterpret_cast<const uint32_t*>(res + (int64_t)mg * p.r_cs + pg));
                                v0 += r2.x;
                                v1 += r2.y;
                            }
                            *reinterpret_cast<uint32_t*>(ob + (int64_t)mg * p.o_cs + pg) = pack2<out_t>(v0, v1);
                        }
                    }
                continue;
            }
        }
        // generic path: warp-private smem patch (16 rows at a time) -> row-contiguous stores
        constexpr int G = 8, GPR = WN / G;  // 8-pixel groups per row
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
            __syncwarp();
#pragma unroll
            for (int nj = 0; nj < NT8; ++nj) {
                const int row = lane >> 2, col = nj * 8 + 2 * (lane & 3);
                *reinterpret_cast<float2*>(&myOut[row * OP + col]) = make_float2(acc[mi][nj][0], acc[mi][nj][1]);
                *reinterpret_cast<float2*>(&myOut[(row + 8) * OP + col]) = make_float2(acc[mi][nj][2], acc[mi][nj][3]);
            }
            __syncwarp();
#pragma unroll
            for (int it = lane; it < 16 * GPR; it += 32) {
                const int row = it / GPR, q = (it % GPR) * G;
                const int mg = m0 + wm * 32 + mi * 16 + row;
                const int pg = p0 + wn * WN + q;
                const int valid = p.P - pg;
                if (mg >= p.M || valid <= 0) continue;
                float v[G];
                {
                    const float4 a0 = *reinterpret_cast<const float4*>(&myOut[row * OP + q]);
                    const float4 a1 = *reinterpret_cast<const float4*>(&myOut[row * OP + q + 4]);
                    v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w;
                    v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
                }
                if (p.bias) {
                    const float bs = p.bias[mg];
#pragma unroll
                    for (int i = 0; i < G; ++i) v[i] += bs;
                }
                if (mg >= p.act_from && mg < p.act_to) {
#pragma unroll
                    for (int i = 0; i < G; ++i) v[i] = silu_f(v[i]);
                }
                if (res) {
                    float rr[G];
                    constexpr int VI = Vec<in_t>::N;
#pragma unroll
                    for (int j = 0; j < G / VI; ++j) load_vec<in_t>(res + (int64_t)mg * p.r_cs + pg + j * VI, rr + j * VI, valid - j * VI, p.vec_ok);
#pragma unroll
                    for (int i = 0; i < G; ++i) v[i] += rr[i];
                }
                constexpr int VO = Vec<out_t>::N;
#pragma unroll
                for (int j = 0; j < G / VO; ++j) store_vec<out_t>(ob + (int64_t)mg * p.o_cs + pg + j * VO, v + j * VO, valid - j * VO, p.vec_ok);
            }
        }
    }
}

// ---- fp32 kernel (FFMA) ----------------------------------------------------------------------------------
template <typename out_t>
__global__ void __launch_bounds__(PL_THREADS) pixlin_f32_kernel(const PixlinParams p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int kpad_all = (p.K + 15) / 16 * 16;
    const int KC = min(kpad_all, PL_KC / 2);
    const int XP = PL_PT + 4, WP = KC + 1, OP = PL_PT + 4;
    float* sX = reinterpret_cast<float*>(smem_raw);   // [KC][XP]
    float* sW = sX + KC * XP;                         // [MT][WP]
    float* sOut = sW + PL_MT * WP;                    // [MT][OP]
    float* sStat = sOut + PL_MT * OP;
    const int b = blockIdx.z, p0 = blockIdx.x * PL_PT;
    const int tm = threadIdx.x / 8, tp = threadIdx.x % 8;  // 16 x 8 thread grid: 4 rows x 8 pixels each
    const int nkc = (kpad_all + KC - 1) / KC;
    const bool resident = nkc == 1;
    if (resident) {
        stage_x<float, float>(sX, XP, p, b, p0, 0, p.K, KC);
        prologue<float>(sX, XP, p, b, p.K, sStat);
    }
    for (int m0 = blockIdx.y * PL_MT; m0 < p.M; m0 += gridDim.y * PL_MT) {
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        for (int kc_i = 0; kc_i < nkc; ++kc_i) {
            const int k0 = kc_i * KC, kc = min(p.K - k0, KC), kpad = (kc + 15) / 16 * 16;
            __syncthreads();
            if (!resident) stage_x<float, float>(sX, XP, p, b, p0, k0, kc, kpad);
            stage_w<float, float>(sW, WP, p, m0, k0, kc, kpad);
            __syncthreads();
            for (int k = 0; k < kc; ++k) {
                const float4 x0 = *reinterpret_cast<const float4*>(&sX[k * XP + tp * 8]);
                const float4 x1 = *reinterpret_cast<const float4*>(&sX[k * XP + tp * 8 + 4]);
                const float xs[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float wv = sW[(tm * 4 + i) * WP + k];
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(wv, xs[j], acc[i][j]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) sOut[(tm * 4 + i) * OP + tp * 8 + j] = acc[i][j];
        __syncthreads();
        epilogue<float, out_t>(sOut, OP, p, b, p0, m0);
    }
}

static size_t pixlin_smem(int K, int elt, int PT = 64, int wtiles = 2) {
    const int kpad = (K + 15) / 16 * 16;
    if (elt == 2) {
        const int KC = kpad < PL2_KC ? kpad : PL2_KC;
        return (size_t)2 * (KC * (PT + 8) + wtiles * PL_MT * (KC + 8)) + 4 * (8 * 16 * (PT / 4 + 4) + 1024);
    }
    const int KC = kpad < PL_KC / 2 ? kpad : PL_KC / 2;
    return (size_t)4 * (KC * (PL_PT + 4) + PL_MT * (KC + 1) + PL_MT * (PL_PT + 4) + 2 * PL_PT);
}

template <typename K>
static int launch2(K kern, PixlinParams p, int PT, cudaStream_t stream) {
    const int ptiles = (p.P + PT - 1) / PT, mtiles = (p.M + PL_MT - 1) / PL_MT;
    const int kpad = (p.K + 15) / 16 * 16;
    // split the output channels over blockIdx.y (a) until the grid covers the SMs ~1.5x and (b), when K is resident,
    // until all weight tiles of a CTA fit in <= 64 KB of smem: then they are fetched in one batch (no per-tile wait)
    int msplit = 1;
    while (msplit < mtiles && (long)ptiles * p.B * msplit < 3L * num_sms() / 2) ++msplit;
    p.w_all = false;
    int wtiles = 2;
    if (kpad <= PL2_KC && p.w_vec) {
        int ms = msplit;
        while (ms < mtiles && (size_t)((mtiles + ms - 1) / ms) * PL_MT * (kpad + 8) * 2 > 64 * 1024) ++ms;
        const int per = (mtiles + ms - 1) / ms;
        if ((size_t)per * PL_MT * (kpad + 8) * 2 <= 64 * 1024) {
            msplit = ms;
            p.w_all = true;
            wtiles = per;
        }
    }
    p.w_tiles = wtiles;
    const size_t smem = pixlin_smem(p.K, 2, PT, wtiles);
    VMB_CHECK(smem <= 227 * 1024, "pixlin: K=%d needs %zu B of shared memory", p.K, smem);
    if (smem > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(ptiles, msplit, p.B);
    VMB_CUDA(launch_pdl(kern, grid, dim3(PL2_THREADS), smem, stream, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

template <typename in_t>
static int launch_mma(const PixlinParams& p, int out_dtype, cudaStream_t stream) {
    // 128-pixel tiles when there are enough pixels to fill the GPU with them, else 64
    bool big = (long)((p.P + 127) / 128) * p.B >= num_sms() && pixlin_smem(p.K, 2, 128, 2) <= 100 * 1024;
    if (const char* e = getenv("VMB_PL_PT")) big = big && atoi(e) == 128;  // tuning override
    const int PT = big ? 128 : 64;
    if (out_dtype == VMB_F32)
        return big ? launch2(pixlin_mma_kernel<in_t, float, 128>, p, PT, stream)
                   : launch2(pixlin_mma_kernel<in_t, float, 64>, p, PT, stream);
    return big ? launch2(pixlin_mma_kernel<in_t, in_t, 128>, p, PT, stream)
               : launch2(pixlin_mma_kernel<in_t, in_t, 64>, p, PT, stream);
}


// ---- K-streamed variant: reduction-heavy plain GEMMs (K > 384, no prologue) ---------------------------------------------------
// The data gradients W^T dY of the EFFN (2h = 510 -> C = 96) and of the folded x_proj / dt_proj (4(C + 2N) = 512 -> 96) in the
// training path: the input (K x P) is the big operand, the output small.  The resident-K kernel above re-stages its activation tile
// per output-channel tile and K chunk without overlap; here a CTA owns 128 output channels x 64 pixels
// and walks K in 32-row stages through a 4-deep cp.async ring (W stage [128][32], X stage [32][64]), mma.sync m16n8k16,
// bias / SiLU range / residual straight from the accumulators.
constexpr int KS_MT = 128, KS_PT = 64, KS_KC = 32, KS_THREADS = 128;
constexpr int KS_WP = KS_KC + 8, KS_XP = KS_PT + 8;
constexpr size_t ks_smem(int stages) { return (size_t)stages * (KS_MT * KS_WP + KS_KC * KS_XP) * 2; }

template <typename in_t, int KS_ST>
__global__ void __launch_bounds__(KS_THREADS) pixlin_kstream_kernel(const PixlinParams p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    in_t* sW = reinterpret_cast<in_t*>(smem_raw);          // [ST][128][WP]
    in_t* sX = sW + (size_t)KS_ST * KS_MT * KS_WP;         // [ST][KC][XP]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 1, wn = warp & 1;               // 2 x 2 warps: 64 output channels x 32 pixels each
    const int b = blockIdx.z, p0 = blockIdx.x * KS_PT, m0 = blockIdx.y * KS_MT;
    const int kpad16 = (p.K + 15) / 16 * 16;
    const int kw = p.w_ld < kpad16 ? (int)p.w_ld : kpad16;  // weight columns that exist (zero-padded beyond K)
    const int nk = (p.K + KS_KC - 1) / KS_KC;
    const in_t* __restrict__ xb = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;
    const in_t* __restrict__ wg = reinterpret_cast<const in_t*>(p.w);

    auto stage = [&](int kt) {
        const int buf = kt % KS_ST, k0 = kt * KS_KC;
        in_t* w_s = sW + (size_t)buf * KS_MT * KS_WP;
        in_t* x_s = sX + (size_t)buf * KS_KC * KS_XP;
#pragma unroll
        for (int it = tid; it < KS_MT * (KS_KC / 8); it += KS_THREADS) {
            const int row = it / (KS_KC / 8), c = (it % (KS_KC / 8)) * 8;
            const int m = m0 + row, k = k0 + c;
            const bool ok = m < p.M && k + 8 <= kw;
            cp_async16_pl(w_s + row * KS_WP + c, ok ? (const void*)(wg + (int64_t)m * p.w_ld + k) : (const void*)wg, ok ? 16 : 0);
        }
#pragma unroll
        for (int it = tid; it < KS_KC * (KS_PT / 8); it += KS_THREADS) {
            const int row = it / (KS_PT / 8), c = (it % (KS_PT / 8)) * 8;
            const int k = k0 + row, px = p0 + c;
            const bool ok = k < p.K && px < p.P;  // P % 8 == 0 (vec_ok): whole vectors
            cp_async16_pl(x_s + row * KS_XP + c, ok ? (const void*)(xb + (int64_t)k * p.x_cs + px) : (const void*)xb, ok ? 16 : 0);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

#pragma unroll
    for (int s = 0; s < KS_ST - 1; ++s) {
        if (s < nk) stage(s);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (int kt = 0; kt < nk; ++kt) {
        asm volatile("cp.async.wait_group %0;" ::"n"(KS_ST - 2) : "memory");
        __syncthreads();  // stage kt landed for everyone; everyone is done with stage kt-1 (whose buffer is refilled next)
        if (kt + KS_ST - 1 < nk) stage(kt + KS_ST - 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        const in_t* w_s = sW + (size_t)(kt % KS_ST) * KS_MT * KS_WP;
        const in_t* x_s = sX + (size_t)(kt % KS_ST) * KS_KC * KS_XP;
#pragma unroll
        for (int kk = 0; kk < KS_KC; kk += 16) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int mi = 0; mi < 4; ++mi) {
                const uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(w_s + (wm * 64 + mi * 16 + (lane & 15)) * KS_WP + kk + ((lane >> 4) << 3)));
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(af[mi][0]), "=r"(af[mi][1]), "=r"(af[mi][2]), "=r"(af[mi][3]) : "r"(sa));
            }
#pragma unroll
            for (int nj = 0; nj < 4; nj += 2) {
                const uint32_t sa = static_cast<uint32_t>(__cvta_generic_to_shared(x_s + (kk + (lane & 15)) * KS_XP + wn * 32 + nj * 8 + ((lane >> 4) << 3)));
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(bf[nj][0]), "=r"(bf[nj][1]), "=r"(bf[nj + 1][0]), "=r"(bf[nj + 1][1]) : "r"(sa));
            }
#pragma unroll
            for (int mi = 0; mi < 4; ++mi)
#pragma unroll
                for (int nj = 0; nj < 4; ++nj) MmaType<in_t>::mma(acc[mi][nj], af[mi], bf[nj]);
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    // epilogue straight from the accumulators: each thread owns 2 adjacent pixels of its (row, n8) fragments
    const in_t* __restrict__ res = p.residual ? reinterpret_cast<const in_t*>(p.residual) + (int64_t)b * p.r_bs : nullptr;
    in_t* __restrict__ ob = reinterpret_cast<in_t*>(p.out) + (int64_t)b * p.o_bs;
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int mg = m0 + wm * 64 + mi * 16 + hf * 8 + (lane >> 2);
            if (mg >= p.M) continue;
            const float bs = p.bias ? p.bias[mg] : 0.f;
            const bool act = mg >= p.act_from && mg < p.act_to;
#pragma unroll
            for (int nj = 0; nj < 4; ++nj) {
                const int pg = p0 + wn * 32 + nj * 8 + 2 * (lane & 3);
                if (pg >= p.P) continue;
                float v0 = acc[mi][nj][hf * 2] + bs, v1 = acc[mi][nj][hf * 2 + 1] + bs;
                if (act) {
                    v0 = silu_f(v0);
                    v1 = silu_f(v1);
                }
                if (res) {
                    const float2 r2 = unpack2<in_t>(*reinterpret_cast<const uint32_t*>(res + (int64_t)mg * p.r_cs + pg));
                    v0 += r2.x;
                    v1 += r2.y;
                }
                *reinterpret_cast<uint32_t*>(ob + (int64_t)mg * p.o_cs + pg) = pack2<in_t>(v0, v1);
            }
        }
}

template <typename in_t, int ST>
static int launch_kstream2(const PixlinParams& p, cudaStream_t stream) {
    auto kern = pixlin_kstream_kernel<in_t, ST>;
    VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ks_smem(ST)));
    dim3 grid((p.P + KS_PT - 1) / KS_PT, (p.M + KS_MT - 1) / KS_MT, p.B);
    VMB_CHECK(grid.y <= 65535, "pixlin: too many output channels");
    VMB_CUDA(launch_pdl(kern, grid, dim3(KS_THREADS), ks_smem(ST), stream, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
template <typename in_t>
static int launch_kstream(const PixlinParams& p, cudaStream_t stream) {
    int st = 6;  // ring depth: bytes in flight per SM
    if (const char* e = getenv("VMB_KS_ST")) st = atoi(e);
    return st == 4 ? launch_kstream2<in_t, 4>(p, stream) : launch_kstream2<in_t, 6>(p, stream);
}

static bool kstream_applicable(const PixlinParams& p, int dtype, int out_dtype) {
    if (const char* e = getenv("VMB_PL_KSTREAM")) {
        if (atoi(e) == 0) return false;
    }
    return (dtype == VMB_BF16 || dtype == VMB_F16) && out_dtype == dtype && p.ln_mode == 0 && p.gate_mode == 0 && p.vec_ok && p.w_vec &&
           p.K > PL2_KC && p.M <= 2 * KS_MT;
}

template <typename K>
static int launch(K kern, const PixlinParams& p, size_t smem, cudaStream_t stream) {
    if (smem > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // split the output channels over blockIdx.y until the grid covers the SMs a few times
    const int ptiles = (p.P + PL_PT - 1) / PL_PT, mtiles = (p.M + PL_MT - 1) / PL_MT;
    int msplit = 1;
    while (msplit < mtiles && (long)ptiles * p.B * msplit < 3L * num_sms()) ++msplit;
    dim3 grid(ptiles, msplit, p.B);
    VMB_CUDA(launch_pdl(kern, grid, dim3(PL_THREADS), smem, stream, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int pixlin_launch(const PixlinParams& p, int dtype, int out_dtype, cudaStream_t stream) {
    VMB_CHECK(p.ln_mode == 0 || p.K <= (dtype == VMB_F32 ? PL_KC / 2 : PL2_KC), "pixlin: LayerNorm prologue needs K <= %d",
              dtype == VMB_F32 ? PL_KC / 2 : PL2_KC);
    VMB_CHECK(p.gate_mode == 0 || p.K <= (dtype == VMB_F32 ? PL_KC / 2 : PL2_KC), "pixlin: gate prologue needs resident K");
    if (pixlin_tc_applicable(p, dtype, out_dtype)) return pixlin_tc_launch(p, dtype, stream);  // wgmma path
    if (kstream_applicable(p, dtype, out_dtype))
        return dtype == VMB_BF16 ? launch_kstream<__nv_bfloat16>(p, stream) : launch_kstream<__half>(p, stream);
    const size_t smem = pixlin_smem(p.K, dtype == VMB_F32 ? 4 : 2);
    if (dtype == VMB_F32) {
        VMB_CHECK(out_dtype == VMB_F32, "pixlin: fp32 input needs fp32 output");
        return launch(pixlin_f32_kernel<float>, p, smem, stream);
    }
    if (dtype == VMB_BF16) return launch_mma<__nv_bfloat16>(p, out_dtype, stream);
    if (dtype == VMB_F16) return launch_mma<__half>(p, out_dtype, stream);
    set_error("pixlin: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

}  // namespace vmb
