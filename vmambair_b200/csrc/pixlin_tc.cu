// pixlin on the Hopper tensor cores: a persistent, warp-specialised wgmma pipeline.
//   out[b, m, p] = epi( sum_k W[m,k] * pro(x)[b,k,p] )      (same contract as pixlin.cu)
// Each CTA (one or two per SM) keeps the whole weight matrix resident in shared memory (K-major canonical GMMA layout) and walks
// 32-pixel tiles of the (b, p) plane:
//   warp 4    producer : cp.async of the next activation tiles into a 6-stage ring (MN-major canonical layout: pixels are
//                        the contiguous dimension of NCHW), 4 tiles in flight, mbarrier "full" per stage
//   warps 5-8 prologue : LayerNorm / channel gate on the resident tile, in place, one 8-pixel column group per warp
//                        (only when the call has one)
//   warps 0-3 consumer : one warpgroup issues the K/16 wgmma.m64n32k16 of 64 output channels back to back into register
//                        accumulators, waits for them, then runs the epilogue: quad transpose to 8 contiguous pixels per
//                        thread and row, bias / SiLU / residual, 16 B vector stores
// so loads, prologue and tensor-core work of different tiles overlap (and, with two CTAs per SM, the MMAs of one CTA with
// the epilogue of the other), and the weights are read once per CTA instead of once per tile.  One accumulator set per
// warpgroup on purpose: with two sets in flight across commit groups ptxas cannot prove the epilogue's reads safe and
// serialises every wgmma (C7514).  Legal for 16-bit I/O with 16 B aligned rows, M <= 512, K <= 256 and weights + ring <= 227 KB; selected by
// VMB_PIXLIN_TC only (pixlin_tc_applicable below), the mma.sync kernel of pixlin.cu is the default; FFMA kernel for fp32.
#include <stdlib.h>

#include "common.cuh"
#include "oss_params.h"

namespace vmb {

constexpr int TC_PT = 32;        // pixels per tile (GMMA N)
constexpr int TC_MT = 128;       // rows of one resident weight tile
constexpr int TC_MB = 64;        // output channels per wgmma (GMMA M)
constexpr int TC_NS = 6;         // activation ring stages
constexpr int TC_LA = 4;         // tiles the producer keeps in flight (cp.async groups)
constexpr int TC_THREADS = 288;  // consumer warpgroup + producer + 4 prologue warps
constexpr int TC_KGMAX = 32;     // K <= 256: a prologue lane keeps its column of the tile in registers
constexpr int TC_MAXMT = 4;      // M <= 512
constexpr size_t TC_SMEM_MAX = 227 * 1024;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// GMMA shared-memory descriptor, no swizzle (layout type 0): start address, leading / stride byte offsets in 16 B units.
// K-major operand: ((8,m),(8,2)):((1,SBO),(1,LBO)) in core-matrix rows; MN-major operand: ((8,n),(8,k)):((1,SBO),(1,LBO)).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;  // base_offset 0, layout_type 0 (no swizzle)
}
// D[64 x 32] (+)= A[64 x 16] * B[16 x 32]: A K-major (no transpose), B MN-major (transposed), fp32 accumulators
template <typename T> __device__ __forceinline__ void wgmma_m64n32k16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
#define VMB_WGMMA(TY)                                                                                                         \
    asm volatile(                                                                                                             \
        "{\n\t"                                                                                                               \
        ".reg .pred p;\n\t"                                                                                                   \
        "setp.ne.b32 p, %18, 0;\n\t"                                                                                          \
        "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " "                                                           \
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 1;\n\t"                               \
        "}\n"                                                                                                                 \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),        \
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])                           \
        : "l"(adesc), "l"(bdesc), "r"(accumulate))
template <> __device__ __forceinline__ void wgmma_m64n32k16<__nv_bfloat16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    VMB_WGMMA("bf16");
}
template <> __device__ __forceinline__ void wgmma_m64n32k16<__half>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    VMB_WGMMA("f16");
}
#undef VMB_WGMMA
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMAs that write them
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
    for (int i = 0; i < 16; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}

__device__ __forceinline__ float silu_tc(float v) { return v * rcp_approx(1.f + ex2(-v * kLog2e)); }
template <typename T> __device__ __forceinline__ float2 unpack2_tc(uint32_t v);
template <> __device__ __forceinline__ float2 unpack2_tc<__nv_bfloat16>(uint32_t v) {
    return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
}
template <> __device__ __forceinline__ float2 unpack2_tc<__half>(uint32_t v) {
    return __half22float2(*reinterpret_cast<const __half2*>(&v));
}
__device__ __forceinline__ void cp16(void* smem_dst, const void* gsrc, int nbytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(nbytes) : "memory");
}

// element (k, n) of one activation stage, canonical MN-major no-swizzle layout: core (k/8, n/8) = 128 B, row k%8, col n%8
__device__ __forceinline__ int b_off(int k, int n) { return (((k >> 3) * (TC_PT / 8) + (n >> 3)) << 6) + ((k & 7) << 3) + (n & 7); }

__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
// long waits (producer / prologue): back off between polls so that the pollers do not crowd the MIO queue that the
// working warps' LDS / STS / SHFL go through
__device__ __forceinline__ void mbar_wait_sleep(uint64_t* bar, uint32_t parity, int backoff_ns) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    for (;;) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) break;
        if (backoff_ns > 0) __nanosleep(backoff_ns);
    }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_wait_pending(int n) {  // at most n of this thread's cp.async groups still pending
    switch (n) {
        case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
        case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
        case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
        default: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
    }
}
__device__ __forceinline__ float2 sel4(const float2* v, int i) {  // v[i] for a run-time i without local memory
    float2 r = v[0];
    r = i == 1 ? v[1] : r;
    r = i == 2 ? v[2] : r;
    r = i == 3 ? v[3] : r;
    return r;
}

// debug trace (VMB_TC_TRACE=1): %globaltimer stamps per CTA -- [0] start, [1] barriers ready, [2] weights resident,
// [3] end; tile i < 10 at 4+6i: +0 copies landed, +1 prologue done, +2 MMA saw the operands, +3 MMAs issued,
// +4 epilogue saw the accumulator, +5 epilogue done
__device__ long long g_tc_trace[160 * 64];
__device__ __forceinline__ long long gtimer() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

struct TcShared {  // control block behind the operand buffers
    uint64_t full[TC_NS], ready[TC_NS], empty[TC_NS], wfull;
};

// KG: compile-time bound on K/8 (a prologue lane keeps that many packed pixel pairs in registers)
template <typename in_t, int KG>
__global__ void __launch_bounds__(TC_THREADS, 2) pixlin_tc_kernel(const PixlinParams p, const int trace, const int backoff) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    pdl_trigger();  // everything up to pdl_wait() below touches only weights / parameters and this CTA's own state
    if (!p.w_static) pdl_wait();  // training: the weights are the preceding kernel's output (vmb_prep_block_weights)
    long long* tr = (trace && blockIdx.x < 160) ? g_tc_trace + blockIdx.x * 64 : nullptr;
    if (tr && threadIdx.x == 0) tr[0] = gtimer();
    const int kpad = (p.K + 15) / 16 * 16;
    const int nmt = (p.M + TC_MT - 1) / TC_MT;
    in_t* sA = reinterpret_cast<in_t*>(smem_raw);                       // [nmt] weight tiles of 128 x kpad
    in_t* sX = sA + (size_t)nmt * TC_MT * kpad;                         // [TC_NS] activation stages of kpad x 32
    float* sLn = reinterpret_cast<float*>(sX + (size_t)TC_NS * kpad * TC_PT);  // [2][kpad] LayerNorm weight / bias
    float* sBias = sLn + 2 * kpad;                                               // [nmt*128] output bias
    TcShared* sh = reinterpret_cast<TcShared*>(sBias + nmt * TC_MT);

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);  // warp-uniform to the compiler: the wgmma issue path is not divergent
    const int ptiles = p.P / TC_PT;
    const int total = ptiles * p.B;
    const int my_n = ((int)blockIdx.x < total) ? (total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const bool has_pro = p.ln_mode != 0 || p.gate_mode != 0;
    const in_t* __restrict__ xg = reinterpret_cast<const in_t*>(p.x);
    const in_t* __restrict__ w = reinterpret_cast<const in_t*>(p.w);

    // ---- setup: barriers, LayerNorm parameters ----
    if (tid == 0) {
        for (int i = 0; i < TC_NS; ++i) {
            mbar_init(&sh->full[i], 32);
            mbar_init(&sh->ready[i], 128);
            mbar_init(&sh->empty[i], 4);  // lane 0 of each consumer warp, once the tile's MMAs have completed
        }
        mbar_init(&sh->wfull, TC_THREADS - 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (p.ln_mode)
        for (int k = tid; k < kpad; k += TC_THREADS) {
            sLn[k] = k < p.K ? p.ln_w[k] : 0.f;
            sLn[kpad + k] = (k < p.K && p.ln_mode == 1) ? p.ln_b[k] : 0.f;
        }
    for (int m = tid; m < nmt * TC_MT; m += TC_THREADS) sBias[m] = (p.bias && m < p.M) ? p.bias[m] : 0.f;
    __syncthreads();
    if (tr && threadIdx.x == 0) tr[1] = gtimer();

    // producer state (warp 4): tiles issued / tiles whose "full" barrier has been signalled
    int issued = 0, arrived = 0;
    auto issue_tile = [&](int it) {  // 16 B = 8 pixels of one k row = one core-matrix row
        const int s = it % TC_NS;
        mbar_wait_sleep(&sh->empty[s], ((it / TC_NS) & 1) ^ 1, backoff);
        const int t = blockIdx.x + it * gridDim.x;
        const int b = t / ptiles, p0 = (t - b * ptiles) * TC_PT;
        const in_t* xb = xg + (int64_t)b * p.x_bs + p0;
        in_t* dst = sX + (size_t)s * kpad * TC_PT;
        for (int i = lane; i < kpad * (TC_PT / 8); i += 32) {
            const int ng = i & (TC_PT / 8 - 1), k = i / (TC_PT / 8);
            const bool ok = k < p.K;
            cp16(dst + b_off(k, ng * 8), ok ? (const void*)(xb + (int64_t)k * p.x_cs + ng * 8) : (const void*)xg, ok ? 16 : 0);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    if (warp == 4) {
        // the first tiles go out before the weights have landed
        pdl_wait();
        while (issued < my_n && issued < TC_LA) issue_tile(issued++);
    } else {
        // resident weights: every tile of 128 rows, rows >= M zero-filled.  A warp request covers 8 rows x 64 B (whole
        // sectors from L2, 4-way instead of 32-way bank conflict on the core-matrix layout); a warp walks 8-row groups,
        // no integer division in the loop
        const int wq = warp < 4 ? warp : warp - 1;          // 0..7 among the eight loading warps
        const int kq = (kpad + 31) / 32;                    // groups of four 8-wide k chunks
        const int rows8 = nmt * (TC_MT / 8);
        const int kg_l = lane >> 3, m_l = lane & 7;
        for (int r8 = wq; r8 < rows8; r8 += 8) {
            const int mrow = r8 * 8 + m_l;
            const bool ok = mrow < p.M;
            const in_t* src = w + (int64_t)(ok ? mrow : 0) * p.w_ld;
            // element (m, k) of a 128-row weight tile, canonical K-major no-swizzle layout: core (k/8, m/8) = 128 B, row m%8, col k%8
            in_t* dst = sA + (size_t)(r8 >> 4) * TC_MT * kpad + (((r8 & 15) << 6) + (m_l << 3));
            for (int q = 0; q < kq; ++q) {
                const int kg = q * 4 + kg_l;
                if (kg * 8 < kpad) cp16(dst + (size_t)kg * (TC_MT / 8) * 64, src + kg * 8, ok ? 16 : 0);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        pdl_wait();  // the weight copies fly while the preceding kernel drains; gate / residual / out are touched after this
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(&sh->wfull);
    }

    if (warp == 4) {
        // ================= producer =================
        // a landed tile is signalled before the warp blocks on a ring stage that the MMAs have not released yet
        while (arrived < my_n) {
            bool can_issue = issued < my_n && issued - arrived < TC_LA;
            if (can_issue && issued > arrived) {
                const bool stage_free = mbar_test(&sh->empty[issued % TC_NS], ((issued / TC_NS) & 1) ^ 1);
                can_issue = __shfl_sync(0xffffffffu, stage_free ? 1 : 0, 0) != 0;
            }
            if (can_issue) {
                issue_tile(issued++);
                continue;
            }
            cp_wait_pending(issued - arrived - 1);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_arrive(&sh->full[arrived % TC_NS]);
            if (tr && lane == 0 && arrived < 10) tr[4 + 6 * arrived] = gtimer();
            ++arrived;
        }
    } else if (warp >= 5) {
        // ================= prologue: LayerNorm / gate in place =================
        // warp 5+ng owns the 8-pixel column group ng of every tile; one warp instruction covers one 128 B core matrix
        // (lane = (k%8, pixel pair)), and a lane keeps its K/8 packed pixel pairs in registers between the passes
        if (has_pro) {
            const int ng = warp - 5, r = lane >> 2;
            const int kgs = kpad / 8;
            for (int it = 0; it < my_n; ++it) {
                const int s = it % TC_NS;
                mbar_wait_sleep(&sh->full[s], (it / TC_NS) & 1, backoff);
                uint32_t* st = reinterpret_cast<uint32_t*>(sX + (size_t)s * kpad * TC_PT) + ng * 32 + lane;
                const int t = blockIdx.x + it * gridDim.x;
                const int b = t / ptiles;
                const float* __restrict__ g = p.gate_mode ? p.gate + (int64_t)b * p.g_bs : nullptr;
                uint32_t xv[KG];
#pragma unroll
                for (int kg = 0; kg < KG; ++kg) xv[kg] = kg < kgs ? st[kg * 128] : 0u;
                float mu0 = 0.f, mu1 = 0.f, rs0 = 1.f, rs1 = 1.f;
                if (p.ln_mode) {
                    float s0 = 0.f, s1 = 0.f;
#pragma unroll
                    for (int kg = 0; kg < KG; ++kg) {
                        const float2 f = unpack2_tc<in_t>(xv[kg]);  // rows >= K are zero
                        s0 += f.x;
                        s1 += f.y;
                    }
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
                        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                    }
                    mu0 = s0 / p.K;
                    mu1 = s1 / p.K;
                    float v0 = 0.f, v1 = 0.f;
#pragma unroll
                    for (int kg = 0; kg < KG; ++kg) {
                        if (kg * 8 + r < p.K) {
                            const float2 f = unpack2_tc<in_t>(xv[kg]);
                            const float d0 = f.x - mu0, d1 = f.y - mu1;
                            v0 = fmaf(d0, d0, v0);
                            v1 = fmaf(d1, d1, v1);
                        }
                    }
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) {
                        v0 += __shfl_xor_sync(0xffffffffu, v0, o);
                        v1 += __shfl_xor_sync(0xffffffffu, v1, o);
                    }
                    rs0 = rsqrtf(v0 / p.K + 1e-5f);
                    rs1 = rsqrtf(v1 / p.K + 1e-5f);
                }
                const bool wb = p.ln_mode == 1;
#pragma unroll
                for (int kg = 0; kg < KG; ++kg) {
                    const int k = kg * 8 + r;
                    if (k < p.K) {  // zero padding rows stay zero
                        float2 f = unpack2_tc<in_t>(xv[kg]);
                        if (p.ln_mode) {
                            const float lw = sLn[k], lb = sLn[kpad + k];
                            if (wb) {
                                f.x = fmaf((f.x - mu0) * rs0, lw, lb);
                                f.y = fmaf((f.y - mu1) * rs1, lw, lb);
                            } else {
                                f.x = f.x * rs0 * lw;
                                f.y = f.y * rs1 * lw;
                            }
                        }
                        if (p.gate_mode) {
                            const float gk = g[k];
                            if (p.gate_mode == 1) {
                                f.x = fmaf(f.x, gk, f.x);
                                f.y = fmaf(f.y, gk, f.y);
                            } else {
                                f.x += gk;
                                f.y += gk;
                            }
                        }
                        st[kg * 128] = pack2<in_t>(f.x, f.y);
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbar_arrive(&sh->ready[s]);
                if (tr && tid == 160 && it < 10) tr[4 + 6 * it + 1] = gtimer();
            }
        }
    } else {
        // ================= consumer warpgroup: wgmma + epilogue =================
        // one job = (tile, 64-channel block): its wgmmas, one commit group, wait, epilogue.  Descriptors advance by adding the byte offset >> 4 to the low word (start-address field; shared addresses
        // < 256 KB never carry out of it)
        const int nmb = (p.M + TC_MB - 1) / TC_MB;
        const int ksteps = kpad / 16;
        // K-major A: SBO = 128 B between 8-row groups, LBO = 16*128 B between the two 8-wide k groups of a k step
        const uint64_t a_desc0 = gmma_desc(smem_u32(sA), (TC_MT / 8) * 128, 128);
        // MN-major B: SBO = 128 B between 8-pixel groups, LBO = 4*128 B between the two 8-row k groups of a k step
        const uint64_t x_desc0 = gmma_desc(smem_u32(sX), (TC_PT / 8) * 128, 128);
        const in_t* __restrict__ resg = reinterpret_cast<const in_t*>(p.residual);
        in_t* __restrict__ og = reinterpret_cast<in_t*>(p.out);
        const int q = lane & 3, row0 = warp * 16 + (lane >> 2);  // accumulator rows row0, row0 + 8; pixel pairs 8j + 2q
        float acc0[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc0[i] = 0.f;

        mbar_wait(&sh->wfull, 0);
        if (tr && tid == 0) tr[2] = gtimer();
        auto issue = [&](int it, int mb, float* acc) {
            const int s = it % TC_NS;
            if (mb == 0) {
                mbar_wait(has_pro ? &sh->ready[s] : &sh->full[s], (it / TC_NS) & 1);
                if (tr && tid == 0 && it < 10) tr[4 + 6 * it + 2] = gtimer();
            }
            // weight tile mb/2, rows 64*(mb%2).. : 8 row groups further in the K-major layout
            uint64_t ad = a_desc0 + (uint64_t)(((mb >> 1) * TC_MT * kpad * 2 + (mb & 1) * 8 * 128) >> 4);
            uint64_t bd = x_desc0 + (uint64_t)((s * kpad * TC_PT * 2) >> 4);
            acc_fence(acc);
            wgmma_fence();
            wgmma_m64n32k16<in_t>(acc, ad, bd, 0u);
            for (int kk = 1; kk < ksteps; ++kk) {
                ad += (2 * (TC_MT / 8) * 128) >> 4;  // next 16 k of the weight tile
                bd += (2 * (TC_PT / 8) * 128) >> 4;
                wgmma_m64n32k16<in_t>(acc, ad, bd, 1u);
            }
            wgmma_commit();
            if (tr && tid == 0 && it < 10 && mb == nmb - 1) tr[4 + 6 * it + 3] = gtimer();
        };
        auto finish = [&](int it, int mb, float* acc) {  // job (it, mb) has completed
            acc_fence(acc);
            if (mb == nmb - 1) {
                if (lane == 0) mbar_arrive(&sh->empty[it % TC_NS]);  // the stage may be refilled
                if (tr && tid == 0 && it < 10) tr[4 + 6 * it + 4] = gtimer();
            }
            const int t = blockIdx.x + it * gridDim.x;
            const int b = t / ptiles, p0 = (t - b * ptiles) * TC_PT;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int mg = mb * TC_MB + row0 + 8 * h;
                const float bs = sBias[mg];
                const bool act = mg >= p.act_from && mg < p.act_to;
                // lane q holds pixels 8j + 2q, +1 (j = 0..3); after the quad transpose it holds pixels 8q .. 8q+7
                float2 v[4], rcv[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    v[j] = make_float2(acc[4 * j + 2 * h] + bs, acc[4 * j + 2 * h + 1] + bs);
                    if (act) v[j] = make_float2(silu_tc(v[j].x), silu_tc(v[j].y));
                }
                rcv[0] = sel4(v, q);
#pragma unroll
                for (int i = 1; i < 4; ++i) {
                    const float2 snd = sel4(v, q ^ i);
                    rcv[i] = make_float2(__shfl_xor_sync(0xffffffffu, snd.x, i), __shfl_xor_sync(0xffffffffu, snd.y, i));
                }
                float2 o[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) o[c] = sel4(rcv, c ^ q);  // pixels 8q + 2c, +1
                if (mg < p.M) {
                    if (resg) {
                        const uint4 r = __ldg(reinterpret_cast<const uint4*>(resg + (int64_t)b * p.r_bs + (int64_t)mg * p.r_cs + p0 + 8 * q));
                        const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const float2 f = unpack2_tc<in_t>(rw[c]);
                            o[c].x += f.x;
                            o[c].y += f.y;
                        }
                    }
                    *reinterpret_cast<uint4*>(og + (int64_t)b * p.o_bs + (int64_t)mg * p.o_cs + p0 + 8 * q) =
                        make_uint4(pack2<in_t>(o[0].x, o[0].y), pack2<in_t>(o[1].x, o[1].y), pack2<in_t>(o[2].x, o[2].y),
                                   pack2<in_t>(o[3].x, o[3].y));
                }
            }
            if (tr && tid == 0 && it < 10 && mb == nmb - 1) tr[4 + 6 * it + 5] = gtimer();
        };
        for (int it = 0; it < my_n; ++it)
            for (int mb = 0; mb < nmb; ++mb) {
                issue(it, mb, acc0);
                wgmma_wait<0>();
                finish(it, mb, acc0);
            }
    }
    __syncthreads();
    if (tr && threadIdx.x == 0) tr[3] = gtimer();
}

static size_t tc_smem_bytes(const PixlinParams& p) {
    const size_t kpad = (p.K + 15) / 16 * 16, nmt = (p.M + TC_MT - 1) / TC_MT;
    return nmt * TC_MT * kpad * 2 + (size_t)TC_NS * kpad * TC_PT * 2 + (2 * kpad + nmt * TC_MT) * sizeof(float) + sizeof(TcShared) + 128;
}

bool pixlin_tc_applicable(const PixlinParams& p, int dtype, int out_dtype) {
    // VMB_PIXLIN_TC: 0 (default) off, otherwise whenever legal (tests).  Off by default: on the H100 this kernel measured 1.2-1.9x
    // slower than the mma.sync kernel of pixlin.cu on every legal 1x1-conv shape of the bench nets (tools/pixlin_bench.py, B = 8
    // inference and B = 4 training, 64x64), and the bench step with it on every legal shape 10 % slower
    int mode = 0;
    if (const char* e = getenv("VMB_PIXLIN_TC")) mode = atoi(e);
    if (mode == 0) return false;
    return (dtype == VMB_BF16 || dtype == VMB_F16) && out_dtype == dtype && p.vec_ok && p.w_vec && p.P % TC_PT == 0 &&
           p.M <= TC_MAXMT * TC_MT && p.K <= 8 * TC_KGMAX && tc_smem_bytes(p) <= TC_SMEM_MAX;
}

int pixlin_tc_launch(const PixlinParams& p, int dtype, cudaStream_t stream) {
    const size_t smem = tc_smem_bytes(p);
    const long total = (long)(p.P / TC_PT) * p.B;
    // two CTAs per SM where their shared memory fits: twice the consumer warpgroups (epilogue latency) per SM
    const long ctas = (long)num_sms() * (2 * (smem + 1024) <= 228 * 1024 ? 2 : 1);
    const int grid = (int)(total < ctas ? total : ctas);
    const char* be = getenv("VMB_TC_BACKOFF");
    const int backoff = be ? atoi(be) : 100;
    const char* te = getenv("VMB_TC_TRACE");
    const int trace = te ? atoi(te) : 0;
    const int kg = (p.K + 7) / 8;
#define VMB_TC_GO(T, KGV)                                                                              \
    do {                                                                                               \
        auto k = pixlin_tc_kernel<T, KGV>;                                                             \
        VMB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));     \
        VMB_CUDA(launch_pdl(k, dim3(grid), dim3(TC_THREADS), smem, stream, p, trace, backoff));        \
    } while (0)
    if (dtype == VMB_BF16) {
        if (kg <= 8) VMB_TC_GO(__nv_bfloat16, 8);
        else if (kg <= 16) VMB_TC_GO(__nv_bfloat16, 16);
        else VMB_TC_GO(__nv_bfloat16, 32);
    } else {
        if (kg <= 8) VMB_TC_GO(__half, 8);
        else if (kg <= 16) VMB_TC_GO(__half, 16);
        else VMB_TC_GO(__half, 32);
    }
#undef VMB_TC_GO
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb

// debug only (not part of the public header): copy the trace stamps of the last traced pixlin launch to the host
extern "C" int vmb_debug_tc_trace(long long* dst, int n) {
    return cudaMemcpyFromSymbol(dst, vmb::g_tc_trace, sizeof(long long) * (size_t)n) == cudaSuccess ? 0 : 1;
}
