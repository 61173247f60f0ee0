// Selective-scan forward, TMA-staged variant (sm_90a) -- the fast path of vmb_selective_scan_fwd[_grouped].
// Replaces selective_scan_fwd_kernel (reference: Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan_fwd_kernel.cuh:61-172).
//
// Same recurrence mapping as scan_fwd.cu (lane = (row, segment of T positions), two register passes per state pair in packed
// f32x2, shuffle scan over the segments of a warp-chunk, chunk-to-chunk carry in the warp's smem), re-plumbed around it:
//   * operand tiles (u, delta rows of the CTA; the 16 B and 16 C state rows of the group) arrive as cp.async.bulk.tensor boxes
//     [rows x CHUNK] issued by ONE thread and tracked by an mbarrier -- no per-thread address arithmetic, bounds predicates or
//     LDGSTS issue slots (15 % of the round-1 kernel's instructions), tails and reversed-walk underflow zero-filled by the TMA unit;
//   * 8 warps per CTA share one fp32 B/C tile (16 rows of a group at RB=2): half the conversion work and smem per warp of the
//     round-1 4-warp CTA -> two 8-warp CTAs (16 warps) per SM at <= 128 registers;
//   * state split (SS): at small batch the 8 state pairs of a row are spread over SS warps (partial y summed through smem), so
//     384 rows (batch 1 at C=96) still fill 1 536 warps;
//   * packed-pair softplus: max(x,0) + log1p(exp(-|x|)) in f32x2, the lg2 MUFU skipped when every exp(-|x|) of the warp is small.
#include <stdlib.h>

#include <type_traits>

#include "scan_common.cuh"
#include "tma.cuh"
#include "scan_tma_common.cuh"

namespace vmb {

template <typename in_t, int RB, int NW, int SS>
struct TmaCfg {
    using Cfg = FwdCfg<RB>;
    static constexpr int CHUNK = Cfg::CHUNK, SLOTS = Cfg::SLOTS;
    static constexpr int ROWS = RB * (NW / SS);  // rows of one CTA
    static constexpr int NPW = 8 / SS;           // state pairs per warp
    static constexpr size_t io_bytes = sizeof(in_t) * (size_t)ROWS * CHUNK;  // one of rawU / rawD
    static constexpr size_t bc_bytes = sizeof(in_t) * (size_t)16 * CHUNK;    // one of rawB / rawC
    static constexpr size_t tile_bytes = sizeof(float4) * (size_t)16 * SLOTS;
    static constexpr size_t warp_bytes = sizeof(float) * 2 * RB * 16;
    static constexpr size_t ypart_bytes = SS > 1 ? sizeof(float) * (size_t)(NW / SS) * (SS - 1) * T * 32 : 0;
    static constexpr size_t smem_bytes = 2 * io_bytes + 2 * bc_bytes + tile_bytes + NW * warp_bytes + ypart_bytes + 16;
    static constexpr uint32_t tx_bytes = (uint32_t)(2 * io_bytes + 2 * bc_bytes);
};

// MODE 0: plain operator   1: plain + checkpoints (training forward)   2: per-group sources, reversed walk (fused OSS block)
//      3: per-group sources + checkpoints (cross_selective_scan forward; indexed by sequence position, like MODE 1 on gathered copies)
//      + kScanGate / kScanPairCkpt (scan_params.h) on MODE 0 / 1 with out_t = in_t: also out_z = out * SiLU(z); pair-layout
//        checkpoints (selective_scan_cuda)
// out_t: element type of `out`; float with 16-bit in_t (MODE 0 / 1 only) stores the fp32 accumulator without rounding
// (selective_scan_cuda_oflex, out_float=True)
template <typename in_t, int RB, int NW, int SS, int MODE, typename out_t>
__global__ void __launch_bounds__(32 * NW, NW == 8 ? 2 : 3)
    scan_fwd_tma_kernel(const ScanFwdParams p, const __grid_constant__ ScanTmaMaps maps) {
    pdl_trigger();
    pdl_wait();
    using K = TmaCfg<in_t, RB, NW, SS>;
    using Cfg = FwdCfg<RB>;
    constexpr int SEGW = Cfg::SEGW, CHUNK = Cfg::CHUNK, SEGQ = Cfg::SEGQ, SLOTS = Cfg::SLOTS;
    constexpr int V = Vec<in_t>::N, NT = 32 * NW, ROWS = K::ROWS, NPW = K::NPW;
    constexpr int VO = Vec<out_t>::N;
    constexpr int M = MODE & 3;  // base mode
    constexpr bool GATE = (MODE & kScanGate) != 0, PAIR = (MODE & kScanPairCkpt) != 0;

    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem_raw = smem_dyn + ((128u - (smem_addr(smem_dyn) & 127u)) & 127u);  // TMA destinations: 128 B aligned
    in_t* rawU = reinterpret_cast<in_t*>(smem_raw);                      // [ROWS][CHUNK]  TMA destinations (dense boxes)
    in_t* rawD = reinterpret_cast<in_t*>(smem_raw + K::io_bytes);
    in_t* rawB = reinterpret_cast<in_t*>(smem_raw + 2 * K::io_bytes);    // [16][CHUNK]
    in_t* rawC = reinterpret_cast<in_t*>(smem_raw + 2 * K::io_bytes + K::bc_bytes);
    float4* sB = reinterpret_cast<float4*>(smem_raw + 2 * K::io_bytes + 2 * K::bc_bytes);  // [8][SLOTS] CTA-shared fp32 pair tile
    float4* sC = sB + 8 * SLOTS;
    unsigned char* after_tile = reinterpret_cast<unsigned char*>(sC + 8 * SLOTS);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float* sCarry = reinterpret_cast<float*>(after_tile + warp * K::warp_bytes);  // [RB][16] chunk-to-chunk state of this warp's rows
    float* sA = sCarry + RB * 16;                                                 // [RB][16] A * log2(e)
    float* ypart = reinterpret_cast<float*>(after_tile + NW * K::warp_bytes);     // SS > 1: [row slot][SS-1][T][32]
    uint64_t* bar = reinterpret_cast<uint64_t*>(after_tile + NW * K::warp_bytes + K::ypart_bytes);

    const int rs = warp / SS, sp = warp % SS;  // row slot of the CTA, state part
    const int r = lane % RB, sl = lane / RB;
    const int ctas_per_batch = p.dim / ROWS;
    const int b = blockIdx.x / ctas_per_batch;
    const int dc0 = (blockIdx.x % ctas_per_batch) * ROWS;  // first row of the CTA
    const int g = dc0 / p.rows_per_group;                  // ROWS divides the group
    const int d0 = dc0 + rs * RB, d = d0 + r;
    const int N = p.N, L = p.L;

    out_t* orow;
    bool rev = false;
    int gi = 0, zbc = g, urow0 = dc0;
    if (M < 2) {
        orow = reinterpret_cast<out_t*>(p.out) + (int64_t)b * p.o_bs + (int64_t)d * p.o_ds;
    } else {
        const ScanGroupDesc& gd = p.grp[g];
        urow0 = dc0 - g * p.rows_per_group;
        orow = reinterpret_cast<out_t*>(gd.out) + (int64_t)b * p.o_bs + (int64_t)(urow0 + rs * RB + r) * p.o_ds;
        rev = gd.rev != 0;
        gi = g;
        zbc = 0;
    }

    auto issue = [&](int c0) {  // one thread: the four boxes of chunk c0 -> raw buffers, completion on `bar`
        const int m0 = rev ? L - c0 - CHUNK : c0;  // reversed walk: mirrored box, may start below 0 (zero-filled)
        mbarrier_expect_tx(bar, K::tx_bytes);
        tma_load_4d(rawU, &maps.u[gi], bar, m0, urow0, 0, b);
        tma_load_4d(rawD, &maps.d[gi], bar, m0, urow0, 0, b);
        tma_load_4d(rawB, &maps.b[gi], bar, m0, 0, zbc, b);
        tma_load_4d(rawC, &maps.c[gi], bar, m0, 0, zbc, b);
    };
    if (tid == 0) {
        mbarrier_init(bar, 1);
        mbarrier_init_fence();
        issue(0);
    }
    for (int i = lane; i < RB * 16; i += 32) {
        const int rr = i / 16, n = i % 16;
        sA[i] = n < N ? p.A[(int64_t)(d0 + rr) * N + n] * kLog2e : 0.f;
        sCarry[i] = 0.f;
    }
    const float Dval = (p.D && sp == 0) ? p.D[d] : 0.f;
    const float bias = p.bias ? p.bias[d] : 0.f;
    __syncthreads();  // barrier initialised before anyone polls it
    uint32_t phase = 0;
    for (int c0 = 0; c0 < L; c0 += CHUNK) {
        const int l0 = c0 + sl * T;
        const int valid = min(max(L - l0, 0), T);
        float uv[T], dt[T];
        mbarrier_wait(bar, phase);
        phase ^= 1;
        if (c0 > 0) __syncthreads();  // every warp is done with the previous fp32 tile
        convert_bc_dense<in_t, RB, NT>(sB, rawB, tid, M >= 2 && rev);
        convert_bc_dense<in_t, RB, NT>(sC, rawC, tid, M >= 2 && rev);
        {
            const in_t* ur = rawU + (rs * RB + r) * CHUNK;
            const in_t* dr = rawD + (rs * RB + r) * CHUNK;
            if (M < 2 || !rev) {
#pragma unroll
                for (int v = 0; v < T / V; ++v) {
                    load_vec_smem<in_t>(ur + sl * T + v * V, uv + v * V);
                    load_vec_smem<in_t>(dr + sl * T + v * V, dt + v * V);
                }
            } else {  // sequence position sl*T+t lives at raw index CHUNK-1-(sl*T+t)
#pragma unroll
                for (int v = 0; v < T / V; ++v) {
                    float tu[V], td[V];
                    load_vec_smem<in_t>(ur + CHUNK - (sl + 1) * T + v * V, tu);
                    load_vec_smem<in_t>(dr + CHUNK - (sl + 1) * T + v * V, td);
#pragma unroll
                    for (int i = 0; i < V; ++i) {
                        uv[T - 1 - (v * V + i)] = tu[i];
                        dt[T - 1 - (v * V + i)] = td[i];
                    }
                }
            }
        }
        __syncthreads();  // fp32 tile complete, raw buffers consumed -> refill them while this chunk computes
        if (tid == 0 && c0 + CHUNK < L) {
            fence_proxy_async();
            issue(c0 + CHUNK);
        }

        // ---- per-position prologue (packed pairs): dt = softplus(delta + bias), dtu = dt*u, y = D*u ----
        float sigma = 0.f;
        float dtu[T], y[T];
        if (p.softplus) {
            float e[T];
            float emax = 0.f;
#pragma unroll
            for (int t = 0; t < T; ++t) {
                dt[t] += bias;
                e[t] = ex2(-fabsf(dt[t]) * kLog2e);
                emax = fmaxf(emax, e[t]);
            }
            if (__all_sync(0xffffffffu, emax < 0.125f)) {  // typical model range (dt <~ 0.12): no second MUFU
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float2 lp = log1p_series2(make_float2(e[t], e[t + 1]));
                    dt[t] = fmaxf(dt[t], 0.f) + lp.x;
                    dt[t + 1] = fmaxf(dt[t + 1], 0.f) + lp.y;
                }
            } else {
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float2 ee = make_float2(e[t], e[t + 1]);
                    const float2 sm = log1p_series2(ee);
                    const float2 w = add2(ee, make_float2(1.f, 1.f));
                    const float2 bg = mul2(make_float2(lg2(w.x), lg2(w.y)), make_float2(kLn2, kLn2));
                    dt[t] = fmaxf(dt[t], 0.f) + (e[t] < 0.125f ? sm.x : bg.x);
                    dt[t + 1] = fmaxf(dt[t + 1], 0.f) + (e[t + 1] < 0.125f ? sm.y : bg.y);
                }
            }
        } else {
#pragma unroll
            for (int t = 0; t < T; ++t) dt[t] += bias;
        }
        if (valid < T) {  // identity element beyond the end: a = 1, b = 0
#pragma unroll
            for (int t = 0; t < T; ++t) dt[t] = t < valid ? dt[t] : 0.f;
        }
#pragma unroll
        for (int t = 0; t < T; t += 2) {
            const float2 d2 = make_float2(dt[t], dt[t + 1]), u2 = make_float2(uv[t], uv[t + 1]);
            const float2 du = mul2(d2, u2);
            const float2 y2 = mul2(u2, make_float2(Dval, Dval));
            dtu[t] = du.x; dtu[t + 1] = du.y;
            y[t] = y2.x; y[t + 1] = y2.y;
            sigma += dt[t] + dt[t + 1];
        }

        // ---- state-pair loop, software-pipelined: the MUFU-heavy pass 1 of pair np+1 (decay factors a = ex2(A dt), local end
        // state) runs inside the same unrolled position loop as the FMA-heavy pass 2 of pair np (true states, y += C h); each a2[t]
        // register is overwritten by the next pair's factor right after pass 2 consumed it, so no second array is live and
        // every warp's instruction stream mixes XU, FMA and LDS work instead of alternating between MUFU-only and FMA-only phases.
        float2 a2[T];
        float2 hend = make_float2(0.f, 0.f), P2;
        {
            const int np = sp * NPW;
            const float2 A2 = *reinterpret_cast<const float2*>(&sA[r * 16 + 2 * np]);
            const float4* __restrict__ bq = sB + np * SLOTS + sl * SEGQ;
#pragma unroll
            for (int t = 0; t < T; t += 2) {
                const float4 Bq = bq[t / 2];
                const float2 e0 = mul2(A2, make_float2(dt[t], dt[t]));
                const float2 e1 = mul2(A2, make_float2(dt[t + 1], dt[t + 1]));
                a2[t] = make_float2(ex2(e0.x), ex2(e0.y));
                a2[t + 1] = make_float2(ex2(e1.x), ex2(e1.y));
                hend = fma2(a2[t], hend, mul2(make_float2(dtu[t], dtu[t]), make_float2(Bq.x, Bq.y)));
                hend = fma2(a2[t + 1], hend, mul2(make_float2(dtu[t + 1], dtu[t + 1]), make_float2(Bq.z, Bq.w)));
            }
            P2 = mul2(A2, make_float2(sigma, sigma));
            P2 = make_float2(ex2(P2.x), ex2(P2.y));
        }
#pragma unroll 1
        for (int np = sp * NPW; np < (sp + 1) * NPW; ++np) {
            const int n0 = 2 * np;
            // ---- inclusive scan over the segments held by this warp (pair np) ----
#pragma unroll
            for (int o = RB; o < 32; o <<= 1) {
                const float2 Pp = shfl_up2(P2, o), Hp = shfl_up2(hend, o);
                if (lane >= o) {
                    hend = fma2(P2, Hp, hend);
                    P2 = mul2(P2, Pp);
                }
            }
            float2 Pe = shfl_up2(P2, RB % 32), He = shfl_up2(hend, RB % 32);
            if (lane < RB) {
                Pe = make_float2(1.f, 1.f);
                He = make_float2(0.f, 0.f);
            }
            float2* carry = reinterpret_cast<float2*>(&sCarry[r * 16 + n0]);
            const float2 st = *carry;  // chunk-start state (written by the last segment's lanes one chunk ago)
            float2 h = fma2(Pe, st, He);
            __syncwarp();
            if (sl == SEGW - 1) *carry = fma2(P2, st, hend);
            const float4* __restrict__ bq = sB + np * SLOTS + sl * SEGQ;
            const float4* __restrict__ cq = sC + np * SLOTS + sl * SEGQ;
            if (np + 1 < (sp + 1) * NPW) {
                // ---- pass 2 of pair np fused with pass 1 of pair np+1 ----
                const float2 A2n = *reinterpret_cast<const float2*>(&sA[r * 16 + n0 + 2]);
                const float4* __restrict__ bqn = bq + SLOTS;
                float2 hn = make_float2(0.f, 0.f);
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float4 Bq = bq[t / 2];
                    const float4 Cq = cq[t / 2];
                    const float4 Bn = bqn[t / 2];
                    const float2 du0 = make_float2(dtu[t], dtu[t]), du1 = make_float2(dtu[t + 1], dtu[t + 1]);
                    h = fma2(a2[t], h, mul2(du0, make_float2(Bq.x, Bq.y)));
                    y[t] = fmaf(h.y, Cq.y, fmaf(h.x, Cq.x, y[t]));
                    const float2 e0 = mul2(A2n, make_float2(dt[t], dt[t]));
                    a2[t] = make_float2(ex2(e0.x), ex2(e0.y));
                    hn = fma2(a2[t], hn, mul2(du0, make_float2(Bn.x, Bn.y)));
                    h = fma2(a2[t + 1], h, mul2(du1, make_float2(Bq.z, Bq.w)));
                    y[t + 1] = fmaf(h.y, Cq.w, fmaf(h.x, Cq.z, y[t + 1]));
                    const float2 e1 = mul2(A2n, make_float2(dt[t + 1], dt[t + 1]));
                    a2[t + 1] = make_float2(ex2(e1.x), ex2(e1.y));
                    hn = fma2(a2[t + 1], hn, mul2(du1, make_float2(Bn.z, Bn.w)));
                }
                hend = hn;
                P2 = mul2(A2n, make_float2(sigma, sigma));
                P2 = make_float2(ex2(P2.x), ex2(P2.y));
            } else {
                // ---- last pair of this warp: pass 2 only ----
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float4 Bq = bq[t / 2];
                    const float4 Cq = cq[t / 2];
                    h = fma2(a2[t], h, mul2(make_float2(dtu[t], dtu[t]), make_float2(Bq.x, Bq.y)));
                    y[t] = fmaf(h.y, Cq.y, fmaf(h.x, Cq.x, y[t]));
                    h = fma2(a2[t + 1], h, mul2(make_float2(dtu[t + 1], dtu[t + 1]), make_float2(Bq.z, Bq.w)));
                    y[t + 1] = fmaf(h.y, Cq.w, fmaf(h.x, Cq.z, y[t + 1]));
                }
            }
            if constexpr (PAIR) {
                store_ckpt_pair(p, b, d, l0, n0, h);
            } else if ((M == 1 || M == 3) && l0 < L && ((l0 + T) % kScanCkpt) == 0) {
                float* ck = p.ckpt + (((int64_t)b * p.dim + d) * p.n_ckpt + ((l0 + T) / kScanCkpt - 1)) * N + n0;
                if (n0 < N) ck[0] = h.x;
                if (n0 + 1 < N) ck[1] = h.y;
            }
        }

        if (SS > 1) {  // sum the partial outputs of the SS warps that share these rows (named barrier per row slot)
            float* yp = ypart + (size_t)rs * (SS - 1) * T * 32;
            if (sp > 0) {
#pragma unroll
                for (int t = 0; t < T; ++t) yp[((sp - 1) * T + t) * 32 + lane] = y[t];
            }
            asm volatile("bar.sync %0, %1;" ::"r"(1 + rs), "r"(32 * SS) : "memory");
            if (sp > 0) continue;
#pragma unroll
            for (int s = 0; s < SS - 1; ++s)
#pragma unroll
                for (int t = 0; t < T; ++t) y[t] += yp[(s * T + t) * 32 + lane];
        }
        if (M < 2 || !rev) {
#pragma unroll
            for (int v = 0; v < T / VO; ++v) store_vec<out_t>(orow + l0 + v * VO, y + v * VO, valid - v * VO, true);
            if constexpr (GATE) store_gated<in_t>(scan_gate_desc(p), b, d, l0, y, valid, true);
        } else if (valid == T) {  // sequence l0+t -> memory L-1-l0-t: one reversed contiguous block
#pragma unroll
            for (int v = 0; v < T / VO; ++v) {
                float yr[VO];
#pragma unroll
                for (int i = 0; i < VO; ++i) yr[i] = y[T - 1 - (v * VO + i)];
                store_vec<out_t>(orow + (L - l0 - T) + v * VO, yr, VO, true);
            }
        } else {
#pragma unroll
            for (int t = 0; t < T; ++t)
                if (t < valid) orow[L - 1 - l0 - t] = from_f32<out_t>(y[t]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            f = nullptr;
        return reinterpret_cast<EncodeTiledFn>(f);
    }();
    return fn;
}

int make_tmap_4d(CUtensorMap* map, int dtype, const void* base, const uint64_t dims[4], const int64_t strides_elts[3],
                 const uint32_t box[4], int swizzle) {
    EncodeTiledFn fn = encode_fn();
    VMB_CHECK(fn != nullptr, "cuTensorMapEncodeTiled not available from the CUDA driver");
    CUtensorMapDataType t;
    VMB_CHECK(dtype_to_tmap(dtype, &t) == VMB_OK, "tensor map: bad dtype %d", dtype);
    const uint64_t es = dtype == VMB_F32 ? 4 : 2;
    cuuint64_t gdim[4], gstr[3];
    cuuint32_t bx[4], estr[4] = {1, 1, 1, 1};
    for (int i = 0; i < 4; ++i) {
        gdim[i] = dims[i];
        bx[i] = box[i];
    }
    uint64_t dense = dims[0] * es;
    for (int i = 0; i < 3; ++i) {
        uint64_t s = (uint64_t)strides_elts[i] * es;
        if (dims[i + 1] == 1) s = (dense + 15) / 16 * 16;  // stride of an extent-1 dimension is never used: any legal value
        VMB_CHECK(s % 16 == 0 && s > 0, "tensor map: stride %d = %llu B is not a positive multiple of 16", i + 1, (unsigned long long)s);
        gstr[i] = s;
        dense = s * dims[i + 1];
    }
    const CUtensorMapSwizzle sw = swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_32B : swizzle == 2 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle == 3 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE;
    const CUresult r = fn(map, t, 4, const_cast<void*>(base), gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    VMB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return VMB_OK;
}

template <typename in_t, int RB, int NW, int SS, int MODE, typename out_t>
static int launch_tma4(const ScanFwdParams& p, const ScanTmaMaps& maps, cudaStream_t stream) {
    using K = TmaCfg<in_t, RB, NW, SS>;
    auto kern = scan_fwd_tma_kernel<in_t, RB, NW, SS, MODE, out_t>;
    constexpr size_t smem = K::smem_bytes + 128;  // + alignment slack
    static_assert(smem <= 227 * 1024, "scan_fwd_tma: shared memory");
    VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long blocks = (long)p.batch * (p.dim / K::ROWS);
    VMB_CUDA(launch_pdl(kern, dim3((unsigned)blocks), dim3(32 * NW), smem, stream, p, maps));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

template <typename in_t, int RB, int NW, int SS, typename out_t>
static int launch_tma3(const ScanFwdParams& p, const ScanTmaMaps& maps, int ext, cudaStream_t stream) {
    if constexpr (std::is_same<in_t, out_t>::value) {  // the grouped modes exist with the input's output type only
        if (p.ndesc) return p.ckpt ? launch_tma4<in_t, RB, NW, SS, 3, out_t>(p, maps, stream) : launch_tma4<in_t, RB, NW, SS, 2, out_t>(p, maps, stream);
    }
    VMB_CHECK(p.ndesc == 0, "selective_scan_fwd_grouped: no fp32 output");
    if (ext == 0)
        return p.ckpt ? launch_tma4<in_t, RB, NW, SS, 1, out_t>(p, maps, stream) : launch_tma4<in_t, RB, NW, SS, 0, out_t>(p, maps, stream);
    // gated / pair-checkpoint modes (input's output type only), instantiated after the plain ones so that those compile as before
    if constexpr (std::is_same<in_t, out_t>::value) {
        if (ext & kScanGate) {
            return p.ckpt ? launch_tma4<in_t, RB, NW, SS, 1 | kScanGate | kScanPairCkpt, out_t>(p, maps, stream)
                          : launch_tma4<in_t, RB, NW, SS, kScanGate, out_t>(p, maps, stream);
        }
        return launch_tma4<in_t, RB, NW, SS, 1 | kScanPairCkpt, out_t>(p, maps, stream);
    }
    set_error("selective_scan_fwd: no z gate / pair checkpoints with fp32 output");
    return VMB_ERR_INVALID;
}

// 4-warp CTAs, three resident per SM: 384 CTAs at (8, 384, 4096) spread 2-3 per SM (8-warp CTAs: 192 on 132 SMs, 1-2 per SM)
constexpr int kTmaWarps = 4;

template <typename in_t, int RB, typename out_t>
static int launch_tma2(const ScanFwdParams& p, const ScanTmaMaps& maps, int ss, int ext, cudaStream_t stream) {
    switch (ss) {
        case 4: return launch_tma3<in_t, RB, kTmaWarps, 4, out_t>(p, maps, ext, stream);
        case 2: return launch_tma3<in_t, RB, kTmaWarps, 2, out_t>(p, maps, ext, stream);
        default: return launch_tma3<in_t, RB, kTmaWarps, 1, out_t>(p, maps, ext, stream);
    }
}

template <typename in_t, typename out_t = in_t>
static int launch_tma1(const ScanFwdParams& p, const ScanTmaMaps& maps, int ss, int ext, cudaStream_t stream) {
    // rows per warp: 2 (scan_fwd_tma_pick; DESIGN §1.1: RB = 4 / 8 lose at every batch size, not instantiated)
    return launch_tma2<in_t, 2, out_t>(p, maps, ss, ext, stream);
}

// (rows per warp, state split) for the TMA kernel; false when the shape is left to the generic kernel.
bool scan_fwd_tma_pick(const ScanFwdParams& p, int& rb, int& ss) {
    if (!p.vec_ok || p.npad != 16 || p.L < 512) return false;
    if (p.ndesc && p.N != 16) return false;  // grouped sources: the B/C boxes are 16 rows of a wider tensor
    const int rpg = p.rows_per_group;
    const long rows = (long)p.batch * p.dim;
    const long want = 8L * num_sms();  // >= 2 warps per scheduler
    // rb = 2 at every batch size (DESIGN §1.1): with more rows per warp the B/C tile reads shrink but the warp count drops, and
    // the MUFU + LDS + SHFL instructions of a warp all queue on one path
    rb = 2;
    ss = 1;
    while (ss < 4 && rows / rb * ss < want) ss <<= 1;
    return rpg % (rb * kTmaWarps / ss) == 0;
}

int scan_fwd_tma_launch(const ScanFwdParams& p_in, int dtype, int rb, int ss, cudaStream_t stream, bool out_f32, int ext) {
    ScanFwdParams p = p_in;
    {
        p.num_sms = num_sms();
    }
    ScanTmaMaps maps;
    const uint32_t chunk = 32 / rb * T, rows = rb * kTmaWarps / ss;
    const uint32_t box_io[4] = {chunk, rows, 1, 1}, box_bc[4] = {chunk, 16, 1, 1};
    if (p.ndesc) {
        for (int g = 0; g < p.ndesc; ++g) {
            const uint64_t dio[4] = {(uint64_t)p.L, (uint64_t)p.rows_per_group, 1, (uint64_t)p.batch};
            const uint64_t dbc[4] = {(uint64_t)p.L, 16, 1, (uint64_t)p.batch};
            const int64_t su[3] = {p.u_ds, 0, p.u_bs}, sd[3] = {p.dl_ds, 0, p.dl_bs}, sb[3] = {p.B_ns, 0, p.B_bs}, sc[3] = {p.C_ns, 0, p.C_bs};
            int rc;
            if ((rc = make_tmap_4d(&maps.u[g], dtype, p.grp[g].u, dio, su, box_io)) != VMB_OK) return rc;
            if ((rc = make_tmap_4d(&maps.d[g], dtype, p.grp[g].delta, dio, sd, box_io)) != VMB_OK) return rc;
            if ((rc = make_tmap_4d(&maps.b[g], dtype, p.grp[g].Bm, dbc, sb, box_bc)) != VMB_OK) return rc;
            if ((rc = make_tmap_4d(&maps.c[g], dtype, p.grp[g].Cm, dbc, sc, box_bc)) != VMB_OK) return rc;
        }
    } else {
        const uint64_t dio[4] = {(uint64_t)p.L, (uint64_t)p.dim, 1, (uint64_t)p.batch};
        const uint64_t dbc[4] = {(uint64_t)p.L, (uint64_t)p.N, (uint64_t)p.G, (uint64_t)p.batch};
        const int64_t su[3] = {p.u_ds, 0, p.u_bs}, sd[3] = {p.dl_ds, 0, p.dl_bs}, sb[3] = {p.B_ns, p.B_gs, p.B_bs}, sc[3] = {p.C_ns, p.C_gs, p.C_bs};
        int rc;
        if ((rc = make_tmap_4d(&maps.u[0], dtype, p.u, dio, su, box_io)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.d[0], dtype, p.delta, dio, sd, box_io)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.b[0], dtype, p.Bm, dbc, sb, box_bc)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.c[0], dtype, p.Cm, dbc, sc, box_bc)) != VMB_OK) return rc;
    }
    if (out_f32) {  // fp32 `out` from 16-bit inputs
        switch (dtype) {
            case VMB_BF16: return launch_tma1<__nv_bfloat16, float>(p, maps, ss, ext, stream);
            case VMB_F16: return launch_tma1<__half, float>(p, maps, ss, ext, stream);
        }
        set_error("selective_scan_fwd: fp32 output needs bf16 / fp16 inputs (dtype %d)", dtype);
        return VMB_ERR_INVALID;
    }
    switch (dtype) {
        case VMB_F32: return launch_tma1<float>(p, maps, ss, ext, stream);
        case VMB_BF16: return launch_tma1<__nv_bfloat16>(p, maps, ss, ext, stream);
        case VMB_F16: return launch_tma1<__half>(p, maps, ss, ext, stream);
    }
    set_error("selective_scan_fwd: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

}  // namespace vmb
