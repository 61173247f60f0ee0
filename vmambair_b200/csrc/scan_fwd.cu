// Selective-scan forward for sm_90a -- replaces selective_scan_fwd_kernel
// (reference: Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan_fwd_kernel.cuh:61-172).
//
// Design (not a port of the CUB block-scan kernel):
//   * one WARP owns RB rows (channels d of one (batch, group)) and walks the sequence in chunks of
//     (32/RB) segments x T=16 positions; lane -> (row = lane % RB, segment = lane / RB).  The WPC warps
//     of a CTA own different rows of the SAME group and share one staged B/C tile; they only meet at
//     the two barriers around tile staging, never inside the state loop.
//   * B/C for the group are staged once per chunk in shared memory as fp32 and read by
//     BROADCAST (all rows of a warp read the same (n,l) word), so smem bandwidth is 1/RB of a
//     row-per-warp design and L2 traffic for B/C is 1/RB of the reference's row-per-CTA design.
//   * u/delta/out go straight between HBM and registers in full 32 B sectors (16 bf16 per lane).
//   * two passes per state pair, both states packed in one fma.rn.f32x2:
//       pass 1: a = ex2(A*log2e*dt) (MUFU), local end state with zero start;
//       segment scan: shuffles inside the warp; the chunk-to-chunk carry lives in the warp's smem;
//       pass 2: h = a*h + b from the true start state, y += h*C.
//     The decay of a whole segment is ex2(A * sum(dt)) -- one MUFU, no product chain.
//   * checkpoints of h every CKPT positions (fp32) feed the backward kernel.
#include <stdlib.h>

#include <type_traits>

#include "scan_common.cuh"

namespace vmb {

// ---- cooperative (whole CTA) staging -------------------------------------------------------------
template <typename in_t, int RB>
struct FwdRaw {
    static constexpr int V = Vec<in_t>::N;
    static constexpr int CHUNK = FwdCfg<RB>::CHUNK;
    static constexpr int PITCH = CHUNK + V;  // +16 B: conflict-free row-strided 128-bit reads
    static constexpr int OPR = CHUNK / V;    // 16-byte ops per row (power of two)
    static constexpr size_t bc_bytes = sizeof(in_t) * (size_t)32 * PITCH;
    static constexpr size_t io_bytes = sizeof(in_t) * (size_t)2 * RB * PITCH;
};

// rows [0,16) = B states, [16,32) = C states of the first state tile, positions [c0, c0+CHUNK)
// m0 = memory index of the chunk's first raw element: c0 (forward) or L - c0 - CHUNK (reversed walk, may be < 0)
template <typename in_t, int RB, int NT>
__device__ __forceinline__ void prefetch_bc_cta(in_t* __restrict__ raw, const in_t* __restrict__ Bg, const in_t* __restrict__ Cg,
                                                int64_t B_ns, int64_t C_ns, int N, int m0, int L, int tid) {
    using R = FwdRaw<in_t, RB>;
    const bool full = m0 >= 0 && m0 + R::CHUNK <= L;
#pragma unroll
    for (int it = tid; it < 32 * R::OPR; it += NT) {
        const int row = it / R::OPR, l = (it % R::OPR) * R::V;
        const int n = row & 15;
        const in_t* src = (row < 16 ? Bg + (int64_t)n * B_ns : Cg + (int64_t)n * C_ns) + m0 + l;
        int nbytes = 16;
        if (!full) nbytes = (m0 + l < 0) ? 0 : min(max((L - (m0 + l)) * (int)sizeof(in_t), 0), 16);
        if (n >= N) nbytes = 0;
        cp_async16(raw + row * R::PITCH + l, nbytes > 0 ? (const void*)src : (const void*)Bg, nbytes);
    }
}
// the warp's own rows: [0,RB) = u, [RB,2RB) = delta
template <typename in_t, int RB>
__device__ __forceinline__ void prefetch_io_warp(in_t* __restrict__ raw, const in_t* __restrict__ ublk, const in_t* __restrict__ dblk,
                                                 int64_t u_ds, int64_t dl_ds, int m0, int L, int lane) {
    using R = FwdRaw<in_t, RB>;
    const bool full = m0 >= 0 && m0 + R::CHUNK <= L;
#pragma unroll
    for (int it = lane; it < 2 * RB * R::OPR; it += 32) {
        const int row = it / R::OPR, l = (it % R::OPR) * R::V;
        const in_t* src = (row < RB ? ublk + (int64_t)row * u_ds : dblk + (int64_t)(row - RB) * dl_ds) + m0 + l;
        int nbytes = 16;
        if (!full) nbytes = (m0 + l < 0) ? 0 : min(max((L - (m0 + l)) * (int)sizeof(in_t), 0), 16);
        cp_async16(raw + row * R::PITCH + l, nbytes > 0 ? (const void*)src : (const void*)ublk, nbytes);
    }
}
// raw B or C rows -> fp32 float4 layout used by the passes (whole CTA)
template <typename in_t, int RB, int NT>
__device__ __forceinline__ void convert_bc_cta(float4* __restrict__ dst, const in_t* __restrict__ rawX, int tid, bool rev) {
    using R = FwdRaw<in_t, RB>;
    using Cfg = FwdCfg<RB>;
    constexpr int V = R::V, LG = R::CHUNK / V;
#pragma unroll
    for (int it = tid; it < 8 * LG; it += NT) {
        const int np = it / LG, l = (it % LG) * V;
        float f0[V], f1[V];
        load_vec_smem<in_t>(rawX + (2 * np) * R::PITCH + l, f0);
        load_vec_smem<in_t>(rawX + (2 * np + 1) * R::PITCH + l, f1);
        if (!rev) {
            float4* d = dst + np * Cfg::SLOTS + (l / T) * Cfg::SEGQ + (l % T) / 2;
#pragma unroll
            for (int i = 0; i < V / 2; ++i) d[i] = make_float4(f0[2 * i], f1[2 * i], f0[2 * i + 1], f1[2 * i + 1]);
        } else {
            // raw index i <-> sequence position CHUNK-1-i: the V raw elements are V descending positions
            const int s_hi = R::CHUNK - 1 - l;  // sequence position of raw element l (odd)
#pragma unroll
            for (int j = 0; j < V / 2; ++j) {
                const int s = s_hi - 1 - 2 * j;  // even position of the pair (s, s+1) <- raw (l+2j+1, l+2j)
                dst[np * Cfg::SLOTS + (s / T) * Cfg::SEGQ + (s % T) / 2] = make_float4(f0[2 * j + 1], f1[2 * j + 1], f0[2 * j], f1[2 * j]);
            }
        }
    }
}
// synchronous fallback (unaligned tensors, state tiles beyond the first), whole CTA
template <typename in_t, int RB, int NT>
__device__ __forceinline__ void stage_bc_cta(float4* __restrict__ dst, const in_t* __restrict__ src, int64_t n_stride, int n0,
                                             int N, int c0, int L, bool vec_ok, int tid) {
    using Cfg = FwdCfg<RB>;
    constexpr int V = Vec<in_t>::N;
    constexpr int LG = Cfg::CHUNK / V;
    for (int it = tid; it < 8 * LG; it += NT) {
        const int np = it / LG, l = (it % LG) * V;
        const int n = n0 + 2 * np;
        float f0[V], f1[V];
        const int valid = L - (c0 + l);
#pragma unroll
        for (int i = 0; i < V; ++i) f0[i] = f1[i] = 0.f;
        if (n < N) load_vec<in_t>(src + (int64_t)n * n_stride + c0 + l, f0, valid, vec_ok);
        if (n + 1 < N) load_vec<in_t>(src + (int64_t)(n + 1) * n_stride + c0 + l, f1, valid, vec_ok);
        float4* d = dst + np * Cfg::SLOTS + (l / T) * Cfg::SEGQ + (l % T) / 2;
#pragma unroll
        for (int i = 0; i < V / 2; ++i) d[i] = make_float4(f0[2 * i], f1[2 * i], f0[2 * i + 1], f1[2 * i + 1]);
    }
}

// MODE 0: plain operator, no checkpoints (inference)   1: plain operator + checkpoints (training forward)
//      2: direction-aware grouped sources (per-group bases, reversed walk), no checkpoints   3: 2 + checkpoints.
// Each mode only compiles what it needs: the state loop sits at the 128-register limit.
//      + kScanGate / kScanPairCkpt (scan_params.h) on MODE 0 / 1 with out_t = in_t: also out_z = out * SiLU(z); pair-layout
//        checkpoints (selective_scan_cuda).
// out_t: element type of `out` (float with 16-bit in_t, MODE 0 / 1 only: the fp32 accumulator stored without rounding).
template <typename in_t, int RB, int WPC, int MODE, typename out_t>
__global__ void __launch_bounds__(32 * WPC, 12 / WPC) scan_fwd_kernel(const ScanFwdParams p) {
    pdl_trigger();
    pdl_wait();
    using Cfg = FwdCfg<RB>;
    using R = FwdRaw<in_t, RB>;
    constexpr int SEGW = Cfg::SEGW, CHUNK = Cfg::CHUNK, SEGQ = Cfg::SEGQ, SLOTS = Cfg::SLOTS;
    constexpr int V = Vec<in_t>::N, NT = 32 * WPC;
    constexpr int VO = Vec<out_t>::N;
    constexpr int M = MODE & 3;  // base mode
    constexpr bool GATE = (MODE & kScanGate) != 0, PAIR = (MODE & kScanPairCkpt) != 0;

    extern __shared__ float4 smem_f4[];
    float4* sB = smem_f4;                                                  // [8][SLOTS]   CTA-shared
    float4* sC = sB + 8 * SLOTS;                                           // [8][SLOTS]
    in_t* rawBC = reinterpret_cast<in_t*>(sC + 8 * SLOTS);                 // [32][PITCH]
    char* warp_base = reinterpret_cast<char*>(rawBC) + R::bc_bytes;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const size_t per_warp = R::io_bytes + sizeof(float) * 2 * RB * p.npad;
    in_t* raw = reinterpret_cast<in_t*>(warp_base + warp * per_warp);      // [2RB][PITCH] this warp's u / delta rows
    float* sCarry = reinterpret_cast<float*>(reinterpret_cast<char*>(raw) + R::io_bytes);  // [RB][npad]
    float* sA = sCarry + RB * p.npad;                                      // [RB][npad]  A * log2(e)

    const int r = lane % RB, sl = lane / RB;
    const int ctas_per_batch = p.dim / (RB * WPC);
    const int b = blockIdx.x / ctas_per_batch;
    const int d0 = ((blockIdx.x % ctas_per_batch) * WPC + warp) * RB, d = d0 + r;
    const int g = d0 / p.rows_per_group;  // same for every warp of the CTA (RB*WPC divides the group)
    const int N = p.N, L = p.L, npad = p.npad;
    const bool async_ok = p.vec_ok;
    constexpr bool HAS_REV = M >= 2;

    const in_t *Bg, *Cg, *ublk, *dblk;
    out_t* orow;
    bool rev = false;
    if (M < 2) {
        Bg = reinterpret_cast<const in_t*>(p.Bm) + (int64_t)b * p.B_bs + (int64_t)g * p.B_gs;
        Cg = reinterpret_cast<const in_t*>(p.Cm) + (int64_t)b * p.C_bs + (int64_t)g * p.C_gs;
        ublk = reinterpret_cast<const in_t*>(p.u) + (int64_t)b * p.u_bs + (int64_t)d0 * p.u_ds;
        dblk = reinterpret_cast<const in_t*>(p.delta) + (int64_t)b * p.dl_bs + (int64_t)d0 * p.dl_ds;
        orow = reinterpret_cast<out_t*>(p.out) + (int64_t)b * p.o_bs + (int64_t)d * p.o_ds;
    } else {  // per-group sources; rows are indexed inside the group
        const ScanGroupDesc& gd = p.grp[g];
        const int dg0 = d0 - g * p.rows_per_group;
        Bg = reinterpret_cast<const in_t*>(gd.Bm) + (int64_t)b * p.B_bs;
        Cg = reinterpret_cast<const in_t*>(gd.Cm) + (int64_t)b * p.C_bs;
        ublk = reinterpret_cast<const in_t*>(gd.u) + (int64_t)b * p.u_bs + (int64_t)dg0 * p.u_ds;
        dblk = reinterpret_cast<const in_t*>(gd.delta) + (int64_t)b * p.dl_bs + (int64_t)dg0 * p.dl_ds;
        orow = reinterpret_cast<out_t*>(gd.out) + (int64_t)b * p.o_bs + (int64_t)(dg0 + r) * p.o_ds;
        if constexpr (HAS_REV) rev = gd.rev != 0;
    }
    const in_t* __restrict__ urow = ublk + (int64_t)r * p.u_ds;
    const in_t* __restrict__ drow = dblk + (int64_t)r * p.dl_ds;

    if (async_ok) {
        const int m0 = rev ? L - CHUNK : 0;
        prefetch_bc_cta<in_t, RB, NT>(rawBC, Bg, Cg, p.B_ns, p.C_ns, N, m0, L, tid);
        prefetch_io_warp<in_t, RB>(raw, ublk, dblk, p.u_ds, p.dl_ds, m0, L, lane);
        cp_async_commit();
    }
    for (int i = lane; i < RB * npad; i += 32) {
        const int rr = i / npad, n = i % npad;
        sA[i] = n < N ? p.A[(int64_t)(d0 + rr) * N + n] * kLog2e : 0.f;
        sCarry[i] = 0.f;
    }
    const float Dval = p.D ? p.D[d] : 0.f;
    const float bias = p.bias ? p.bias[d] : 0.f;
    const int ntiles = npad / 16;

    for (int c0 = 0; c0 < L; c0 += CHUNK) {
        const int l0 = c0 + sl * T;
        const int valid = min(max(L - l0, 0), T);
        float uv[T], dt[T];
        if (async_ok) {
            cp_async_wait_all();
            __syncthreads();  // every copy has landed; every warp is done with the previous B/C tile
            convert_bc_cta<in_t, RB, NT>(sB, rawBC, tid, HAS_REV && rev);
            convert_bc_cta<in_t, RB, NT>(sC, rawBC + 16 * R::PITCH, tid, HAS_REV && rev);
            if (!HAS_REV || !rev) {
#pragma unroll
                for (int v = 0; v < T / V; ++v) {
                    load_vec_smem<in_t>(raw + r * R::PITCH + sl * T + v * V, uv + v * V);
                    load_vec_smem<in_t>(raw + (RB + r) * R::PITCH + sl * T + v * V, dt + v * V);
                }
            } else {  // sequence positions sl*T+t live at raw index CHUNK-1-(sl*T+t): load each vector, place it mirrored
#pragma unroll
                for (int v = 0; v < T / V; ++v) {
                    float tu[V], td[V];
                    load_vec_smem<in_t>(raw + r * R::PITCH + CHUNK - (sl + 1) * T + v * V, tu);
                    load_vec_smem<in_t>(raw + (RB + r) * R::PITCH + CHUNK - (sl + 1) * T + v * V, td);
#pragma unroll
                    for (int i = 0; i < V; ++i) {
                        uv[T - 1 - (v * V + i)] = tu[i];
                        dt[T - 1 - (v * V + i)] = td[i];
                    }
                }
            }
            __syncthreads();  // fp32 tile complete, raw buffers free -> refill them while we compute
            if (c0 + CHUNK < L) {
                const int m0 = rev ? L - c0 - 2 * CHUNK : c0 + CHUNK;
                prefetch_bc_cta<in_t, RB, NT>(rawBC, Bg, Cg, p.B_ns, p.C_ns, N, m0, L, tid);
                prefetch_io_warp<in_t, RB>(raw, ublk, dblk, p.u_ds, p.dl_ds, m0, L, lane);
                cp_async_commit();
            }
        } else {
#pragma unroll
            for (int v = 0; v < T / V; ++v) {
                load_vec<in_t>(urow + l0 + v * V, uv + v * V, valid - v * V, false);
                load_vec<in_t>(drow + l0 + v * V, dt + v * V, valid - v * V, false);
            }
        }
        float sigma = 0.f;
        float dtu[T];
        float y[T];  // scalar accumulators (a packed pair per position would cost 16 more registers)
#pragma unroll
        for (int t = 0; t < T; ++t) {
            float x = dt[t] + bias;
            if (p.softplus) x = softplus_f(x);
            x = t < valid ? x : 0.f;  // identity element beyond the end: a=1, b=0
            dt[t] = x;
            dtu[t] = x * uv[t];
            sigma += x;
            y[t] = Dval * uv[t];
        }

        for (int nt = 0; nt < ntiles; ++nt) {
            if (!async_ok || nt > 0) {  // synchronous staging: unaligned tensors, or state tiles beyond the first
                __syncthreads();
                stage_bc_cta<in_t, RB, NT>(sB, Bg, p.B_ns, nt * 16, N, c0, L, p.vec_ok, tid);
                stage_bc_cta<in_t, RB, NT>(sC, Cg, p.C_ns, nt * 16, N, c0, L, p.vec_ok, tid);
                __syncthreads();
            }

#pragma unroll 1
            for (int np = 0; np < 8; ++np) {
                const int n0 = nt * 16 + 2 * np;
                const float2 A2 = *reinterpret_cast<const float2*>(&sA[r * npad + n0]);
                const float4* __restrict__ bq = sB + np * SLOTS + sl * SEGQ;
                const float4* __restrict__ cq = sC + np * SLOTS + sl * SEGQ;
                // ---- pass 1: decay factors + local end state ----
                float2 a2[T];
                float2 hend = make_float2(0.f, 0.f);
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float4 Bq = bq[t / 2];
                    float2 e0 = mul2(A2, make_float2(dt[t], dt[t]));
                    float2 e1 = mul2(A2, make_float2(dt[t + 1], dt[t + 1]));
                    a2[t] = make_float2(ex2(e0.x), ex2(e0.y));
                    a2[t + 1] = make_float2(ex2(e1.x), ex2(e1.y));
                    hend = fma2(a2[t], hend, mul2(make_float2(dtu[t], dtu[t]), make_float2(Bq.x, Bq.y)));
                    hend = fma2(a2[t + 1], hend, mul2(make_float2(dtu[t + 1], dtu[t + 1]), make_float2(Bq.z, Bq.w)));
                }
                float2 P2 = mul2(A2, make_float2(sigma, sigma));
                P2 = make_float2(ex2(P2.x), ex2(P2.y));
                // ---- inclusive scan over the segments held by this warp ----
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
                float2* carry = reinterpret_cast<float2*>(&sCarry[r * npad + n0]);
                const float2 st = *carry;  // chunk-start state (written by the last segment's lanes one chunk ago)
                float2 h = fma2(Pe, st, He);
                __syncwarp();
                if (sl == SEGW - 1) *carry = fma2(P2, st, hend);
                // ---- pass 2: true states, output contraction ----
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float4 Bq = bq[t / 2];
                    const float4 Cq = cq[t / 2];
                    h = fma2(a2[t], h, mul2(make_float2(dtu[t], dtu[t]), make_float2(Bq.x, Bq.y)));
                    y[t] = fmaf(h.y, Cq.y, fmaf(h.x, Cq.x, y[t]));
                    h = fma2(a2[t + 1], h, mul2(make_float2(dtu[t + 1], dtu[t + 1]), make_float2(Bq.z, Bq.w)));
                    y[t + 1] = fmaf(h.y, Cq.w, fmaf(h.x, Cq.z, y[t + 1]));
                }
                if constexpr (PAIR) {
                    store_ckpt_pair(p, b, d, l0, n0, h);
                } else if ((M == 1 || M == 3) && l0 < L && ((l0 + T) % kScanCkpt) == 0) {
                    float* ck = p.ckpt + (((int64_t)b * p.dim + d) * p.n_ckpt + ((l0 + T) / kScanCkpt - 1)) * N + n0;
                    if (n0 < N) ck[0] = h.x;
                    if (n0 + 1 < N) ck[1] = h.y;
                }
            }
        }
        if (!HAS_REV || !rev) {
#pragma unroll
            for (int v = 0; v < T / VO; ++v) store_vec<out_t>(orow + l0 + v * VO, y + v * VO, valid - v * VO, p.vec_ok);
            if constexpr (GATE) store_gated<in_t>(scan_gate_desc(p), b, d, l0, y, valid, p.vec_ok);
        } else if (valid == T) {  // sequence l0+t -> memory L-1-l0-t: one reversed contiguous block
#pragma unroll
            for (int v = 0; v < T / VO; ++v) {
                float yr[VO];
#pragma unroll
                for (int i = 0; i < VO; ++i) yr[i] = y[T - 1 - (v * VO + i)];
                store_vec<out_t>(orow + (L - l0 - T) + v * VO, yr, VO, p.vec_ok);
            }
        } else {
#pragma unroll
            for (int t = 0; t < T; ++t)
                if (t < valid) orow[L - 1 - l0 - t] = from_f32<out_t>(y[t]);
        }
    }
}

template <typename in_t, int RB, int WPC, int MODE, typename out_t>
static int launch_cfg2(const ScanFwdParams& p, cudaStream_t stream) {
    using Cfg = FwdCfg<RB>;
    using R = FwdRaw<in_t, RB>;
    auto kern = scan_fwd_kernel<in_t, RB, WPC, MODE, out_t>;
    const size_t smem = sizeof(float4) * 16 * Cfg::SLOTS + R::bc_bytes + WPC * (R::io_bytes + sizeof(float) * 2 * RB * p.npad);
    VMB_CHECK(smem <= 227 * 1024, "selective_scan_fwd: dstate=%d needs %zu B of shared memory", p.N, smem);
    if (smem > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long blocks = (long)p.batch * (p.dim / (RB * WPC));
    VMB_CUDA(launch_pdl(kern, dim3((unsigned)blocks), dim3(32 * WPC), smem, stream, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

template <typename in_t, int RB, int WPC, typename out_t>
static int launch_cfg(const ScanFwdParams& p, int ext, cudaStream_t stream) {
    if constexpr (std::is_same<in_t, out_t>::value) {  // the grouped modes exist with the input's output type only
        if (p.ndesc) {
            if constexpr (RB <= 2) {
                if (p.ckpt) return launch_cfg2<in_t, RB, WPC, 3, out_t>(p, stream);
            }
            VMB_CHECK(p.ckpt == nullptr, "grouped scan: checkpoints need RB <= 2 (pick_cfg)");
            return launch_cfg2<in_t, RB, WPC, 2, out_t>(p, stream);
        }
    }
    VMB_CHECK(p.ndesc == 0, "grouped scan: no fp32 output");
    if (ext == 0) return p.ckpt ? launch_cfg2<in_t, RB, WPC, 1, out_t>(p, stream) : launch_cfg2<in_t, RB, WPC, 0, out_t>(p, stream);
    // gated / pair-checkpoint modes (input's output type only), instantiated after the plain ones so that those compile as before
    if constexpr (std::is_same<in_t, out_t>::value) {
        if (ext & kScanGate) {
            return p.ckpt ? launch_cfg2<in_t, RB, WPC, 1 | kScanGate | kScanPairCkpt, out_t>(p, stream)
                          : launch_cfg2<in_t, RB, WPC, kScanGate, out_t>(p, stream);
        }
        return launch_cfg2<in_t, RB, WPC, 1 | kScanPairCkpt, out_t>(p, stream);
    }
    set_error("selective_scan_fwd: no z gate / pair checkpoints with fp32 output");
    return VMB_ERR_INVALID;
}

// (rows per warp RB, warps per CTA WPC): RB*WPC must divide the rows of a group.  Small RB = more warps and
// longer chunks (more parallelism, more shuffle steps); the CTA shares one B/C tile, so WPC as large as fits.
static void pick_cfg(const ScanFwdParams& p, int& rb, int& wpc) {
    const int rpg = p.rows_per_group;
    const long rows = (long)p.batch * p.dim;
    // aim for >= ~1500 warps, then grow RB for cheaper scans (tools/scan_sustained.py sweeps RB per shape)
    rb = rows < 1536 ? 1 : rows < 8192 ? 2 : rows < 32768 ? 4 : 8;
    while (rb > 1 && rpg % rb) rb >>= 1;
    // short sequences: a warp-chunk should not be much longer than L
    while (rb < 8 && rpg % (rb * 2) == 0 && (32 / rb) * T >= 2 * p.L) rb *= 2;
    if (p.ndesc && p.ckpt && rb > 2) rb = 2;  // grouped + checkpoints (MODE 3) is instantiated at RB <= 2 only: RB 4 / 8 spill
    wpc = 4;
    while (wpc > 1 && (rpg % (rb * wpc) != 0)) wpc >>= 1;
}

template <typename in_t, int RB, typename out_t>
static int launch_rb(const ScanFwdParams& p, int wpc, int ext, cudaStream_t stream) {
    switch (wpc) {
        case 4: return launch_cfg<in_t, RB, 4, out_t>(p, ext, stream);
        case 2: return launch_cfg<in_t, RB, 2, out_t>(p, ext, stream);
        default: return launch_cfg<in_t, RB, 1, out_t>(p, ext, stream);
    }
}

template <typename in_t, typename out_t = in_t>
static int launch_t(const ScanFwdParams& p, int ext, cudaStream_t stream) {
    int rb, wpc;
    pick_cfg(p, rb, wpc);
    switch (rb) {
        case 8: return launch_rb<in_t, 8, out_t>(p, wpc, ext, stream);
        case 4: return launch_rb<in_t, 4, out_t>(p, wpc, ext, stream);
        case 2: return launch_rb<in_t, 2, out_t>(p, wpc, ext, stream);
        default: return launch_rb<in_t, 1, out_t>(p, wpc, ext, stream);
    }
}

int scan_fwd_launch(const ScanFwdParams& p, int dtype, cudaStream_t stream, bool out_f32, int ext) {
    VMB_CHECK((long)p.batch * p.dim < (1L << 31), "selective_scan_fwd: batch*dim too large");
    VMB_CHECK(!out_f32 || (p.ndesc == 0 && (dtype == VMB_BF16 || dtype == VMB_F16)),
              "selective_scan_fwd: fp32 output needs bf16 / fp16 inputs and the flat operator");
    VMB_CHECK(ext == 0 || (p.ndesc == 0 && !out_f32), "selective_scan_fwd: the z gate exists for the flat operator without fp32 output");
    VMB_CHECK(!(ext & kScanPairCkpt) || p.ckpt, "selective_scan_fwd: pair-layout checkpoints without a checkpoint buffer");
    {  // fast path: TMA-staged kernel (scan_fwd_tma.cu); this file keeps the generic shapes (unaligned rows, dstate > 16, short L)
        int rb, ss;
        if (scan_fwd_tma_pick(p, rb, ss)) return scan_fwd_tma_launch(p, dtype, rb, ss, stream, out_f32, ext);
    }
    if (p.ndesc) {
        VMB_CHECK(p.vec_ok && p.npad == 16, "grouped scan: needs 16 B-aligned rows (L %% 8 == 0) and dstate <= 16");
    }
    if (out_f32) return dtype == VMB_BF16 ? launch_t<__nv_bfloat16, float>(p, ext, stream) : launch_t<__half, float>(p, ext, stream);
    switch (dtype) {
        case VMB_F32: return launch_t<float>(p, ext, stream);
        case VMB_BF16: return launch_t<__nv_bfloat16>(p, ext, stream);
        case VMB_F16: return launch_t<__half>(p, ext, stream);
    }
    set_error("selective_scan_fwd: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

}  // namespace vmb
