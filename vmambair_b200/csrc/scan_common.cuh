// Pieces shared by the forward and backward selective-scan kernels (warp-autonomous design).
#pragma once
#include "common.cuh"
#include "scan_params.h"

namespace vmb {

constexpr int T = kScanT;  // positions per lane per chunk

// One WARP is an autonomous unit: RB rows (channels of one (batch, group)) x SEGW = 32/RB
// consecutive segments of T positions -> a warp-chunk of SEGW*T positions.  No block barriers:
// warps de-synchronise, so MUFU-heavy pass 1 of one warp overlaps FMA-heavy pass 2 of another.
template <int RB>
struct FwdCfg {
    static constexpr int SEGW = 32 / RB;
    static constexpr int CHUNK = SEGW * T;
    static constexpr int SEGQ = T / 2 + 1;  // float4 slots per segment (one pad slot: conflict-free broadcast)
    static constexpr int SLOTS = SEGW * SEGQ;
    static size_t smem_bytes(int npad) { return sizeof(float4) * (2 * 8 * SLOTS) + sizeof(float) * (2 * RB * npad); }
};

// Stage B or C rows [n0, n0+16) x [c0, c0+CHUNK) of one (batch, group) into the warp's smem as
// float4 = (X[n][l], X[n+1][l], X[n][l+1], X[n+1][l+1]) at [n/2][seg*SEGQ + (l%T)/2].
template <typename in_t, typename Cfg>
__device__ __forceinline__ void stage_bc(float4* __restrict__ dst, const in_t* __restrict__ src, int64_t n_stride,
                                         int n0, int N, int c0, int L, bool vec_ok, int lane) {
    constexpr int V = Vec<in_t>::N;
    constexpr int LG = Cfg::CHUNK / V;  // l-groups per row
#pragma unroll
    for (int it = lane; it < 8 * LG; it += 32) {
        const int np = it / LG, lg = it % LG;
        const int l = lg * V;  // offset inside chunk
        const int n = n0 + 2 * np;
        float f0[V], f1[V];
        const int valid = L - (c0 + l);
        if (n < N) load_vec<in_t>(src + (int64_t)n * n_stride + c0 + l, f0, valid, vec_ok);
        else {
#pragma unroll
            for (int i = 0; i < V; ++i) f0[i] = 0.f;
        }
        if (n + 1 < N) load_vec<in_t>(src + (int64_t)(n + 1) * n_stride + c0 + l, f1, valid, vec_ok);
        else {
#pragma unroll
            for (int i = 0; i < V; ++i) f1[i] = 0.f;
        }
        const int seg = l / T, tq = (l % T) / 2;
        float4* d = dst + np * Cfg::SLOTS + seg * Cfg::SEGQ + tq;
#pragma unroll
        for (int i = 0; i < V / 2; ++i) d[i] = make_float4(f0[2 * i], f1[2 * i], f0[2 * i + 1], f1[2 * i + 1]);
    }
}

// cp.async (LDGSTS) 16-byte copy, zero-filling bytes beyond src_bytes.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Raw (input dtype) staging buffer of one warp-chunk, filled asynchronously one chunk ahead:
// rows [0,RB) = u, [RB,2RB) = delta, ([2RB,3RB) = dout when NIO==3), then 16 rows of B (states 0..15)
// and 16 rows of C.
template <typename in_t, int RB, int NIO = 2>
struct RawCfg {
    static constexpr int V = Vec<in_t>::N;
    static constexpr int CHUNK = FwdCfg<RB>::CHUNK;
    static constexpr int PITCH = CHUNK + V;  // +16 B: conflict-free row-strided 128-bit reads
    static constexpr int ROWS = NIO * RB + 32;
    static constexpr size_t bytes = sizeof(in_t) * (size_t)ROWS * PITCH;
};

template <typename in_t, int RB, int NIO>
__device__ __forceinline__ void prefetch_chunk(in_t* __restrict__ raw, const in_t* const* __restrict__ io_base,
                                               const int64_t* __restrict__ io_ds, const in_t* __restrict__ Bg,
                                               const in_t* __restrict__ Cg, int64_t B_ns, int64_t C_ns, int N, int c0,
                                               int L, int lane) {
    using R = RawCfg<in_t, RB, NIO>;
    constexpr int V = R::V, OPR = R::CHUNK / V;  // 16-byte ops per row
#pragma unroll
    for (int it = lane; it < R::ROWS * OPR; it += 32) {
        const int row = it / OPR, l = (it % OPR) * V;
        const in_t* src;
        bool row_ok = true;
        if (row < NIO * RB) {
            const int k = row / RB;
            src = io_base[k] + (int64_t)(row - k * RB) * io_ds[k];
        } else if (row < NIO * RB + 16) {
            src = Bg + (int64_t)(row - NIO * RB) * B_ns;
            row_ok = (row - NIO * RB) < N;
        } else {
            src = Cg + (int64_t)(row - NIO * RB - 16) * C_ns;
            row_ok = (row - NIO * RB - 16) < N;
        }
        int nbytes = (L - (c0 + l)) * (int)sizeof(in_t);
        nbytes = row_ok ? min(max(nbytes, 0), 16) : 0;
        cp_async16(raw + row * R::PITCH + l, nbytes > 0 ? (const void*)(src + c0 + l) : (const void*)io_base[0], nbytes);
    }
    cp_async_commit();
}

// raw B/C rows (states 0..15 of this chunk) -> fp32 float4 layout used by the passes
template <typename in_t, int RB, int NIO>
__device__ __forceinline__ void convert_bc(float4* __restrict__ dst, const in_t* __restrict__ rawX, int lane) {
    using R = RawCfg<in_t, RB, NIO>;
    using Cfg = FwdCfg<RB>;
    constexpr int V = R::V, LG = R::CHUNK / V;
#pragma unroll
    for (int it = lane; it < 8 * LG; it += 32) {
        const int np = it / LG, l = (it % LG) * V;
        float f0[V], f1[V];
        load_vec_smem<in_t>(rawX + (2 * np) * R::PITCH + l, f0);
        load_vec_smem<in_t>(rawX + (2 * np + 1) * R::PITCH + l, f1);
        float4* d = dst + np * Cfg::SLOTS + (l / T) * Cfg::SEGQ + (l % T) / 2;
#pragma unroll
        for (int i = 0; i < V / 2; ++i) d[i] = make_float4(f0[2 * i], f1[2 * i], f0[2 * i + 1], f1[2 * i + 1]);
    }
}
// z * sigmoid(z): the gate of the z-gated forward and of its backward (one expression, so a recomputed out_z equals the forward's
// when `out` is fp32)
__device__ __forceinline__ float silu_gate(float z) { return z / (1.f + __expf(-z)); }

// out_z at positions [l0, l0+T) of row (b, d): y (the fp32 accumulator, already summed over state parts) * SiLU(z), rounded once
template <typename in_t>
__device__ __forceinline__ void store_gated(const ScanGateDesc& gt, int b, int d, int l0, const float* y, int valid, bool vec_ok) {
    constexpr int V = Vec<in_t>::N;
    const in_t* zr = reinterpret_cast<const in_t*>(gt.z) + (int64_t)b * gt.z_bs + (int64_t)d * gt.z_ds + l0;
    in_t* ozr = reinterpret_cast<in_t*>(gt.out_z) + (int64_t)b * gt.oz_bs + (int64_t)d * gt.oz_ds + l0;
#pragma unroll
    for (int v = 0; v < T / V; ++v) {
        float zv[V];
        load_vec<in_t>(zr + v * V, zv, valid - v * V, vec_ok);
#pragma unroll
        for (int i = 0; i < V; ++i) zv[i] = y[v * V + i] * silu_gate(zv[i]);
        store_vec<in_t>(ozr + v * V, zv, valid - v * V, vec_ok);
    }
}

// pair-layout checkpoint (kScanPairCkpt): states n0, n0+1 after the last position of the lane's segment, written by the segment
// that ends a 64-position interval or holds position L-1 (so row n_ckpt-1 is the last state for every L); row k, slots 2n / 2n+1 =
// (0, h_n).  The base is 16 B aligned (vmb_selective_scan_fwd checks it), so with even N every pair is one 16 B store.
__device__ __forceinline__ void store_ckpt_pair(const ScanFwdParams& p, int b, int d, int l0, int n0, float2 h) {
    if (l0 >= p.L || ((l0 + T) % kScanCkpt != 0 && l0 + T < p.L)) return;
    const int N = p.N;
    float* ck = p.ckpt + (((int64_t)b * p.dim + d) * p.n_ckpt + (l0 + T - 1) / kScanCkpt) * (2 * N) + 2 * n0;
    if ((N & 1) == 0 && n0 < N) {
        *reinterpret_cast<float4*>(ck) = make_float4(0.f, h.x, 0.f, h.y);
    } else {
        if (n0 < N) { ck[0] = 0.f; ck[1] = h.x; }
        if (n0 + 1 < N) { ck[2] = 0.f; ck[3] = h.y; }
    }
}

}  // namespace vmb
