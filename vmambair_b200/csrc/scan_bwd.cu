// Selective-scan backward for sm_90a -- replaces selective_scan_bwd_kernel
// (reference: Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan_bwd_kernel.cuh:66-273).
//
// Same warp-autonomous mapping as the forward (scan_fwd.cu): a warp owns RB rows x (32/RB) segments
// of T=16 positions and walks the sequence BACKWARDS in warp-chunks; the state at each chunk start
// comes from the forward's checkpoints (interval kScanCkpt), so nothing is recomputed across chunks.
// Per state pair (packed f32x2):
//   F1  a=ex2(A' dt), local end state  -> forward segment scan -> true segment start state
//   F2  g_t = a_t h_{t-1}  (kept in registers; h_t = g_t + b_t)
//   R1  local reverse recurrence dh_t = C_t dout_t + a_{t+1} dh_{t+1} -> reverse segment scan
//   R2  true dh_t and every gradient term:
//         du  += dt * sum_n dh B            ddt += u * sum_n dh B + sum_n A dh g
//         dA  += dt dh g                    dB  += dh dt u  (reduced over the rows of the group)
//         dC  += dout h                     (reduced over the rows of the group)
// dB/dC row reduction: inside the warp through a conflict-free smem transpose, across warps with one
// 16-byte vector reduction (REDG.F32x4) per (state pair, position) into an fp32 scratch laid out
// [b][g][n/2][l][4]; a small finalize kernel converts it to (B,G,N,L) in the I/O dtype -- the
// reference does one scalar atomicAdd per ROW per (n,l) (bwd kernel :209-221) and casts in torch.
#include <stdlib.h>

#include <type_traits>

#include "scan_common.cuh"

namespace vmb {

template <typename in_t, int RB, int NIO = 3>
struct BwdSmem {
    using Cfg = FwdCfg<RB>;
    using R = RawCfg<in_t, RB, NIO>;
    static constexpr size_t red_bytes = sizeof(float4) * Cfg::SEGW * T * RB;  // [sl][t][r] float4
    static size_t bytes(int npad) {
        return sizeof(float4) * (2 * 8 * Cfg::SLOTS) + R::bytes + red_bytes + sizeof(float) * (4 * RB * npad + RB);
    }
};

__device__ __forceinline__ void red_add_f32x4(float4* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

// g_t: element type of dout.  float with 16-bit in_t (selective_scan_cuda_oflex's fp32 dout): dout is read straight from global
// memory (16 B vectors when aligned) and only u / delta are staged (NIO = 2); every output keeps its type.
// DET (deterministic mode, scan_params.h): plain stores into the warp's own partial slots instead of float atomics; the contributor
// of a (batch, group) is the warp's index inside the group.
template <typename in_t, int RB, typename g_t, bool DET = false>
__global__ void __launch_bounds__(32, 8) scan_bwd_kernel(const ScanBwdParams p) {
    pdl_wait();
    constexpr bool G_IN = std::is_same<g_t, in_t>::value;
    constexpr int NIO = G_IN ? 3 : 2;
    using Cfg = FwdCfg<RB>;
    using R = RawCfg<in_t, RB, NIO>;
    constexpr int SEGW = Cfg::SEGW, CHUNK = Cfg::CHUNK, SEGQ = Cfg::SEGQ, SLOTS = Cfg::SLOTS;
    constexpr int V = Vec<in_t>::N;

    extern __shared__ float4 smem_f4[];
    float4* sB = smem_f4;
    float4* sC = sB + 8 * SLOTS;
    float4* sRed = sC + 8 * SLOTS;                                     // [SEGW*T][RB]
    in_t* raw = reinterpret_cast<in_t*>(sRed + SEGW * T * RB);
    float* sSt = reinterpret_cast<float*>(reinterpret_cast<char*>(raw) + R::bytes);  // [RB][npad] fwd state at chunk start
    float* sCarryD = sSt + RB * p.npad;                                // [RB][npad] dh at the first position of the next chunk
    float* sA = sCarryD + RB * p.npad;                                 // [RB][npad] A * log2(e)
    float* sdA = sA + RB * p.npad;                                     // [RB][npad] dA accumulators
    float* sDtNext = sdA + RB * p.npad;                                // [RB] dt of the first position of the next chunk

    const int lane = threadIdx.x;
    const int r = lane % RB, sl = lane / RB;
    const int blocks_per_batch = p.dim / RB;
    const int b = blockIdx.x / blocks_per_batch;
    const int d0 = (blockIdx.x % blocks_per_batch) * RB, d = d0 + r;
    const int g = d0 / p.rows_per_group;
    const int N = p.N, L = p.L, npad = p.npad;
    const bool async_ok = p.vec_ok;

    const in_t* __restrict__ Bg = reinterpret_cast<const in_t*>(p.Bm) + (int64_t)b * p.B_bs + (int64_t)g * p.B_gs;
    const in_t* __restrict__ Cg = reinterpret_cast<const in_t*>(p.Cm) + (int64_t)b * p.C_bs + (int64_t)g * p.C_gs;
    const in_t* io_base[3] = {reinterpret_cast<const in_t*>(p.u) + (int64_t)b * p.u_bs + (int64_t)d0 * p.u_ds,
                              reinterpret_cast<const in_t*>(p.delta) + (int64_t)b * p.dl_bs + (int64_t)d0 * p.dl_ds,
                              reinterpret_cast<const in_t*>(p.dout) + (int64_t)b * p.do_bs + (int64_t)d0 * p.do_ds};
    const int64_t io_ds[3] = {p.u_ds, p.dl_ds, p.do_ds};
    const in_t* __restrict__ urow = io_base[0] + (int64_t)r * p.u_ds;
    const in_t* __restrict__ drow = io_base[1] + (int64_t)r * p.dl_ds;
    const in_t* __restrict__ gorow = io_base[2] + (int64_t)r * p.do_ds;
    in_t* __restrict__ durow = reinterpret_cast<in_t*>(p.du) + (int64_t)b * p.du_bs + (int64_t)d * p.du_ds;
    in_t* __restrict__ ddrow = reinterpret_cast<in_t*>(p.ddelta) + (int64_t)b * p.dd_bs + (int64_t)d * p.dd_ds;
    int64_t slot = (int64_t)b * p.G + g;
    if constexpr (DET) slot += (int64_t)((d0 % p.rows_per_group) / RB) * p.batch * p.G;
    float4* __restrict__ scratch = reinterpret_cast<float4*>(p.dBC) + slot * (npad / 2) * (int64_t)L;
    const float* __restrict__ ckrow = p.ckpt + ((int64_t)b * p.dim + d0) * p.n_ckpt * N;  // + (rr*n_ckpt + k)*N + n

    const int nchunks = (L + CHUNK - 1) / CHUNK;
    if (async_ok) prefetch_chunk<in_t, RB, NIO>(raw, io_base, io_ds, Bg, Cg, p.B_ns, p.C_ns, N, (nchunks - 1) * CHUNK, L, lane);
    for (int i = lane; i < RB * npad; i += 32) {
        const int rr = i / npad, n = i % npad;
        sA[i] = n < N ? p.A[(int64_t)(d0 + rr) * N + n] * kLog2e : 0.f;
        sCarryD[i] = 0.f;
        sdA[i] = 0.f;
    }
    if (lane < RB) sDtNext[lane] = 0.f;
    const float Dval = p.D ? p.D[d] : 0.f;
    const float bias = p.bias ? p.bias[d] : 0.f;
    const int ntiles = npad / 16;
    float dD_acc = 0.f, dbias_acc = 0.f;

    for (int ci = nchunks - 1; ci >= 0; --ci) {
        const int c0 = ci * CHUNK;
        const int l0 = c0 + sl * T;
        const int valid = min(max(L - l0, 0), T);
        float uv[T], dt[T], go[T];
        if (async_ok) {
            cp_async_wait_all();
            __syncwarp();
            convert_bc<in_t, RB, NIO>(sB, raw + (NIO * RB) * R::PITCH, lane);
            convert_bc<in_t, RB, NIO>(sC, raw + (NIO * RB + 16) * R::PITCH, lane);
#pragma unroll
            for (int v = 0; v < T / V; ++v) {
                load_vec_smem<in_t>(raw + r * R::PITCH + sl * T + v * V, uv + v * V);
                load_vec_smem<in_t>(raw + (RB + r) * R::PITCH + sl * T + v * V, dt + v * V);
                if constexpr (G_IN) load_vec_smem<in_t>(raw + (2 * RB + r) * R::PITCH + sl * T + v * V, go + v * V);
            }
            __syncwarp();
            if (ci > 0) prefetch_chunk<in_t, RB, NIO>(raw, io_base, io_ds, Bg, Cg, p.B_ns, p.C_ns, N, c0 - CHUNK, L, lane);
        } else {
#pragma unroll
            for (int v = 0; v < T / V; ++v) {
                load_vec<in_t>(urow + l0 + v * V, uv + v * V, valid - v * V, false);
                load_vec<in_t>(drow + l0 + v * V, dt + v * V, valid - v * V, false);
                if constexpr (G_IN) load_vec<in_t>(gorow + l0 + v * V, go + v * V, valid - v * V, false);
            }
        }
        if constexpr (!G_IN) {
            constexpr int VG = Vec<g_t>::N;
            const g_t* __restrict__ grow = reinterpret_cast<const g_t*>(p.dout) + (int64_t)b * p.do_bs + (int64_t)d * p.do_ds;
#pragma unroll
            for (int v = 0; v < T / VG; ++v) load_vec<g_t>(grow + l0 + v * VG, go + v * VG, valid - v * VG, p.vec_ok);
        }
        // forward state at the chunk start (checkpoint written by the forward; zero for the first chunk)
        for (int i = lane; i < RB * npad; i += 32) {
            const int rr = i / npad, n = i % npad;
            sSt[i] = (c0 > 0 && n < N) ? ckrow[((int64_t)rr * p.n_ckpt + (c0 / kScanCkpt - 1)) * N + n] : 0.f;
        }
        float sigma = 0.f;
        float dtu[T], s1[T], s2[T];
#pragma unroll
        for (int t = 0; t < T; ++t) {
            float x = dt[t] + bias;
            if (p.softplus) x = softplus_f(x);
            x = t < valid ? x : 0.f;
            dt[t] = x;
            dtu[t] = x * uv[t];
            sigma += x;
            s1[t] = 0.f;
            s2[t] = 0.f;
            dD_acc = fmaf(go[t], uv[t], dD_acc);
        }
        // dt of the position right after this segment (first position of the next segment / next chunk)
        float dt_next = __shfl_down_sync(0xffffffffu, dt[0], RB % 32);
        if (sl == SEGW - 1) dt_next = sDtNext[r];
        const float sigma_r = sigma - dt[0] + dt_next;
        __syncwarp();
        if (sl == 0) sDtNext[r] = dt[0];

        for (int nt = 0; nt < ntiles; ++nt) {
            if (!async_ok || nt > 0) {
                __syncwarp();
                stage_bc<in_t, Cfg>(sB, Bg, p.B_ns, nt * 16, N, c0, L, p.vec_ok, lane);
                stage_bc<in_t, Cfg>(sC, Cg, p.C_ns, nt * 16, N, c0, L, p.vec_ok, lane);
            }
            __syncwarp();

#pragma unroll 1
            for (int np = 0; np < 8; ++np) {
                const int n0 = nt * 16 + 2 * np;
                const float2 A2 = *reinterpret_cast<const float2*>(&sA[r * npad + n0]);
                const float4* __restrict__ bq = sB + np * SLOTS + sl * SEGQ;
                const float4* __restrict__ cq = sC + np * SLOTS + sl * SEGQ;
                // ---- F1: decay factors, local end state ----
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
                float2 E2 = mul2(A2, make_float2(sigma_r, sigma_r));
                E2 = make_float2(ex2(E2.x), ex2(E2.y));
                float2 elast = mul2(A2, make_float2(dt_next, dt_next));
                elast = make_float2(ex2(elast.x), ex2(elast.y));
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
                const float2 st = *reinterpret_cast<const float2*>(&sSt[r * npad + n0]);
                float2 h = fma2(Pe, st, He);
                // ---- F2: g_t = a_t * h_{t-1} ----
                float2 g2[T];
#pragma unroll
                for (int t = 0; t < T; t += 2) {
                    const float4 Bq = bq[t / 2];
                    g2[t] = mul2(a2[t], h);
                    h = add2(g2[t], mul2(make_float2(dtu[t], dtu[t]), make_float2(Bq.x, Bq.y)));
                    g2[t + 1] = mul2(a2[t + 1], h);
                    h = add2(g2[t + 1], mul2(make_float2(dtu[t + 1], dtu[t + 1]), make_float2(Bq.z, Bq.w)));
                }
                // ---- R1: local reverse recurrence (zero incoming) ----
                float2 dl = make_float2(0.f, 0.f);
#pragma unroll
                for (int t = T - 2; t >= 0; t -= 2) {
                    const float4 Cq = cq[t / 2];
                    const float2 e_hi = (t + 1 == T - 1) ? elast : a2[t + 2];
                    dl = fma2(e_hi, dl, mul2(make_float2(go[t + 1], go[t + 1]), make_float2(Cq.z, Cq.w)));
                    dl = fma2(a2[t + 1], dl, mul2(make_float2(go[t], go[t]), make_float2(Cq.x, Cq.y)));
                }
#pragma unroll
                for (int o = RB; o < 32; o <<= 1) {
                    const float2 Ep = shfl_down2(E2, o), Dp = shfl_down2(dl, o);
                    if (lane + o < 32) {
                        dl = fma2(E2, Dp, dl);
                        E2 = mul2(E2, Ep);
                    }
                }
                float2 Ee = shfl_down2(E2, RB % 32), De = shfl_down2(dl, RB % 32);
                if (sl == SEGW - 1) {
                    Ee = make_float2(1.f, 1.f);
                    De = make_float2(0.f, 0.f);
                }
                float2* carry = reinterpret_cast<float2*>(&sCarryD[r * npad + n0]);
                const float2 Xw = *carry;
                float2 dh = fma2(Ee, Xw, De);
                __syncwarp();
                if (sl == 0) *carry = fma2(E2, Xw, dl);
                // ---- R2: true dh_t and the gradient terms ----
                const float2 A2r = mul2(A2, make_float2(kLn2, kLn2));  // un-scaled A
                float2 dA2 = make_float2(0.f, 0.f);
                float4* red = sRed + (sl * T) * RB;
#pragma unroll
                for (int t = T - 2; t >= 0; t -= 2) {
                    const float4 Bq = bq[t / 2];
                    const float4 Cq = cq[t / 2];
#pragma unroll
                    for (int k = 1; k >= 0; --k) {
                        const int tt = t + k;
                        const float2 Bv = k ? make_float2(Bq.z, Bq.w) : make_float2(Bq.x, Bq.y);
                        const float2 Cv = k ? make_float2(Cq.z, Cq.w) : make_float2(Cq.x, Cq.y);
                        const float2 e = (tt == T - 1) ? elast : a2[tt + 1];
                        dh = fma2(e, dh, mul2(make_float2(go[tt], go[tt]), Cv));
                        s1[tt] = fmaf(dh.y, Bv.y, fmaf(dh.x, Bv.x, s1[tt]));
                        const float2 q = mul2(dh, g2[tt]);
                        s2[tt] = fmaf(A2r.y, q.y, fmaf(A2r.x, q.x, s2[tt]));
                        dA2 = fma2(q, make_float2(dt[tt], dt[tt]), dA2);
                        const float2 vB = mul2(dh, make_float2(dtu[tt], dtu[tt]));
                        const float2 hh = add2(g2[tt], mul2(make_float2(dtu[tt], dtu[tt]), Bv));
                        const float2 vC = mul2(hh, make_float2(go[tt], go[tt]));
                        red[tt * RB + ((r + tt) % RB)] = make_float4(vB.x, vB.y, vC.x, vC.y);
                    }
                }
                // dA: reduce over the warp's segments, accumulate in smem (single writer per (row, n))
#pragma unroll
                for (int o = RB; o < 32; o <<= 1) {
                    dA2.x += __shfl_xor_sync(0xffffffffu, dA2.x, o);
                    dA2.y += __shfl_xor_sync(0xffffffffu, dA2.y, o);
                }
                if (sl == 0) {
                    float2* da = reinterpret_cast<float2*>(&sdA[r * npad + n0]);
                    *da = add2(*da, dA2);
                }
                __syncwarp();
                // dB/dC: sum the RB rows of each (segment, position) cell, one vector reduction per cell
#pragma unroll
                for (int cell = lane; cell < SEGW * T; cell += 32) {
                    const float4* src = sRed + cell * RB;
                    float4 acc = src[cell % RB];
#pragma unroll
                    for (int j = 1; j < RB; ++j) {
                        const float4 v = src[(j + cell) % RB];
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    }
                    const int l = c0 + cell;
                    if constexpr (DET) {
                        if (l < L && n0 < N) scratch[(int64_t)(n0 / 2) * L + l] = acc;
                    } else {
                        if (l < L && n0 < N) red_add_f32x4(scratch + (int64_t)(n0 / 2) * L + l, acc);
                    }
                }
                __syncwarp();
            }
        }
        // ---- per-position outputs ----
        float duo[T], ddo[T];
#pragma unroll
        for (int t = 0; t < T; ++t) {
            duo[t] = fmaf(Dval, go[t], dt[t] * s1[t]);
            float dd = fmaf(uv[t], s1[t], s2[t]);
            // d softplus(x)/dx = sigmoid(x) = 1 - exp(-softplus(x));  for x > 20 the reference passes dd through (=1 to fp32)
            if (p.softplus) dd *= 1.f - ex2(-dt[t] * kLog2e);
            dd = t < valid ? dd : 0.f;
            ddo[t] = dd;
            dbias_acc += dd;
        }
#pragma unroll
        for (int v = 0; v < T / V; ++v) {
            store_vec<in_t>(durow + l0 + v * V, duo + v * V, valid - v * V, p.vec_ok);
            store_vec<in_t>(ddrow + l0 + v * V, ddo + v * V, valid - v * V, p.vec_ok);
        }
    }
    // ---- per-row parameter gradients ----
#pragma unroll
    for (int o = RB; o < 32; o <<= 1) {
        dD_acc += __shfl_xor_sync(0xffffffffu, dD_acc, o);
        dbias_acc += __shfl_xor_sync(0xffffffffu, dbias_acc, o);
    }
    if (sl == 0) {
        if constexpr (DET) {
            if (p.dD) p.dD[(int64_t)b * p.dim + d] = dD_acc;
            if (p.dbias) p.dbias[(int64_t)b * p.dim + d] = dbias_acc;
        } else {
            if (p.dD) atomicAdd(p.dD + d, dD_acc);
            if (p.dbias) atomicAdd(p.dbias + d, dbias_acc);
        }
    }
    __syncwarp();
    for (int i = lane; i < RB * npad; i += 32) {
        const int rr = i / npad, n = i % npad;
        if constexpr (DET) {
            if (n < N) p.dA[((int64_t)b * p.dim + d0 + rr) * N + n] = sdA[i];
        } else {
            if (n < N) atomicAdd(p.dA + (int64_t)(d0 + rr) * N + n, sdA[i]);
        }
    }
}

// scratch [b][g][npad/2][L][4] fp32 -> dB, dC (B,G,N,L) in the I/O dtype
template <typename in_t>
__global__ void scan_bwd_finalize_kernel(const float4* __restrict__ scratch, in_t* __restrict__ dB, in_t* __restrict__ dC,
                                         int N, int npad, int L, long total) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over (b*g, np, l)
    if (i >= total) return;
    const int l = (int)(i % L);
    const long t = i / L;
    const int np = (int)(t % (npad / 2));
    const long bg = t / (npad / 2);
    const float4 v = scratch[i];
    const int n0 = 2 * np;
    if (n0 < N) {
        dB[(bg * N + n0) * L + l] = from_f32<in_t>(v.x);
        dC[(bg * N + n0) * L + l] = from_f32<in_t>(v.z);
    }
    if (n0 + 1 < N) {
        dB[(bg * N + n0 + 1) * L + l] = from_f32<in_t>(v.y);
        dC[(bg * N + n0 + 1) * L + l] = from_f32<in_t>(v.w);
    }
}

// deterministic mode: the sums over contributors (in index order), then over the batch (in index order) -- dB / dC are written in the
// I/O dtype, dA / dD / ddelta_bias receive ONE addition each.  Threads [0, n_bc) own a (b, g, n/2, l) cell, the rest a (row, n) of
// the parameter gradients (n = N: dD, n = N+1: ddelta_bias).
template <typename in_t, bool GRP>
__global__ void scan_bwd_det_finalize_kernel(const ScanBwdDetFin f, const ScanBwdGroups gr, long n_bc, long n_prm) {
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_bc) {
        const int L = f.L, N = f.N;
        const int l = (int)(i % L);
        const long t = i / L;
        const int np = (int)(t % (f.npad / 2));
        const long bg = t / (f.npad / 2);
        const int n0 = 2 * np;
        if (n0 >= N) return;  // padding states: never written
        float4 v = f.bc[i];
        for (int c = 1; c < f.nc; ++c) {
            const float4 w = f.bc[(long)c * n_bc + i];
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        in_t *dB, *dC;
        int64_t sB, sC;
        if constexpr (GRP) {
            const int g = (int)(bg % gr.ndesc);
            const int64_t b = bg / gr.ndesc;
            const ScanBwdGroupDesc& gd = gr.grp[g];
            const int m = gd.rev ? L - 1 - l : l;
            dB = reinterpret_cast<in_t*>(gd.dB) + b * gr.dB_bs + m + n0 * gr.dB_ns;
            dC = reinterpret_cast<in_t*>(gd.dC) + b * gr.dC_bs + m + n0 * gr.dC_ns;
            sB = gr.dB_ns;
            sC = gr.dC_ns;
        } else {
            dB = reinterpret_cast<in_t*>(f.dB) + (bg * N + n0) * L + l;
            dC = reinterpret_cast<in_t*>(f.dC) + (bg * N + n0) * L + l;
            sB = sC = L;
        }
        dB[0] = from_f32<in_t>(v.x);
        dC[0] = from_f32<in_t>(v.z);
        if (n0 + 1 < N) {
            dB[sB] = from_f32<in_t>(v.y);
            dC[sC] = from_f32<in_t>(v.w);
        }
        return;
    }
    const long j = i - n_bc;
    if (j >= n_prm) return;
    const int N2 = f.N + 2;
    const long d = j / N2;
    const int n = (int)(j % N2);
    const float* src;
    float* dst;
    long stride, off;
    if (n < f.N) {
        src = f.pA; dst = f.dA + d * f.N + n; stride = (long)f.dim * f.N; off = d * f.N + n;
    } else {
        src = n == f.N ? f.pD : f.pbias;
        dst = n == f.N ? f.dD + d : f.dbias + d;
        stride = f.dim;
        off = d;
        if (!src) return;
    }
    float s = 0.f;
    for (int b = 0; b < f.batch; ++b) s += src[b * stride + off];
    *dst += s;
}

template <typename in_t>
static int det_finalize_t(const ScanBwdDetFin& f, const ScanBwdGroups* gr, cudaStream_t stream) {
    const long n_bc = (long)f.batch * f.G * (f.npad / 2) * f.L, n_prm = (long)f.dim * (f.N + 2);
    const unsigned blocks = (unsigned)((n_bc + n_prm + 255) / 256);
    if (gr) VMB_CUDA(launch_pdl(scan_bwd_det_finalize_kernel<in_t, true>, dim3(blocks), dim3(256), 0, stream, f, *gr, n_bc, n_prm));
    else VMB_CUDA(launch_pdl(scan_bwd_det_finalize_kernel<in_t, false>, dim3(blocks), dim3(256), 0, stream, f, ScanBwdGroups{}, n_bc, n_prm));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int scan_bwd_det_finalize(const ScanBwdDetFin& f, const ScanBwdGroups* gr, int dtype, cudaStream_t stream) {
    switch (dtype) {
        case VMB_F32: return det_finalize_t<float>(f, gr, stream);
        case VMB_BF16: return det_finalize_t<__nv_bfloat16>(f, gr, stream);
        case VMB_F16: return det_finalize_t<__half>(f, gr, stream);
    }
    set_error("selective_scan_bwd: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

template <typename in_t, int RB, typename g_t, bool DET = false>
static int launch_cfg(const ScanBwdParams& p, cudaStream_t stream) {
    auto kern = scan_bwd_kernel<in_t, RB, g_t, DET>;
    const size_t smem = BwdSmem<in_t, RB, std::is_same<g_t, in_t>::value ? 3 : 2>::bytes(p.npad);
    VMB_CHECK(smem <= 227 * 1024, "selective_scan_bwd: dstate=%d needs %zu B of shared memory", p.N, smem);
    if (smem > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long blocks = (long)p.batch * (p.dim / RB);
    if constexpr (DET) VMB_CUDA(launch_pdl(kern, dim3((unsigned)blocks), dim3(32), smem, stream, p));
    else kern<<<(unsigned)blocks, 32, smem, stream>>>(p);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// warp-chunks must be a multiple of the checkpoint interval (64): RB in {8,4,2,1}
static int pick_rb_bwd(const ScanBwdParams& p) {
    const int rpg = p.rows_per_group;
    // few rows -> fewer rows per warp (more warps; their smem footprint still allows >= 3 warps per SM at RB=2)
    const long rows = (long)p.batch * p.dim;
    int rb = rows < 1536 ? 2 : rows < 6144 ? 4 : 8;
    while (rb > 1 && rpg % rb) rb >>= 1;
    return rb;
}

template <typename in_t> struct DtOf;
template <> struct DtOf<float> { static constexpr int v = VMB_F32; };
template <> struct DtOf<__nv_bfloat16> { static constexpr int v = VMB_BF16; };
template <> struct DtOf<__half> { static constexpr int v = VMB_F16; };

template <typename in_t, typename g_t = in_t>
static int launch_t(const ScanBwdParams& p, cudaStream_t stream) {
    constexpr bool dout_f32 = !std::is_same<g_t, in_t>::value;
    const size_t scratch_bytes = sizeof(float4) * (size_t)p.batch * p.G * (p.npad / 2) * p.L;
    VMB_CUDA(cudaMemsetAsync(p.dBC, 0, scratch_bytes, stream));
    int rc;
    int trb, tss;
    if (scan_bwd_tma_pick(p, trb, tss)) {  // fast path: TMA-staged 4-warp CTAs (scan_bwd_tma.cu)
        rc = scan_bwd_tma_launch(p, DtOf<in_t>::v, trb, tss, stream, dout_f32);
    } else
    switch (pick_rb_bwd(p)) {
        case 8: rc = launch_cfg<in_t, 8, g_t>(p, stream); break;
        case 4: rc = launch_cfg<in_t, 4, g_t>(p, stream); break;
        case 2: rc = launch_cfg<in_t, 2, g_t>(p, stream); break;
        default: rc = launch_cfg<in_t, 1, g_t>(p, stream); break;
    }
    if (rc != VMB_OK) return rc;
    const long total = (long)p.batch * p.G * (p.npad / 2) * p.L;
    scan_bwd_finalize_kernel<in_t><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(p.dBC), reinterpret_cast<in_t*>(p.dB), reinterpret_cast<in_t*>(p.dC), p.N, p.npad,
        p.L, total);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// deterministic mode: contributors of one (batch, group) -- the CTAs (TMA path) or warps (generic path) that share it
static int det_contributors(const ScanBwdParams& p, int& trb, int& tss, int& rb) {
    if (scan_bwd_tma_pick(p, trb, tss)) return p.rows_per_group / (trb * 4 / tss);
    trb = 0;
    rb = pick_rb_bwd(p);
    return p.rows_per_group / rb;
}

int64_t scan_bwd_det_workspace(const ScanBwdParams& p) {
    int trb, tss, rb;
    return scan_bwd_det_bytes(p, det_contributors(p, trb, tss, rb));
}

template <typename in_t, typename g_t = in_t>
static int launch_det_t(const ScanBwdParams& p_in, cudaStream_t stream) {
    constexpr bool dout_f32 = !std::is_same<g_t, in_t>::value;
    ScanBwdParams p = p_in;
    int trb, tss, rb = 1;
    const ScanBwdDetFin f = scan_bwd_det_carve(p, det_contributors(p, trb, tss, rb));
    int rc;
    if (trb) {
        rc = scan_bwd_tma_launch(p, DtOf<in_t>::v, trb, tss, stream, dout_f32, true);
    } else
    switch (rb) {
        case 8: rc = launch_cfg<in_t, 8, g_t, true>(p, stream); break;
        case 4: rc = launch_cfg<in_t, 4, g_t, true>(p, stream); break;
        case 2: rc = launch_cfg<in_t, 2, g_t, true>(p, stream); break;
        default: rc = launch_cfg<in_t, 1, g_t, true>(p, stream); break;
    }
    if (rc != VMB_OK) return rc;
    return det_finalize_t<in_t>(f, nullptr, stream);
}

int scan_bwd_launch(const ScanBwdParams& p, int dtype, cudaStream_t stream, bool dout_f32, bool det) {
    VMB_CHECK((long)p.batch * p.dim < (1L << 31), "selective_scan_bwd: batch*dim too large");
    if (dout_f32) {  // fp32 dout against 16-bit inputs
        switch (dtype) {
            case VMB_BF16: return det ? launch_det_t<__nv_bfloat16, float>(p, stream) : launch_t<__nv_bfloat16, float>(p, stream);
            case VMB_F16: return det ? launch_det_t<__half, float>(p, stream) : launch_t<__half, float>(p, stream);
        }
        set_error("selective_scan_bwd: fp32 dout needs bf16 / fp16 inputs (dtype %d)", dtype);
        return VMB_ERR_INVALID;
    }
    switch (dtype) {
        case VMB_F32: return det ? launch_det_t<float>(p, stream) : launch_t<float>(p, stream);
        case VMB_BF16: return det ? launch_det_t<__nv_bfloat16>(p, stream) : launch_t<__nv_bfloat16>(p, stream);
        case VMB_F16: return det ? launch_det_t<__half>(p, stream) : launch_t<__half>(p, stream);
    }
    set_error("selective_scan_bwd: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

}  // namespace vmb
