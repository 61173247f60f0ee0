// Selective-scan backward, TMA-staged multi-warp variant (sm_90a) -- the fast path of vmb_selective_scan_bwd.
// Replaces selective_scan_bwd_kernel (reference: Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan_bwd_kernel.cuh:66-273).
//
// Same per-pair math as scan_bwd.cu (F1 decay factors + local end state, forward segment scan from the forward's checkpoints,
// F2 g_t = a_t h_{t-1}, R1 local reverse recurrence, reverse segment scan, R2 true dh_t and every gradient term), re-plumbed like
// the forward (scan_fwd_tma.cu):
//   * a CTA of 4 warps owns RB*4/SS rows of one (batch, group); u / delta / dout rows and the 16 B and 16 C state rows arrive as
//     cp.async.bulk.tensor boxes (one issuing thread, mbarrier completion) one chunk ahead, walking the sequence backwards;
//   * ONE fp32 B/C pair tile per CTA instead of one per warp (single-warp CTAs would each convert their own tile) -> RB = 2
//     rows per warp is affordable: 768 warps at batch 4, 4-8 per SM;
//   * state split (SS): the 8 state pairs of a row over SS warps at small batch; the per-position sums over states (s1, s2) meet in
//     shared memory, du / ddelta are written by the first warp of the row slot;
//   * the dB/dC row reduction: warp-local smem transpose ([row][segment][T + 1] float4: the (row, segment) lanes write without bank
//     conflicts, the position-per-lane reads are contiguous; the round-1 layout had 13.7 M conflicts per launch), then the warps of the CTA that share the state pair meet at a named barrier and issue ONE
//     red.global.add.v4.f32 per (pair, position, CTA).
#include <stdlib.h>

#include <type_traits>

#include "scan_tma_common.cuh"

namespace vmb {

// plain operator: index 0 only (B/C group = z coordinate); grouped (NM = 4): one map per group and operand
template <int NM>
struct ScanBwdTmaMapsN {
    CUtensorMap u[NM], d[NM], g[NM], b[NM], c[NM];
};
struct ScanBwdTmaMapsG : ScanBwdTmaMapsN<4> {
    ScanBwdGroups gr;
};
template <bool GRP>
using BwdMaps = typename std::conditional<GRP, ScanBwdTmaMapsG, ScanBwdTmaMapsN<1>>::type;

// g_t: element type of dout (float with 16-bit in_t: selective_scan_cuda_oflex's fp32 dout); its tile has its own width
template <typename in_t, int RB, int SS, typename g_t = in_t>
struct BwdTmaCfg {
    using Cfg = FwdCfg<RB>;
    static constexpr int NW = 4;
    static constexpr int CHUNK = Cfg::CHUNK, SLOTS = Cfg::SLOTS, SEGW = Cfg::SEGW;
    static constexpr int ROWS = RB * (NW / SS);
    static constexpr int NPW = 8 / SS;
    static constexpr int CELLS = SEGW * T;                      // positions of a warp-chunk (= CHUNK)
    static constexpr int RED_RS = SEGW * (T + 1) + 4;           // float4 slots of one row of a warp's dB/dC transpose: [segment][T + 1 pad] (+4: rows half a wavefront apart)
    static constexpr int RED_F4 = RED_RS * RB + 8;              // (odd segment pitch: conflict-free writes by (row, segment) lanes, contiguous reads)
    static constexpr size_t io_bytes = sizeof(in_t) * (size_t)ROWS * CHUNK;  // one of rawU / rawD
    static constexpr size_t g_bytes = sizeof(g_t) * (size_t)ROWS * CHUNK;    // rawG
    static constexpr size_t bc_bytes = sizeof(in_t) * (size_t)16 * CHUNK;
    static constexpr size_t tile_bytes = sizeof(float4) * (size_t)16 * SLOTS;
    static constexpr size_t red_bytes = sizeof(float4) * (size_t)RED_F4;
    static constexpr size_t warp_f32 = 4 * RB * 16 + RB;  // sSt, sCarryD, sA, sdA [RB][16] + sDtNext [RB]
    static constexpr size_t warp_bytes = red_bytes + sizeof(float) * ((warp_f32 + 3) / 4 * 4);
    static constexpr size_t part_bytes = SS > 1 ? sizeof(float) * (size_t)(NW / SS) * (SS - 1) * 2 * T * 32 : 0;
    static constexpr size_t smem_bytes = 2 * io_bytes + g_bytes + 2 * bc_bytes + tile_bytes + NW * warp_bytes + part_bytes + 16;
    static constexpr uint32_t tx_bytes = (uint32_t)(2 * io_bytes + g_bytes + 2 * bc_bytes);
};

__device__ __forceinline__ void red_add_f32x4_g(float4* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// DET: a plain store into this CTA's own partial slot (summed in a fixed order by scan_bwd_det_finalize_kernel)
template <bool DET>
__device__ __forceinline__ void put_bc(float4* addr, float4 v) {
    if constexpr (DET) *addr = v;
    else red_add_f32x4_g(addr, v);
}


// named barrier BASE + idx (idx < 4) with an immediate id, so that ptxas counts the barriers really used
template <int BASE>
__device__ __forceinline__ void named_bar_sync(int idx, int count) {
    switch (idx) {
        case 0: asm volatile("bar.sync %0, %1;" ::"n"(BASE), "r"(count) : "memory"); break;
        case 1: asm volatile("bar.sync %0, %1;" ::"n"(BASE + 1), "r"(count) : "memory"); break;
        case 2: asm volatile("bar.sync %0, %1;" ::"n"(BASE + 2), "r"(count) : "memory"); break;
        default: asm volatile("bar.sync %0, %1;" ::"n"(BASE + 3), "r"(count) : "memory"); break;
    }
}

// GRP: per-group sources and destinations (vmb_selective_scan_bwd_grouped); a reversed group loads mirrored boxes (m0 = L - c0 - CHUNK,
// underflow zero-filled as in the forward), reads them back to front and stores du / ddelta at memory index L-1-l.
// g_t = float with 16-bit in_t (flat operator only): fp32 dout, converted on read; every output keeps its type.
// DET (deterministic mode): no float atomics.  The launcher points p.dBC / p.dA / p.dD / p.dbias at partial slots of the workspace;
// the CTA stores its dB/dC row sums into slot [contributor][b][g][n/2][l] (contributor = the CTA's index inside its group) and its
// dA / dD / ddelta_bias into [b][row](..), each slot written by exactly one CTA.
template <typename in_t, int RB, int SS, bool GRP, typename g_t, bool DET = false>
__global__ void __launch_bounds__(128, sizeof(in_t) == 4 ? 1 : 2)
    scan_bwd_tma_kernel(const ScanBwdParams p, const __grid_constant__ BwdMaps<GRP> maps) {
    pdl_wait();
    using K = BwdTmaCfg<in_t, RB, SS, g_t>;
    using Cfg = FwdCfg<RB>;
    constexpr int SEGW = Cfg::SEGW, CHUNK = Cfg::CHUNK, SEGQ = Cfg::SEGQ, SLOTS = Cfg::SLOTS;
    constexpr int V = Vec<in_t>::N, NW = K::NW, NT = 32 * NW, ROWS = K::ROWS, NPW = K::NPW;
    constexpr int GW = NW / SS;  // warps of the CTA that share a state-pair set (different rows of the same group)

    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem_raw = smem_dyn + ((128u - (smem_addr(smem_dyn) & 127u)) & 127u);
    in_t* rawU = reinterpret_cast<in_t*>(smem_raw);
    in_t* rawD = reinterpret_cast<in_t*>(smem_raw + K::io_bytes);
    g_t* rawG = reinterpret_cast<g_t*>(smem_raw + 2 * K::io_bytes);
    in_t* rawB = reinterpret_cast<in_t*>(smem_raw + 2 * K::io_bytes + K::g_bytes);
    in_t* rawC = reinterpret_cast<in_t*>(smem_raw + 2 * K::io_bytes + K::g_bytes + K::bc_bytes);
    float4* sB = reinterpret_cast<float4*>(smem_raw + 2 * K::io_bytes + K::g_bytes + 2 * K::bc_bytes);
    float4* sC = sB + 8 * SLOTS;
    unsigned char* after_tile = reinterpret_cast<unsigned char*>(sC + 8 * SLOTS);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float4* sRed = reinterpret_cast<float4*>(after_tile + warp * K::warp_bytes);  // this warp's dB/dC transpose
    float* sSt = reinterpret_cast<float*>(sRed + K::RED_F4);                       // [RB][16] forward state at the chunk start
    float* sCarryD = sSt + RB * 16;                                               // [RB][16] dh at the first position of the next chunk
    float* sA = sCarryD + RB * 16;                                                // [RB][16] A * log2(e)
    float* sdA = sA + RB * 16;                                                    // [RB][16] dA accumulators
    float* sDtNext = sdA + RB * 16;                                               // [RB] dt of the first position of the next chunk
    float* spart = reinterpret_cast<float*>(after_tile + NW * K::warp_bytes);     // SS > 1: [row slot][SS-1][2][T][32]
    uint64_t* bar = reinterpret_cast<uint64_t*>(after_tile + NW * K::warp_bytes + K::part_bytes);

    const int rs = warp / SS, sp = warp % SS;
    const int r = lane % RB, sl = lane / RB;
    const int ctas_per_batch = p.dim / ROWS;
    const int b = blockIdx.x / ctas_per_batch;
    const int dc0 = (blockIdx.x % ctas_per_batch) * ROWS;
    const int g = dc0 / p.rows_per_group;
    const int d0 = dc0 + rs * RB, d = d0 + r;
    const int N = p.N, L = p.L;

    // grouped: group g's own tensors, rows indexed inside the group
    const void *du_base = p.du, *dd_base = p.ddelta;
    bool rev = false;
    int gi = 0, zbc = g, urow0 = dc0, dg = d;
    if constexpr (GRP) {
        const ScanBwdGroupDesc& gd = maps.gr.grp[g];
        urow0 = dc0 - g * p.rows_per_group;
        dg = urow0 + rs * RB + r;
        du_base = gd.du;
        dd_base = gd.ddelta;
        rev = gd.rev != 0;
        gi = g;
        zbc = 0;
    }
    in_t* __restrict__ durow = reinterpret_cast<in_t*>(const_cast<void*>(du_base)) + (int64_t)b * p.du_bs + (int64_t)dg * p.du_ds;
    in_t* __restrict__ ddrow = reinterpret_cast<in_t*>(const_cast<void*>(dd_base)) + (int64_t)b * p.dd_bs + (int64_t)dg * p.dd_ds;
    float4* __restrict__ scratch = reinterpret_cast<float4*>(p.dBC) + ((int64_t)b * p.G + g) * 8 * (int64_t)L;
    if constexpr (DET) scratch += (int64_t)((dc0 % p.rows_per_group) / ROWS) * p.batch * p.G * 8 * L;  // this CTA's own slot
    const float* __restrict__ ckrow = p.ckpt + ((int64_t)b * p.dim + d0) * p.n_ckpt * N;

    const int nchunks = (L + CHUNK - 1) / CHUNK;
    auto issue = [&](int c0) {
        mbarrier_expect_tx(bar, K::tx_bytes);
        if constexpr (!GRP) {
            tma_load_4d(rawU, &maps.u[0], bar, c0, dc0, 0, b);
            tma_load_4d(rawD, &maps.d[0], bar, c0, dc0, 0, b);
            tma_load_4d(rawG, &maps.g[0], bar, c0, dc0, 0, b);
            tma_load_4d(rawB, &maps.b[0], bar, c0, 0, g, b);
            tma_load_4d(rawC, &maps.c[0], bar, c0, 0, g, b);
        } else {
            const int m0 = rev ? L - c0 - CHUNK : c0;  // reversed walk: mirrored box, may start below 0 (zero-filled)
            tma_load_4d(rawU, &maps.u[gi], bar, m0, urow0, 0, b);
            tma_load_4d(rawD, &maps.d[gi], bar, m0, urow0, 0, b);
            tma_load_4d(rawG, &maps.g[gi], bar, m0, urow0, 0, b);
            tma_load_4d(rawB, &maps.b[gi], bar, m0, 0, zbc, b);
            tma_load_4d(rawC, &maps.c[gi], bar, m0, 0, zbc, b);
        }
    };
    if (tid == 0) {
        mbarrier_init(bar, 1);
        mbarrier_init_fence();
        issue((nchunks - 1) * CHUNK);
    }
    for (int i = lane; i < RB * 16; i += 32) {
        const int rr = i / 16, n = i % 16;
        sA[i] = n < N ? p.A[(int64_t)(d0 + rr) * N + n] * kLog2e : 0.f;
        sCarryD[i] = 0.f;
        sdA[i] = 0.f;
    }
    if (lane < RB) sDtNext[lane] = 0.f;
    const float Dval = p.D ? p.D[d] : 0.f;
    const float bias = p.bias ? p.bias[d] : 0.f;
    float dD_acc = 0.f, dbias_acc = 0.f;
    __syncthreads();
    uint32_t phase = 0;

    for (int ci = nchunks - 1; ci >= 0; --ci) {
        const int c0 = ci * CHUNK;
        const int l0 = c0 + sl * T;
        const int valid = min(max(L - l0, 0), T);
        float uv[T], dt[T], go[T];
        mbarrier_wait(bar, phase);
        phase ^= 1;
        if (ci < nchunks - 1) __syncthreads();  // every warp is done with the previous fp32 tile
        convert_bc_dense<in_t, RB, NT>(sB, rawB, tid, GRP && rev);
        convert_bc_dense<in_t, RB, NT>(sC, rawC, tid, GRP && rev);
        if constexpr (!std::is_same<g_t, in_t>::value) {  // fp32 dout: its own vector width
            static_assert(!GRP, "scan_bwd_tma: fp32 dout is a flat-operator mode");
            constexpr int VG = Vec<g_t>::N;
            const int row = rs * RB + r;
#pragma unroll
            for (int v = 0; v < T / V; ++v) {
                load_vec_smem<in_t>(rawU + row * CHUNK + sl * T + v * V, uv + v * V);
                load_vec_smem<in_t>(rawD + row * CHUNK + sl * T + v * V, dt + v * V);
            }
#pragma unroll
            for (int v = 0; v < T / VG; ++v) load_vec_smem<g_t>(rawG + row * CHUNK + sl * T + v * VG, go + v * VG);
        } else {
            const int row = rs * RB + r;
            if (!GRP || !rev) {
#pragma unroll
                for (int v = 0; v < T / V; ++v) {
                    load_vec_smem<in_t>(rawU + row * CHUNK + sl * T + v * V, uv + v * V);
                    load_vec_smem<in_t>(rawD + row * CHUNK + sl * T + v * V, dt + v * V);
                    load_vec_smem<in_t>(rawG + row * CHUNK + sl * T + v * V, go + v * V);
                }
            } else {  // sequence position sl*T+t lives at raw index CHUNK-1-(sl*T+t)
#pragma unroll
                for (int v = 0; v < T / V; ++v) {
                    float tu[V], td[V], tg[V];
                    const int o = row * CHUNK + CHUNK - (sl + 1) * T + v * V;
                    load_vec_smem<in_t>(rawU + o, tu);
                    load_vec_smem<in_t>(rawD + o, td);
                    load_vec_smem<in_t>(rawG + o, tg);
#pragma unroll
                    for (int i = 0; i < V; ++i) {
                        uv[T - 1 - (v * V + i)] = tu[i];
                        dt[T - 1 - (v * V + i)] = td[i];
                        go[T - 1 - (v * V + i)] = tg[i];
                    }
                }
            }
        }
        __syncthreads();  // tile complete, raw buffers consumed
        if (tid == 0 && ci > 0) {
            fence_proxy_async();
            issue(c0 - CHUNK);
        }
        // forward state at the chunk start (checkpoint written by the forward; zero for the first chunk): this warp's pairs
        for (int i = lane; i < RB * 2 * NPW; i += 32) {
            const int rr = i / (2 * NPW), n = sp * 2 * NPW + i % (2 * NPW);
            sSt[rr * 16 + n] = (c0 > 0 && n < N) ? ckrow[((int64_t)rr * p.n_ckpt + (c0 / kScanCkpt - 1)) * N + n] : 0.f;
        }
        softplus_block(dt, bias, p.softplus != 0);
        float sigma = 0.f;
        float dtu[T], s1[T], s2[T];
#pragma unroll
        for (int t = 0; t < T; ++t) {
            dt[t] = t < valid ? dt[t] : 0.f;
            dtu[t] = dt[t] * uv[t];
            sigma += dt[t];
            s1[t] = 0.f;
            s2[t] = 0.f;
            if (sp == 0) dD_acc = fmaf(go[t], uv[t], dD_acc);
        }
        // dt of the position right after this segment (first position of the next segment / next chunk)
        float dt_next = __shfl_down_sync(0xffffffffu, dt[0], RB % 32);
        if (sl == SEGW - 1) dt_next = sDtNext[r];
        const float sigma_r = sigma - dt[0] + dt_next;
        __syncwarp();
        if (sl == 0) sDtNext[r] = dt[0];
        __syncwarp();

#pragma unroll 1
        for (int np = sp * NPW; np < (sp + 1) * NPW; ++np) {
            const int n0 = 2 * np;
            const float2 A2 = *reinterpret_cast<const float2*>(&sA[r * 16 + n0]);
            const float4* __restrict__ bq = sB + np * SLOTS + sl * SEGQ;
            const float4* __restrict__ cq = sC + np * SLOTS + sl * SEGQ;
            // ---- F1: decay factors, local end state ----
            float2 a2[T];
            float2 hend = make_float2(0.f, 0.f);
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
            const float2 st = *reinterpret_cast<const float2*>(&sSt[r * 16 + n0]);
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
            float2* carry = reinterpret_cast<float2*>(&sCarryD[r * 16 + n0]);
            const float2 Xw = *carry;
            float2 dh = fma2(Ee, Xw, De);
            __syncwarp();
            if (sl == 0) *carry = fma2(E2, Xw, dl);
            // ---- R2: true dh_t and the gradient terms ----
            const float2 A2r = mul2(A2, make_float2(kLn2, kLn2));  // un-scaled A
            float2 dA2 = make_float2(0.f, 0.f);
            // the warps that share this pair set have finished reading every sRed of the previous pair (deferred second barrier)
            if (GW > 1 && np > sp * NPW) named_bar_sync<1 + (SS > 1 ? GW : 0)>(SS > 1 ? sp : 0, 32 * GW);
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
                    sRed[r * K::RED_RS + sl * (T + 1) + tt] = make_float4(vB.x, vB.y, vC.x, vC.y);
                }
            }
            // dA: reduce over the warp's segments, accumulate in smem (single writer per (row, n))
#pragma unroll
            for (int o = RB; o < 32; o <<= 1) {
                dA2.x += __shfl_xor_sync(0xffffffffu, dA2.x, o);
                dA2.y += __shfl_xor_sync(0xffffffffu, dA2.y, o);
            }
            if (sl == 0) {
                float2* da = reinterpret_cast<float2*>(&sdA[r * 16 + n0]);
                *da = add2(*da, dA2);
            }
            __syncwarp();
            if (GW > 1) {
                // dB/dC: the GW warps of the CTA that work on this pair set (different rows of the same group) meet, then each sums
                // the RB * GW rows of its share of the cells: ONE vector reduction per (pair, position, CTA) instead of one per warp
                // (the global reductions were 19-25 % of the kernel, DESIGN §1.2)
                named_bar_sync<1 + (SS > 1 ? GW : 0)>(SS > 1 ? sp : 0, 32 * GW);
                constexpr int CPW = K::CELLS / GW;
#pragma unroll
                for (int i = lane; i < CPW; i += 32) {
                    const int cell = rs * CPW + i;
                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    float2 acc_b = make_float2(0.f, 0.f), acc_c = make_float2(0.f, 0.f);
#pragma unroll
                    for (int w = 0; w < GW; ++w) {
                        const float4* src = reinterpret_cast<const float4*>(after_tile + (size_t)(w * SS + sp) * K::warp_bytes) + (cell / T) * (T + 1) + cell % T;
#pragma unroll
                        for (int j = 0; j < RB; ++j) {
                            const float4 v = src[j * K::RED_RS];
                            acc_b = add2(acc_b, make_float2(v.x, v.y));
                            acc_c = add2(acc_c, make_float2(v.z, v.w));
                        }
                    }
                    acc = make_float4(acc_b.x, acc_b.y, acc_c.x, acc_c.y);
                    const int l = c0 + cell;
                    if (l < L && n0 < N) put_bc<DET>(scratch + (int64_t)np * L + l, acc);
                }
            } else {
                // dB/dC: sum the RB rows of each (segment, position) cell, one vector reduction per cell
#pragma unroll
                for (int cell = lane; cell < K::CELLS; cell += 32) {
                    const float4* src = sRed + (cell / T) * (T + 1) + cell % T;
                    float4 acc = src[0];
#pragma unroll
                    for (int j = 1; j < RB; ++j) {
                        const float4 v = src[j * K::RED_RS];
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    }
                    const int l = c0 + cell;
                    if (l < L && n0 < N) put_bc<DET>(scratch + (int64_t)np * L + l, acc);
                }
                __syncwarp();
            }
        }

        if (SS > 1) {  // sums over the states handled by the other warps of this row slot
            float* pp = spart + (size_t)rs * (SS - 1) * 2 * T * 32;
            if (sp > 0) {
#pragma unroll
                for (int t = 0; t < T; ++t) {
                    pp[(((sp - 1) * 2 + 0) * T + t) * 32 + lane] = s1[t];
                    pp[(((sp - 1) * 2 + 1) * T + t) * 32 + lane] = s2[t];
                }
            }
            named_bar_sync<1>(rs, 32 * SS);
            if (sp > 0) continue;
#pragma unroll
            for (int s = 0; s < SS - 1; ++s)
#pragma unroll
                for (int t = 0; t < T; ++t) {
                    s1[t] += pp[((s * 2 + 0) * T + t) * 32 + lane];
                    s2[t] += pp[((s * 2 + 1) * T + t) * 32 + lane];
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
        if (!GRP || !rev) {
#pragma unroll
            for (int v = 0; v < T / V; ++v) {
                store_vec<in_t>(durow + l0 + v * V, duo + v * V, valid - v * V, true);
                store_vec<in_t>(ddrow + l0 + v * V, ddo + v * V, valid - v * V, true);
            }
        } else if (valid == T) {  // sequence l0+t -> memory L-1-l0-t: one reversed contiguous block
#pragma unroll
            for (int v = 0; v < T / V; ++v) {
                float ur[V], dr[V];
#pragma unroll
                for (int i = 0; i < V; ++i) {
                    ur[i] = duo[T - 1 - (v * V + i)];
                    dr[i] = ddo[T - 1 - (v * V + i)];
                }
                store_vec<in_t>(durow + (L - l0 - T) + v * V, ur, V, true);
                store_vec<in_t>(ddrow + (L - l0 - T) + v * V, dr, V, true);
            }
        } else {
#pragma unroll
            for (int t = 0; t < T; ++t)
                if (t < valid) {
                    durow[L - 1 - l0 - t] = from_f32<in_t>(duo[t]);
                    ddrow[L - 1 - l0 - t] = from_f32<in_t>(ddo[t]);
                }
        }
    }
    // ---- per-row parameter gradients ----
#pragma unroll
    for (int o = RB; o < 32; o <<= 1) {
        dD_acc += __shfl_xor_sync(0xffffffffu, dD_acc, o);
        dbias_acc += __shfl_xor_sync(0xffffffffu, dbias_acc, o);
    }
    if (sl == 0 && sp == 0) {
        if constexpr (DET) {
            if (p.dD) p.dD[(int64_t)b * p.dim + d] = dD_acc;
            if (p.dbias) p.dbias[(int64_t)b * p.dim + d] = dbias_acc;
        } else {
            if (p.dD) atomicAdd(p.dD + d, dD_acc);
            if (p.dbias) atomicAdd(p.dbias + d, dbias_acc);
        }
    }
    __syncwarp();
    for (int i = lane; i < RB * 2 * NPW; i += 32) {
        const int rr = i / (2 * NPW), n = sp * 2 * NPW + i % (2 * NPW);
        if constexpr (DET) {
            if (n < N) p.dA[((int64_t)b * p.dim + d0 + rr) * N + n] = sdA[rr * 16 + n];
        } else {
            if (n < N) atomicAdd(p.dA + (int64_t)(d0 + rr) * N + n, sdA[rr * 16 + n]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------- host
template <typename in_t, int RB, int SS, bool GRP, typename g_t, bool DET>
static int launch_bt3(const ScanBwdParams& p, const BwdMaps<GRP>& maps, cudaStream_t stream) {
    using K = BwdTmaCfg<in_t, RB, SS, g_t>;
    auto kern = scan_bwd_tma_kernel<in_t, RB, SS, GRP, g_t, DET>;
    constexpr size_t smem = K::smem_bytes + 128;
    static_assert(sizeof(in_t) == 4 ? smem <= 227 * 1024 : smem <= 113 * 1024, "scan_bwd_tma: two CTAs per SM (one for fp32 I/O)");
    VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long blocks = (long)p.batch * (p.dim / K::ROWS);
    VMB_CUDA(launch_pdl(kern, dim3((unsigned)blocks), dim3(128), smem, stream, p, maps));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

template <typename in_t, int RB, bool GRP, typename g_t, bool DET>
static int launch_bt2(const ScanBwdParams& p, const BwdMaps<GRP>& maps, int ss, cudaStream_t stream) {
    switch (ss) {
        case 4: return launch_bt3<in_t, RB, 4, GRP, g_t, DET>(p, maps, stream);
        case 2: return launch_bt3<in_t, RB, 2, GRP, g_t, DET>(p, maps, stream);
        default: return launch_bt3<in_t, RB, 1, GRP, g_t, DET>(p, maps, stream);
    }
}

template <typename in_t, bool GRP, typename g_t = in_t>
static int launch_bt1(const ScanBwdParams& p, const BwdMaps<GRP>& maps, int ss, cudaStream_t stream, bool det = false) {
    // rows per warp: 2 (scan_bwd_tma_pick)
    return det ? launch_bt2<in_t, 2, GRP, g_t, true>(p, maps, ss, stream) : launch_bt2<in_t, 2, GRP, g_t, false>(p, maps, ss, stream);
}

// state split at RB = 2: the 255-register kernel keeps 2 CTAs x 4 warps per SM resident (2 x SMs CTAs per wave)
static int bwd_tma_ss(const ScanBwdParams& p, int rb) {
    const long rows = (long)p.batch * p.dim;
    int ss = 1;
    while (ss < 4 && rows / (rb * 4 / ss) * 2 <= 2L * num_sms()) ss <<= 1;
    return ss;
}

// (rows per warp, state split): RB = 2 at every batch; the state split while the CTAs still fit one resident wave
// (DESIGN §1.2)
bool scan_bwd_tma_pick(const ScanBwdParams& p, int& rb, int& ss) {
    if (!p.vec_ok || p.npad != 16 || p.L < 512 || p.ckpt == nullptr) return false;
    rb = 2;
    ss = bwd_tma_ss(p, rb);
    return p.rows_per_group % (rb * 4 / ss) == 0;
}

int scan_bwd_tma_launch(const ScanBwdParams& p, int dtype, int rb, int ss, cudaStream_t stream, bool dout_f32, bool det) {
    ScanBwdTmaMapsN<1> maps;
    const uint32_t chunk = 32 / rb * T, rows = rb * 4 / ss;
    const uint32_t box_io[4] = {chunk, rows, 1, 1}, box_bc[4] = {chunk, 16, 1, 1};
    const uint64_t dio[4] = {(uint64_t)p.L, (uint64_t)p.dim, 1, (uint64_t)p.batch};
    const uint64_t dbc[4] = {(uint64_t)p.L, (uint64_t)p.N, (uint64_t)p.G, (uint64_t)p.batch};
    const int64_t su[3] = {p.u_ds, 0, p.u_bs}, sd[3] = {p.dl_ds, 0, p.dl_bs}, sg[3] = {p.do_ds, 0, p.do_bs};
    const int64_t sb[3] = {p.B_ns, p.B_gs, p.B_bs}, sc[3] = {p.C_ns, p.C_gs, p.C_bs};
    int rc;
    if ((rc = make_tmap_4d(&maps.u[0], dtype, p.u, dio, su, box_io)) != VMB_OK) return rc;
    if ((rc = make_tmap_4d(&maps.d[0], dtype, p.delta, dio, sd, box_io)) != VMB_OK) return rc;
    if ((rc = make_tmap_4d(&maps.g[0], dout_f32 ? VMB_F32 : dtype, p.dout, dio, sg, box_io)) != VMB_OK) return rc;
    if ((rc = make_tmap_4d(&maps.b[0], dtype, p.Bm, dbc, sb, box_bc)) != VMB_OK) return rc;
    if ((rc = make_tmap_4d(&maps.c[0], dtype, p.Cm, dbc, sc, box_bc)) != VMB_OK) return rc;
    if (dout_f32) {  // fp32 dout against 16-bit inputs: a dout tile twice as wide (+4 / 2 / 1 KB at SS = 1 / 2 / 4), still two CTAs
                     // per SM (static_assert in launch_bt3)
        switch (dtype) {
            case VMB_BF16: return launch_bt1<__nv_bfloat16, false, float>(p, maps, ss, stream, det);
            case VMB_F16: return launch_bt1<__half, false, float>(p, maps, ss, stream, det);
        }
        set_error("selective_scan_bwd: fp32 dout needs bf16 / fp16 inputs (dtype %d)", dtype);
        return VMB_ERR_INVALID;
    }
    switch (dtype) {
        case VMB_F32: return launch_bt1<float, false>(p, maps, ss, stream, det);  // 130 KB of tiles: one CTA per SM
        case VMB_BF16: return launch_bt1<__nv_bfloat16, false>(p, maps, ss, stream, det);
        case VMB_F16: return launch_bt1<__half, false>(p, maps, ss, stream, det);
    }
    set_error("selective_scan_bwd: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

// scratch [b][g][npad/2][L][4] fp32 (sequence order) -> every group's dB, dC (B,N,L) in the I/O dtype, in that group's memory order
template <typename in_t>
__global__ void scan_bwd_finalize_grouped_kernel(const float4* __restrict__ scratch, const ScanBwdGroups gr, int N, int L, long total) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over (b, g, np, l)
    if (i >= total) return;
    const int l = (int)(i % L);
    const long t = i / L;
    const int np = (int)(t % 8);
    const long bg = t / 8;
    const int g = (int)(bg % gr.ndesc);
    const int64_t b = bg / gr.ndesc;
    const ScanBwdGroupDesc& gd = gr.grp[g];
    const int m = gd.rev ? L - 1 - l : l;
    in_t* __restrict__ dB = reinterpret_cast<in_t*>(gd.dB) + b * gr.dB_bs + m;
    in_t* __restrict__ dC = reinterpret_cast<in_t*>(gd.dC) + b * gr.dC_bs + m;
    const float4 v = scratch[i];
    const int n0 = 2 * np;
    if (n0 < N) {
        dB[n0 * gr.dB_ns] = from_f32<in_t>(v.x);
        dC[n0 * gr.dC_ns] = from_f32<in_t>(v.z);
    }
    if (n0 + 1 < N) {
        dB[(n0 + 1) * gr.dB_ns] = from_f32<in_t>(v.y);
        dC[(n0 + 1) * gr.dC_ns] = from_f32<in_t>(v.w);
    }
}

template <typename in_t>
static int launch_grouped_det_t(const ScanBwdParams& p, const ScanBwdTmaMapsG& maps, int ss, int dtype, cudaStream_t stream) {
    ScanBwdParams q = p;
    const ScanBwdDetFin f = scan_bwd_det_carve(q, p.rows_per_group / (2 * 4 / ss));
    int rc = launch_bt1<in_t, true>(q, maps, ss, stream, true);
    if (rc != VMB_OK) return rc;
    return scan_bwd_det_finalize(f, &maps.gr, dtype, stream);
}

template <typename in_t>
static int launch_grouped_t(const ScanBwdParams& p, const ScanBwdTmaMapsG& maps, int ss, cudaStream_t stream) {
    int rc = launch_bt1<in_t, true>(p, maps, ss, stream);
    if (rc != VMB_OK) return rc;
    const long total = (long)p.batch * p.G * (p.npad / 2) * p.L;
    scan_bwd_finalize_grouped_kernel<in_t><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(p.dBC), maps.gr,
                                                                                                 p.N, p.L, total);
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

// the grouped mode always runs the TMA kernel (any seqlen: tails and the reversed walk's underflow are zero-filled boxes); the state
// split grows until the CTA's rows divide the group
static int grouped_ss(const ScanBwdParams& p) {
    int ss = bwd_tma_ss(p, 2);
    while (ss < 4 && p.rows_per_group % (2 * 4 / ss)) ss <<= 1;
    return ss;
}

int64_t scan_bwd_grouped_det_workspace(const ScanBwdParams& p) {
    const int ss = grouped_ss(p);
    if (p.rows_per_group % (2 * 4 / ss)) return -1;
    return scan_bwd_det_bytes(p, p.rows_per_group / (2 * 4 / ss));
}

int scan_bwd_grouped_launch(const ScanBwdParams& p, const ScanBwdGroups& gr, int dtype, cudaStream_t stream, bool det) {
    VMB_CHECK(gr.ndesc == p.G && p.G >= 1 && p.G <= 4 && p.vec_ok && p.npad == 16, "selective_scan_bwd_grouped: needs 16 B-aligned rows and dstate <= 16");
    const int rb = 2;
    const int ss = grouped_ss(p);
    VMB_CHECK(p.rows_per_group % (rb * 4 / ss) == 0, "selective_scan_bwd_grouped: rows per group (%d) must be even", p.rows_per_group);
    ScanBwdTmaMapsG maps;
    maps.gr = gr;
    const uint32_t chunk = 32 / rb * T, rows = rb * 4 / ss;
    const uint32_t box_io[4] = {chunk, rows, 1, 1}, box_bc[4] = {chunk, 16, 1, 1};
    const uint64_t dio[4] = {(uint64_t)p.L, (uint64_t)p.rows_per_group, 1, (uint64_t)p.batch};
    const uint64_t dbc[4] = {(uint64_t)p.L, (uint64_t)p.N, 1, (uint64_t)p.batch};
    const int64_t su[3] = {p.u_ds, 0, p.u_bs}, sd[3] = {p.dl_ds, 0, p.dl_bs}, sg[3] = {p.do_ds, 0, p.do_bs};
    const int64_t sb[3] = {p.B_ns, 0, p.B_bs}, sc[3] = {p.C_ns, 0, p.C_bs};
    for (int g = 0; g < gr.ndesc; ++g) {
        const ScanBwdGroupDesc& gd = gr.grp[g];
        int rc;
        if ((rc = make_tmap_4d(&maps.u[g], dtype, gd.u, dio, su, box_io)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.d[g], dtype, gd.delta, dio, sd, box_io)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.g[g], dtype, gd.dout, dio, sg, box_io)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.b[g], dtype, gd.Bm, dbc, sb, box_bc)) != VMB_OK) return rc;
        if ((rc = make_tmap_4d(&maps.c[g], dtype, gd.Cm, dbc, sc, box_bc)) != VMB_OK) return rc;
    }
    if (det) {  // no memset: every partial slot is written
        switch (dtype) {
            case VMB_F32: return launch_grouped_det_t<float>(p, maps, ss, dtype, stream);
            case VMB_BF16: return launch_grouped_det_t<__nv_bfloat16>(p, maps, ss, dtype, stream);
            case VMB_F16: return launch_grouped_det_t<__half>(p, maps, ss, dtype, stream);
        }
        set_error("selective_scan_bwd_grouped: unsupported dtype %d", dtype);
        return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaMemsetAsync(p.dBC, 0, sizeof(float4) * (size_t)p.batch * p.G * (p.npad / 2) * p.L, stream));
    switch (dtype) {
        case VMB_F32: return launch_grouped_t<float>(p, maps, ss, stream);
        case VMB_BF16: return launch_grouped_t<__nv_bfloat16>(p, maps, ss, stream);
        case VMB_F16: return launch_grouped_t<__half>(p, maps, ss, stream);
    }
    set_error("selective_scan_bwd_grouped: unsupported dtype %d", dtype);
    return VMB_ERR_INVALID;
}

}  // namespace vmb
