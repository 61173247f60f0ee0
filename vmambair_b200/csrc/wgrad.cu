// Weight gradient of the 1x1 convs of the OSS block: dW[m][k] = sum_{b,p} dY[b][m][p] * X[b][k][p]  (training path, SURVEY.md 8 a15).
// Both operands are pixel-contiguous (B, rows, L) activations, i.e. the reduction dimension is the contiguous one of BOTH -- the
// "TN" case: A = dY (M x P row-major), B = X^T given as (K x P row-major).  K <= 384 and M <= ~2 k while P = B*L is 16 k - 260 k, so the
// kernel is split over pixels: CTA (m-tile 64, k-tile 64, pixel range), mma.sync m16n8k16 (bf16 / fp16 in, fp32 accumulate) from
// cp.async double-buffered [64 rows][32 pixels] tiles, fp32 atomicAdd of the 64 x 64 partial into dW (the caller zero-fills).
// Tensor cores are the right unit here (a dense contraction) but the shape is tiny and reduction-dominated: the legacy mma.sync
// path is used on purpose -- a wgmma pipeline needs 64-row warpgroup tiles and a persistent set-up that these short launches cannot amortise.
#include "common.cuh"
#include "train_params.h"

namespace vmb {

constexpr int WG_TM = 64, WG_TN = 64, WG_PK = 32;  // output tile, pixels per stage
constexpr int WG_PITCH = WG_PK + 8;                // +16 B: conflict-free ldmatrix rows

__device__ __forceinline__ void wg_cp16(void* smem_dst, const void* gsrc, int src_bytes) {
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void wg_ldsm4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
    const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
template <typename in_t> __device__ __forceinline__ void wg_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void wg_mma<__nv_bfloat16>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void wg_mma<__half>(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// grid (m tiles, k tiles, batch * splits); 128 threads: warp w owns the 32 x 32 quadrant (w/2, w%2) of the tile
template <typename in_t>
__global__ void __launch_bounds__(128) wgrad_mma_kernel(const WgradParams p) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) in_t sA[2][WG_TM][WG_PITCH];
    __shared__ __align__(16) in_t sX[2][WG_TN][WG_PITCH];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * WG_TM, k0 = blockIdx.y * WG_TN;
    const int b = blockIdx.z / p.splits, sp = blockIdx.z % p.splits;
    const int per = ((p.L + p.splits - 1) / p.splits + WG_PK - 1) / WG_PK * WG_PK;  // pixels of one split (multiple of the stage)
    const int p_lo = sp * per, p_hi = min(p.L, p_lo + per);
    if (p_lo >= p_hi) return;
    const in_t* __restrict__ dy = reinterpret_cast<const in_t*>(p.dy) + (int64_t)b * p.dy_bs;
    const in_t* __restrict__ x = reinterpret_cast<const in_t*>(p.x) + (int64_t)b * p.x_bs;

    auto stage = [&](int buf, int pp) {  // rows beyond M / K and pixels beyond the split are zero-filled
#pragma unroll
        for (int it = tid; it < WG_TM * (WG_PK / 8); it += 128) {
            const int row = it / (WG_PK / 8), c = (it % (WG_PK / 8)) * 8;
            const int m = m0 + row, px = pp + c;
            const int nbytes = (m < p.M && px < p_hi) ? min(16, (p_hi - px) * 2) : 0;
            wg_cp16(&sA[buf][row][c], nbytes > 0 ? (const void*)(dy + (int64_t)m * p.dy_cs + px) : (const void*)dy, nbytes);
        }
#pragma unroll
        for (int it = tid; it < WG_TN * (WG_PK / 8); it += 128) {
            const int row = it / (WG_PK / 8), c = (it % (WG_PK / 8)) * 8;
            const int k = k0 + row, px = pp + c;
            const int nbytes = (k < p.K && px < p_hi) ? min(16, (p_hi - px) * 2) : 0;
            wg_cp16(&sX[buf][row][c], nbytes > 0 ? (const void*)(x + (int64_t)k * p.x_cs + px) : (const void*)x, nbytes);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    const bool do_bias = p.dbias != nullptr && blockIdx.y == 0;
    float bsum = 0.f;

    stage(0, p_lo);
    int buf = 0;
    for (int pp = p_lo; pp < p_hi; pp += WG_PK, buf ^= 1) {
        if (pp + WG_PK < p_hi) {
            stage(buf ^ 1, pp + WG_PK);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        if (do_bias) {  // row sums of dY (the bias gradient): thread t sums half a row of the staged tile
            float f[8];
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                unpack8<in_t>(*reinterpret_cast<const uint4*>(&sA[buf][tid >> 1][(tid & 1) * 16 + v * 8]), f);
#pragma unroll
                for (int e = 0; e < 8; ++e) bsum += f[e];
            }
        }
#pragma unroll
        for (int ks = 0; ks < WG_PK; ks += 16) {
            uint32_t a[2][4], bq[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
                wg_ldsm4(a[i][0], a[i][1], a[i][2], a[i][3], &sA[buf][wm + i * 16 + (lane & 15)][ks + (lane >> 4) * 8]);
#pragma unroll
            for (int j = 0; j < 2; ++j)
                wg_ldsm4(bq[j][0], bq[j][1], bq[j][2], bq[j][3],
                         &sX[buf][wn + j * 16 + (lane & 7) + ((lane >> 4) << 3)][ks + ((lane >> 3) & 1) * 8]);
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    wg_mma<in_t>(acc[i][2 * j], a[i], bq[j][0], bq[j][1]);
                    wg_mma<in_t>(acc[i][2 * j + 1], a[i], bq[j][2], bq[j][3]);
                }
        }
        __syncthreads();
    }
    if (do_bias) {
        bsum += __shfl_xor_sync(0xffffffffu, bsum, 1);
        const int m = m0 + (tid >> 1);
        if ((tid & 1) == 0 && m < p.M) atomicAdd(p.dbias + m, bsum);
    }
    float* __restrict__ out = p.out + (p.per_batch ? (int64_t)b * p.M * p.K : 0);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = m0 + wm + i * 16 + (lane >> 2) + (e >> 1) * 8;
                const int k = k0 + wn + j * 8 + (lane & 3) * 2 + (e & 1);
                if (m < p.M && k < p.K) atomicAdd(out + (int64_t)m * p.K + k, acc[i][j][e]);
            }
}

int wgrad_launch(const WgradParams& p, int dtype, cudaStream_t stream) {
    dim3 grid((p.M + WG_TM - 1) / WG_TM, (p.K + WG_TN - 1) / WG_TN, p.B * p.splits);
    VMB_CHECK(grid.y <= 65535 && grid.z <= 65535, "wgrad: grid too large");
    switch (dtype) {
        case VMB_BF16: VMB_CUDA(launch_pdl(wgrad_mma_kernel<__nv_bfloat16>, grid, dim3(128), 0, stream, p)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(wgrad_mma_kernel<__half>, grid, dim3(128), 0, stream, p)); break;
        default: set_error("wgrad: 16-bit activations only (fp32 goes to the library GEMM)"); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb

using namespace vmb;

extern "C" int vmb_pixlin_wgrad(const vmb_wgrad_args* a, void* stream) {
    VMB_CHECK(a && a->dy && a->x && a->out, "pixlin_wgrad: null pointer");
    VMB_CHECK(a->dtype == VMB_BF16 || a->dtype == VMB_F16, "pixlin_wgrad: bf16 / fp16 activations only");
    VMB_CHECK(a->batch > 0 && a->M > 0 && a->K > 0 && a->L > 0, "pixlin_wgrad: bad sizes");
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    VMB_CHECK(al16(a->dy) && al16(a->x) && a->dy_bs % 8 == 0 && a->dy_cs % 8 == 0 && a->x_bs % 8 == 0 && a->x_cs % 8 == 0,
              "pixlin_wgrad: rows must be 16 B aligned (L %% 8 == 0)");
    WgradParams p{a->dy, a->x, a->out, a->batch, a->M, a->K, a->L, a->dy_bs, a->dy_cs, a->x_bs, a->x_cs, 1, a->per_batch, a->dbias};
    // pixel splits: enough CTAs for ~2 waves, at least 512 pixels per CTA
    const long tiles = (long)((a->M + WG_TM - 1) / WG_TM) * ((a->K + WG_TN - 1) / WG_TN) * a->batch;
    int splits = (int)((2 * num_sms() + tiles - 1) / tiles);
    const int max_splits = (a->L + 511) / 512;
    p.splits = splits < 1 ? 1 : (splits > max_splits ? max_splits : splits);
    return wgrad_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}
