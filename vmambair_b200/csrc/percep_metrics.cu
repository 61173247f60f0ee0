// The perceptual metrics LPIPS (VGG, version 0.1) and DISTS between their VGG16 convolutions (vmambair_b200.lpips, .dists): the
// input preparation of both images of each pair into one 2B batch, one kernel per feature layer (LPIPS: the per-pixel channel norms
// and the weighted squared difference of the normalised features; DISTS: the per-channel sums in fp64 and the L2 pooling that feeds
// the next convolution), and the per-image result in one CTA.  The ReLUs and max-pools between the convolutions are
// vmb_percep_stage (perceptual.cu).  Every partial has one writer and every sum one fixed order: no atomics, bitwise reproducible.
// Nothing reads the host.
#include <math.h>

#include "common.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;       // prep, DISTS layer and final kernels
constexpr int kTargetCtas = 2048;   // CTAs a statistics layer is split into (over all planes), when it has the items
constexpr int kLpGroups = 16;       // LPIPS layer: warps per CTA, each holding C / 16 channels of 32 pixels
constexpr int kLpThreads = 32 * kLpGroups;

__device__ __forceinline__ float relu(float v) { return v > 0.f ? v : 0.f; }

// sum of v over the CTA in one fixed order (butterfly within each warp, then thread 0 adds the warp sums in index order); the result
// is valid in thread 0.  `red` holds blockDim.x / 32 values.
template <typename T>
__device__ T block_sum(T v, T* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = v;
    __syncthreads();
    T s = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)blockDim.x / 32; ++w) s += red[w];
    return s;
}

// the five statistics of one tile, block-summed and written by thread 0 to st[0..4]
__device__ void write_stats(const double (&acc)[5], double* red, double* st) {
#pragma unroll
    for (int s = 0; s < 5; ++s) {
        const double v = block_sum(acc[s], red);
        if (threadIdx.x == 0) st[s] = v;
    }
}

__device__ __forceinline__ void add_stats(double (&acc)[5], float f0, float f1) {
    const double d0 = f0, d1 = f1;
    acc[0] += d0;
    acc[1] += d1;
    acc[2] += d0 * d0;
    acc[3] += d1 * d1;
    acc[4] += d0 * d1;
}

int64_t tiles_of(int planes, int64_t items) {
    const int64_t need = (items + kThreads - 1) / kThreads;
    int64_t cap = (kTargetCtas + planes - 1) / planes;
    cap = cap > 1 ? cap : 1;
    const int64_t t = need < cap ? need : cap;
    return t > 1 ? t : 1;
}

int lpips_ctas(int B, int H, int W) {
    const int64_t need = ((int64_t)H * W + 31) / 32;
    int64_t cap = (kTargetCtas + B - 1) / B;
    const int64_t t = need < cap ? need : cap;
    return (int)(t > 1 ? t : 1);
}

// ---- input: out[b] = prep(src[0] image b), out[B + b] = prep(src[1] image b); CTA (tile, c, b), DISTS statistics of the raw v ----
__device__ __forceinline__ float load_src(const vmb_pmetric_src& s, int64_t b, int c, int h, int w) {
    const int64_t o = b * s.stride[0] + c * s.stride[1] + h * s.stride[2] + w * s.stride[3];
    return s.u8 ? (float)static_cast<const uint8_t*>(s.data)[o] : static_cast<const float*>(s.data)[o];
}

__global__ void __launch_bounds__(kThreads) prep_kernel(const vmb_pmetric_prep_args a, const int tiles) {
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int t = blockIdx.x, c = blockIdx.y, b = blockIdx.z, W = a.W;
    const int64_t hw = (int64_t)a.H * W, per = (hw + tiles - 1) / tiles, p0 = t * per, p1 = p0 + per < hw ? p0 + per : hw;
    const float shift = a.shift[c], scale = a.scale[c];
    const bool lp = a.metric == VMB_PMETRIC_LPIPS;
    float* o0 = a.out + ((int64_t)b * 3 + c) * hw;
    float* o1 = a.out + ((int64_t)(a.B + b) * 3 + c) * hw;
    double acc[5] = {0., 0., 0., 0., 0.};
    for (int64_t p = p0 + threadIdx.x; p < p1; p += kThreads) {
        const int h = (int)(p / W), w = (int)(p % W);
        float v[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float x = load_src(a.src[i], b, c, h, w);
            if (a.src[i].u8) {
                x = __fdiv_rn(x, 255.f);                                  // astype(float32) / 255. ; ToTensor's div(255)
                if (lp) x = __fdiv_rn(__fsub_rn(x, 0.5f), 0.5f);          // normalize(mean=.5, std=.5)
            } else if (lp && a.normalize) {
                x = __fsub_rn(__fmul_rn(2.f, x), 1.f);                    // 2 * in0 - 1
            }
            v[i] = x;
        }
        if (a.stats) add_stats(acc, v[0], v[1]);
        o0[p] = __fdiv_rn(__fsub_rn(v[0], shift), scale);
        o1[p] = __fdiv_rn(__fsub_rn(v[1], shift), scale);
    }
    if (a.stats) write_stats(acc, red, a.stats + (((int64_t)b * 3 + c) * tiles + t) * 5);
}

// ---- LPIPS layer: CTA (i, b) takes pixel tiles i, i + gridDim.x, ... of image pair b; warp g holds channels [g K, (g + 1) K) of 32
// consecutive pixels (one per lane) of both images in registers, read once with the ReLU applied ----
template <int K>
__global__ void __launch_bounds__(kLpThreads) lpips_layer_kernel(const vmb_lpips_layer_args a) {
    __shared__ float r0[kLpGroups][32], r1[kLpGroups][32];
    pdl_trigger();
    pdl_wait();
    const int lane = threadIdx.x % 32, g = threadIdx.x / 32, b = blockIdx.y, C = kLpGroups * K;
    const int64_t hw = (int64_t)a.H * a.W, ntile = (hw + 31) / 32;
    const float* y0 = a.y + ((int64_t)b * C + g * K) * hw;
    const float* y1 = a.y + ((int64_t)(a.B + b) * C + g * K) * hw;
    const float* w = a.w + g * K;
    float acc = 0.f;
    for (int64_t tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
        const int64_t p = tile * 32 + lane;
        const bool in = p < hw;
        float f0[K], f1[K];
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            f0[k] = in ? relu(__ldg(y0 + k * hw + p)) : 0.f;
            f1[k] = in ? relu(__ldg(y1 + k * hw + p)) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            s0 = __fmaf_rn(f0[k], f0[k], s0);
            s1 = __fmaf_rn(f1[k], f1[k], s1);
        }
        r0[g][lane] = s0;
        r1[g][lane] = s1;
        __syncthreads();
        float n0 = 0.f, n1 = 0.f;
#pragma unroll
        for (int j = 0; j < kLpGroups; ++j) {
            n0 += r0[j][lane];
            n1 += r1[j][lane];
        }
        n0 = __fadd_rn(__fsqrt_rn(n0), 1e-10f);
        n1 = __fadd_rn(__fsqrt_rn(n1), 1e-10f);
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const float e = __fsub_rn(__fdiv_rn(f0[k], n0), __fdiv_rn(f1[k], n1));
            d = __fmaf_rn(w[k], __fmul_rn(e, e), d);
        }
        __syncthreads();  // every warp has read the norms
        r0[g][lane] = d;
        __syncthreads();
        if (g == 0) {
            float v = 0.f;
#pragma unroll
            for (int j = 0; j < kLpGroups; ++j) v += r0[j][lane];
            acc += v;
        }
        __syncthreads();
    }
    if (g == 0) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) a.partial[(int64_t)b * gridDim.x + blockIdx.x] = acc;
    }
}

__global__ void __launch_bounds__(kThreads) lpips_final_kernel(const vmb_lpips_final_args a) {
    __shared__ float red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    for (int b = 0; b < a.B; ++b) {
        float val = 0.f;
        for (int k = 0; k < a.layers; ++k) {
            const float* p = a.partial + a.offset[k] + (int64_t)b * a.ctas[k];
            float s = 0.f;
            for (int i = threadIdx.x; i < a.ctas[k]; i += kThreads) s += p[i];
            s = block_sum(s, red);
            if (threadIdx.x == 0) {
                const float r = __fdiv_rn(s, (float)a.hw[k]);
                a.layer[(int64_t)k * a.B + b] = r;
                val = __fadd_rn(val, r);
            }
        }
        if (threadIdx.x == 0) a.out[b] = val;
    }
}

// ---- DISTS layer: CTA (tile, c, b) takes a contiguous range of the 2 x 2 cells of plane c of both images of pair b ----
__global__ void __launch_bounds__(kThreads) dists_layer_kernel(const vmb_dists_layer_args a, const int tiles) {
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int t = blockIdx.x, c = blockIdx.y, b = blockIdx.z, H = a.H, W = a.W, Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    const int64_t cells = (int64_t)Ho * Wo, per = (cells + tiles - 1) / tiles, q0 = t * per, q1 = q0 + per < cells ? q0 + per : cells;
    const int64_t hw = (int64_t)H * W;
    const float* y0 = a.y + ((int64_t)b * a.C + c) * hw;
    const float* y1 = a.y + ((int64_t)(a.B + b) * a.C + c) * hw;
    const float tap[3] = {0.25f, 0.5f, 0.25f};
    double acc[5] = {0., 0., 0., 0., 0.};
    for (int64_t q = q0 + threadIdx.x; q < q1; q += kThreads) {
        const int i = (int)(q / Wo), j = (int)(q % Wo);
        float p0 = 0.f, p1 = 0.f;
#pragma unroll
        for (int di = 0; di < 3; ++di) {
            const int h = 2 * i - 1 + di;
            if (h < 0 || h >= H) continue;
#pragma unroll
            for (int dj = 0; dj < 3; ++dj) {
                const int x = 2 * j - 1 + dj;
                if (x < 0 || x >= W) continue;
                const int64_t o = (int64_t)h * W + x;
                const float f0 = relu(__ldg(y0 + o)), f1 = relu(__ldg(y1 + o));
                if (di > 0 && dj > 0) add_stats(acc, f0, f1);  // the cell's own pixels: rows 2i, 2i + 1, columns 2j, 2j + 1
                const float wt = __fmul_rn(tap[di], tap[dj]);
                p0 = __fmaf_rn(wt, __fmul_rn(f0, f0), p0);
                p1 = __fmaf_rn(wt, __fmul_rn(f1, f1), p1);
            }
        }
        if (a.pooled) {
            const int64_t ho = (int64_t)Ho * Wo;
            a.pooled[((int64_t)b * a.C + c) * ho + q] = __fsqrt_rn(__fadd_rn(p0, 1e-12f));
            a.pooled[((int64_t)(a.B + b) * a.C + c) * ho + q] = __fsqrt_rn(__fadd_rn(p1, 1e-12f));
        }
    }
    write_stats(acc, red, a.stats + (((int64_t)b * a.C + c) * tiles + t) * 5);
}

__global__ void __launch_bounds__(kThreads) dists_final_kernel(const vmb_dists_final_args a) {
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    int total = 0;
    for (int k = 0; k < a.layers; ++k) total += a.C[k];
    double wsum = 0.;
    for (int j = threadIdx.x; j < total; j += kThreads) wsum += (double)a.alpha[j] + (double)a.beta[j];
    wsum = block_sum(wsum, red);
    float mean = 0.f;
    for (int b = 0; b < a.B; ++b) {
        double num = 0.;
        for (int j = threadIdx.x; j < total; j += kThreads) {
            int k = 0, c = j;
            while (c >= a.C[k]) c -= a.C[k++];
            const double* st = a.stats + (a.offset[k] + ((int64_t)b * a.C[k] + c) * a.tiles[k]) * 5;
            double s[5] = {0., 0., 0., 0., 0.};
            for (int i = 0; i < a.tiles[k]; ++i)
#pragma unroll
                for (int e = 0; e < 5; ++e) s[e] += st[(int64_t)i * 5 + e];
            const double n = (double)a.n[k], m0 = s[0] / n, m1 = s[1] / n;
            const double v0 = s[2] / n - m0 * m0, v1 = s[3] / n - m1 * m1, cov = s[4] / n - m0 * m1;
            const double S1 = (2. * m0 * m1 + 1e-6) / (m0 * m0 + m1 * m1 + 1e-6);
            const double S2 = (2. * cov + 1e-6) / (v0 + v1 + 1e-6);
            num += (double)a.alpha[j] * S1 + (double)a.beta[j] * S2;
        }
        num = block_sum(num, red);
        if (threadIdx.x == 0) {
            const float sc = (float)(1. - num / wsum);
            a.score[b] = sc;
            mean += sc;
        }
    }
    if (threadIdx.x == 0 && a.mean) *a.mean = __fdiv_rn(mean, (float)a.B);
}

bool src_ok(const vmb_pmetric_src& s) { return s.data != nullptr && (s.u8 == 0 || s.u8 == 1); }

}  // namespace

}  // namespace vmb

using namespace vmb;

extern "C" int vmb_pmetric_tiles(int planes, int64_t items) {
    if (planes < 1 || items < 1) return -1;
    return (int)tiles_of(planes, items);
}

extern "C" int vmb_lpips_layer_ctas(int B, int H, int W) {
    if (B < 1 || H < 1 || W < 1) return -1;
    return lpips_ctas(B, H, W);
}

extern "C" int vmb_pmetric_prep(const vmb_pmetric_prep_args* a, void* stream) {
    VMB_CHECK(a != nullptr && src_ok(a->src[0]) && src_ok(a->src[1]) && a->shift && a->scale && a->out, "pmetric_prep: null pointer");
    VMB_CHECK(a->metric == VMB_PMETRIC_LPIPS || a->metric == VMB_PMETRIC_DISTS, "pmetric_prep: metric %d", a->metric);
    VMB_CHECK(a->B >= 1 && a->B <= 65535 && a->H >= 1 && a->W >= 1, "pmetric_prep: bad shape (%d x 3 x %d x %d)", a->B, a->H, a->W);
    VMB_CHECK(!a->stats || a->metric == VMB_PMETRIC_DISTS, "pmetric_prep: statistics are DISTS's");
    const int tiles = (int)tiles_of(3 * a->B, (int64_t)a->H * a->W);
    VMB_CUDA(launch_pdl(prep_kernel, dim3(tiles, 3, a->B), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a, tiles));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_lpips_layer(const vmb_lpips_layer_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->y && a->w && a->partial, "lpips_layer: null pointer");
    VMB_CHECK(a->B >= 1 && a->B <= 65535 && a->H >= 1 && a->W >= 1, "lpips_layer: bad shape");
    const int K = a->C / kLpGroups;
    VMB_CHECK(a->C % kLpGroups == 0 && (K == 4 || K == 8 || K == 16 || K == 32), "lpips_layer: %d channels (64, 128, 256 or 512)", a->C);
    const dim3 grid(lpips_ctas(a->B, a->H, a->W), a->B);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (K) {
        case 4: VMB_CUDA(launch_pdl(lpips_layer_kernel<4>, grid, dim3(kLpThreads), 0, s, *a)); break;
        case 8: VMB_CUDA(launch_pdl(lpips_layer_kernel<8>, grid, dim3(kLpThreads), 0, s, *a)); break;
        case 16: VMB_CUDA(launch_pdl(lpips_layer_kernel<16>, grid, dim3(kLpThreads), 0, s, *a)); break;
        default: VMB_CUDA(launch_pdl(lpips_layer_kernel<32>, grid, dim3(kLpThreads), 0, s, *a)); break;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_lpips_final(const vmb_lpips_final_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->partial && a->layer && a->out, "lpips_final: null pointer");
    VMB_CHECK(a->B >= 1 && a->layers >= 1 && a->layers <= VMB_PMETRIC_MAX_LAYERS, "lpips_final: %d images, %d layers", a->B, a->layers);
    for (int k = 0; k < a->layers; ++k) VMB_CHECK(a->ctas[k] >= 1 && a->hw[k] >= 1, "lpips_final: layer %d is empty", k);
    VMB_CUDA(launch_pdl(lpips_final_kernel, dim3(1), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_dists_layer(const vmb_dists_layer_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->y && a->stats, "dists_layer: null pointer");
    VMB_CHECK(a->B >= 1 && a->B <= 65535 && a->C >= 1 && a->C <= 65535 && a->H >= 1 && a->W >= 1, "dists_layer: bad shape");
    const int tiles = (int)tiles_of(a->B * a->C, (int64_t)((a->H + 1) / 2) * ((a->W + 1) / 2));
    VMB_CUDA(launch_pdl(dists_layer_kernel, dim3(tiles, a->C, a->B), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a, tiles));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_dists_final(const vmb_dists_final_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->stats && a->alpha && a->beta && a->score, "dists_final: null pointer");
    VMB_CHECK(a->B >= 1 && a->layers >= 1 && a->layers <= VMB_PMETRIC_MAX_LAYERS, "dists_final: %d images, %d layers", a->B, a->layers);
    for (int k = 0; k < a->layers; ++k)
        VMB_CHECK(a->C[k] >= 1 && a->tiles[k] >= 1 && a->n[k] >= 1 && a->offset[k] >= 0, "dists_final: layer %d is empty", k);
    VMB_CUDA(launch_pdl(dists_final_kernel, dim3(1), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
