// PSNR and SSIM of the reference's metric code (Deraining/basicsr/metrics/psnr_ssim.py, Deraining/Deraining/utils.py) on the device.
// Sources are decoded in the loads (dtype, tensor2img quantisation, channel order, the Y channel: metric_src.cuh); nothing
// intermediate is written.  Every sum is deterministic: per-CTA partials in a fixed order, then one CTA per image adds them in
// index order (no floating-point atomics), so a result depends on the image size only, never on scheduling.
#include <math.h>

#include "metric_src.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;
constexpr int kPsnrItems = 8;               // pixels per thread a PSNR CTA aims at (its grid is sized from H W only)
constexpr int kPsnrMaxBlocks = 1024;        // per image
constexpr int kTW = 32, kTH = 16, kR = 5;   // SSIM output tile (x, y) and the window's radius
constexpr int kInW = kTW + 2 * kR, kInH = kTH + 2 * kR;

// the value a metric sees at plane c of pixel (b, y, x): the source value, or (plane 0) its Y
__device__ __forceinline__ double metric_val(const vmb_metric_src& s, int channels, int y_channel, int b, int y, int x, int c) {
    if (!y_channel) return load_val(s, b, y, x, c);
    if (channels == 1) return (double)y_gray(load_val(s, b, y, x, 0));
    return (double)y_bgr(load_val(s, b, y, x, 0), load_val(s, b, y, x, 1), load_val(s, b, y, x, 2));
}

// fixed-order block reductions (every thread gets the result)
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x / 32); ++w) s += red[w];
    return s;
}

__device__ __forceinline__ double block_max(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double m = -INFINITY;
    for (int w = 0; w < (int)(blockDim.x / 32); ++w) m = fmax(m, red[w]);
    return m;
}

// ---- to_y_channel ----
__global__ void __launch_bounds__(kThreads) to_y_kernel(const vmb_to_y_args a) {
    pdl_trigger();
    pdl_wait();
    const int64_t hw = (int64_t)a.H * a.W, i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= hw) return;
    const int b = blockIdx.y, y = (int)(i / a.W), x = (int)(i % a.W);
    a.out[b * hw + i] = (float)metric_val(a.src, a.channels, 1, b, y, x, 0);
}

// ---- PSNR ----
int psnr_blocks(int H, int W) {
    const int64_t per = kThreads * kPsnrItems, n = ((int64_t)H * W + per - 1) / per;
    return (int)(n < kPsnrMaxBlocks ? n : kPsnrMaxBlocks);
}

// partials[b][blk] = (sum of squared differences, max of img1) over pixels blk * 256 + tid + k * gridDim.x * 256
__global__ void __launch_bounds__(kThreads) psnr_partial_kernel(const vmb_psnr_args a) {
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.y;
    const int64_t hw = (int64_t)a.H * a.W;
    double sse = 0.0, mx = -INFINITY;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < hw; i += (int64_t)gridDim.x * kThreads) {
        const int y = (int)(i / a.W), x = (int)(i % a.W);
        if (a.y_channel) {
            const float v1 = (float)metric_val(a.img1, a.channels, 1, b, y, x, 0);
            const float d = __fsub_rn(v1, (float)metric_val(a.img2, a.channels, 1, b, y, x, 0));
            sse += (double)__fmul_rn(d, d);
            mx = fmax(mx, (double)v1);
        } else {
            for (int c = 0; c < a.channels; ++c) {
                const double v1 = load_val(a.img1, b, y, x, c), d = __dsub_rn(v1, load_val(a.img2, b, y, x, c));
                sse += __dmul_rn(d, d);
                mx = fmax(mx, v1);
            }
        }
    }
    sse = block_sum(sse, red);
    mx = block_max(mx, red);
    if (threadIdx.x == 0) {
        double* p = reinterpret_cast<double*>(a.workspace) + 2 * ((int64_t)b * gridDim.x + blockIdx.x);
        p[0] = sse;
        p[1] = mx;
    }
}

__global__ void __launch_bounds__(kThreads) psnr_final_kernel(const vmb_psnr_args a, int nblk) {
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x;
    const double* p = reinterpret_cast<const double*>(a.workspace) + 2 * (int64_t)b * nblk;
    double sse = 0.0, mx = -INFINITY;
    for (int i = threadIdx.x; i < nblk; i += kThreads) {
        sse += p[2 * i];
        mx = fmax(mx, p[2 * i + 1]);
    }
    sse = block_sum(sse, red);
    mx = block_max(mx, red);
    if (threadIdx.x == 0) {
        const double n = (double)a.H * a.W * (a.y_channel ? 1 : a.channels);
        const double mse = __ddiv_rn(sse, n), m = mx <= 1.0 ? 1.0 : 255.0;
        a.mse[b] = mse;
        a.max_value[b] = mx;
        a.psnr[b] = mse == 0.0 ? INFINITY : 20.0 * log10(m / sqrt(mse));
    }
}

// ---- SSIM ----
__device__ __forceinline__ double ssim_px(double mu1, double mu2, double xx, double yy, double xy, double C1, double C2) {
    // ((2 mu1 mu2 + C1)(2 s12 + C2)) / ((mu1^2 + mu2^2 + C1)(s1 + s2 + C2)), each operation rounded as numpy's
    const double m11 = __dmul_rn(mu1, mu1), m22 = __dmul_rn(mu2, mu2), m12 = __dmul_rn(mu1, mu2);
    const double s1 = __dsub_rn(xx, m11), s2 = __dsub_rn(yy, m22), s12 = __dsub_rn(xy, m12);
    const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, m12), C1), __dadd_rn(__dmul_rn(2.0, s12), C2));
    const double den = __dmul_rn(__dadd_rn(__dadd_rn(m11, m22), C1), __dadd_rn(__dadd_rn(s1, s2), C2));
    return __ddiv_rn(num, den);
}

// One CTA: a kTH x kTW tile of the SSIM map of image blockIdx.z.  The tile and its halo of every plane of both images are staged in
// shared memory once (indices clamped: replicated borders; in VALID mode every kept output's window lies inside the image).  Then, per
// output channel c, a horizontal 11-tap pass of the five moments goes to shared memory and a vertical pass to registers.  REPLICATE3D
// filters across the channels as well; that filter is linear, so it folds into the horizontal pass: plane p's terms (x, y, x^2, y^2, xy)
// enter channel c's moments with weight mix[c][p].  partials[b][c][tile] = the tile's map sum of channel c.
__host__ __device__ constexpr size_t ssim_smem_bytes(int planes) { return (2 * planes * kInH * kInW + 5 * kInH * kTW) * sizeof(double); }

__global__ void __launch_bounds__(kThreads, 2) ssim_tile_kernel(const vmb_ssim_args a, int OH, int OW) {
    extern __shared__ double smem[];
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int planes = a.y_channel ? 1 : a.channels;
    double* in1 = smem;                               // [planes][kInH][kInW]
    double* in2 = in1 + planes * kInH * kInW;         // [planes][kInH][kInW]
    double* hm = in2 + planes * kInH * kInW;          // [5][kInH][kTW]
    const int b = blockIdx.z, tx = threadIdx.x % kTW, ty = threadIdx.x / kTW;  // ty in [0, 8): output rows ty and ty + 8
    const int off = a.mode == VMB_SSIM_VALID ? kR : 0;                        // output (oy, ox) is centred on (oy + off, ox + off)
    const int y0 = blockIdx.y * kTH + off - kR, x0 = blockIdx.x * kTW + off - kR;
    const bool mix3d = a.mode == VMB_SSIM_REPLICATE3D;
    const double m = mix3d && a.max_value[b] <= 1.0 ? 1.0 : 255.0;
    const double C1 = __dmul_rn(__dmul_rn(0.01, m), __dmul_rn(0.01, m)), C2 = __dmul_rn(__dmul_rn(0.03, m), __dmul_rn(0.03, m));
    for (int i = threadIdx.x; i < planes * kInH * kInW; i += kThreads) {
        const int p = i / (kInH * kInW), j = i % (kInH * kInW);
        const int y = min(max(y0 + j / kInW, 0), a.H - 1), x = min(max(x0 + j % kInW, 0), a.W - 1);
        in1[i] = metric_val(a.img1, a.channels, a.y_channel, b, y, x, p);
        in2[i] = metric_val(a.img2, a.channels, a.y_channel, b, y, x, p);
    }
    const int64_t tiles = (int64_t)gridDim.x * gridDim.y, t = (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
    for (int c = 0; c < planes; ++c) {
        __syncthreads();  // staging done; the previous channel's vertical pass is done with hm
        const int p0 = mix3d ? 0 : c, p1 = mix3d ? planes : c + 1;
        for (int i = threadIdx.x; i < kInH * kTW; i += kThreads) {
            const int r = i / kTW, col = i % kTW;
            double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
            for (int p = p0; p < p1; ++p) {
                const double* u1 = in1 + (p * kInH + r) * kInW + col;
                const double* u2 = in2 + (p * kInH + r) * kInW + col;
                double h[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
                for (int k = 0; k < 2 * kR + 1; ++k) {
                    const double u = u1[k], v = u2[k], w = a.taps[k];
                    h[0] = fma(w, u, h[0]);
                    h[1] = fma(w, v, h[1]);
                    h[2] = fma(w, __dmul_rn(u, u), h[2]);
                    h[3] = fma(w, __dmul_rn(v, v), h[3]);
                    h[4] = fma(w, __dmul_rn(u, v), h[4]);
                }
                const double w = mix3d ? a.mix[c * planes + p] : 1.0;
#pragma unroll
                for (int q = 0; q < 5; ++q) s[q] = fma(w, h[q], s[q]);
            }
#pragma unroll
            for (int q = 0; q < 5; ++q) hm[(q * kInH + r) * kTW + col] = s[q];
        }
        __syncthreads();
        double part = 0.0;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int row = ty + 8 * r;
            double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < 2 * kR + 1; ++k)
#pragma unroll
                for (int q = 0; q < 5; ++q) s[q] = fma(a.taps[k], hm[(q * kInH + row + k) * kTW + tx], s[q]);
            if (blockIdx.y * kTH + row < OH && blockIdx.x * kTW + tx < OW) part += ssim_px(s[0], s[1], s[2], s[3], s[4], C1, C2);
        }
        part = block_sum(part, red);
        if (threadIdx.x == 0) reinterpret_cast<double*>(a.workspace)[((int64_t)b * planes + c) * tiles + t] = part;
    }
}

// ssim[b]: per channel, the tile sums in index order over the map size; VALID: the channels' mean of those; otherwise the mean over
// every channel's map
__global__ void __launch_bounds__(kThreads) ssim_final_kernel(const vmb_ssim_args a, int64_t tiles, int64_t n) {
    __shared__ double red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, planes = a.y_channel ? 1 : a.channels;
    const double* p = reinterpret_cast<const double*>(a.workspace) + (int64_t)b * planes * tiles;
    double mean = 0.0, total = 0.0;
    for (int c = 0; c < planes; ++c) {
        double s = 0.0;
        for (int64_t i = threadIdx.x; i < tiles; i += kThreads) s += p[c * tiles + i];
        s = block_sum(s, red);
        mean += s / (double)n;
        total += s;
    }
    if (threadIdx.x == 0)
        a.ssim[b] = a.mode == VMB_SSIM_VALID ? mean / planes : total / ((double)n * planes);
}

void ssim_map_size(const vmb_ssim_args& a, int& OH, int& OW) {
    OH = a.mode == VMB_SSIM_VALID ? max(a.H - 2 * kR, 0) : a.H;
    OW = a.mode == VMB_SSIM_VALID ? max(a.W - 2 * kR, 0) : a.W;
}

int64_t ssim_tiles(const vmb_ssim_args& a) {
    int OH, OW;
    ssim_map_size(a, OH, OW);
    return (int64_t)cdiv(OW, kTW) * cdiv(OH, kTH);
}

}  // namespace

}  // namespace vmb

using namespace vmb;

static int check_pair(const vmb_metric_src& s1, const vmb_metric_src& s2, int batch, int H, int W, int channels, int y_channel,
                      const char* who) {
    VMB_CHECK(metric_src_ok(s1) && metric_src_ok(s2), "%s: null image or unknown source dtype (%d, %d)", who, s1.dtype, s2.dtype);
    VMB_CHECK(batch > 0 && batch < 65536 && H > 0 && W > 0 && (channels == 1 || channels == 3) && (y_channel == 0 || y_channel == 1),
              "%s: bad batch %d, size %d x %d, channels %d (1 or 3) or y_channel %d", who, batch, H, W, channels, y_channel);
    return VMB_OK;
}

extern "C" int vmb_to_y_channel(const vmb_to_y_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->out, "to_y_channel: null pointer");
    const int st = check_pair(a->src, a->src, a->batch, a->H, a->W, a->channels, 1, "to_y_channel");
    if (st != VMB_OK) return st;
    const dim3 grid((unsigned)(((int64_t)a->H * a->W + kThreads - 1) / kThreads), (unsigned)a->batch);
    VMB_CHECK(grid.x < (1u << 31), "to_y_channel: image too large");
    VMB_CUDA(launch_pdl(to_y_kernel, grid, dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int64_t vmb_psnr_workspace_bytes(const vmb_psnr_args* a) {
    return a == nullptr || a->batch <= 0 || a->H <= 0 || a->W <= 0 ? 0 : (int64_t)a->batch * psnr_blocks(a->H, a->W) * 2 * sizeof(double);
}

extern "C" int vmb_psnr(const vmb_psnr_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->mse && a->max_value && a->psnr && a->workspace, "psnr: null pointer");
    const int st = check_pair(a->img1, a->img2, a->batch, a->H, a->W, a->channels, a->y_channel, "psnr");
    if (st != VMB_OK) return st;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int nblk = psnr_blocks(a->H, a->W);
    VMB_CUDA(launch_pdl(psnr_partial_kernel, dim3((unsigned)nblk, (unsigned)a->batch), dim3(kThreads), 0, s, *a));
    VMB_CUDA(launch_pdl(psnr_final_kernel, dim3((unsigned)a->batch), dim3(kThreads), 0, s, *a, nblk));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int64_t vmb_ssim_workspace_bytes(const vmb_ssim_args* a) {
    if (a == nullptr || a->batch <= 0 || a->H <= 0 || a->W <= 0) return 0;
    return (int64_t)a->batch * (a->y_channel ? 1 : a->channels) * ssim_tiles(*a) * (int64_t)sizeof(double);
}

extern "C" int vmb_ssim(const vmb_ssim_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->ssim, "ssim: null pointer");
    const int st = check_pair(a->img1, a->img2, a->batch, a->H, a->W, a->channels, a->y_channel, "ssim");
    if (st != VMB_OK) return st;
    VMB_CHECK(a->mode == VMB_SSIM_VALID || a->mode == VMB_SSIM_REPLICATE || a->mode == VMB_SSIM_REPLICATE3D, "ssim: unknown mode %d", a->mode);
    VMB_CHECK(a->mode != VMB_SSIM_REPLICATE || a->y_channel || a->channels == 1, "ssim: REPLICATE takes one channel (y_channel or gray)");
    VMB_CHECK(a->mode != VMB_SSIM_REPLICATE3D || a->max_value, "ssim: REPLICATE3D needs max_value");
    int OH, OW;
    ssim_map_size(*a, OH, OW);
    const int64_t tiles = ssim_tiles(*a);
    VMB_CHECK(tiles == 0 || a->workspace, "ssim: null workspace");
    VMB_CHECK(cdiv(OH, kTH) < 65536, "ssim: image too tall (%d rows)", a->H);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (tiles > 0) {
        const size_t smem = ssim_smem_bytes(a->y_channel ? 1 : a->channels);
        VMB_CUDA(cudaFuncSetAttribute(ssim_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssim_smem_bytes(3)));
        const dim3 grid((unsigned)cdiv(OW, kTW), (unsigned)cdiv(OH, kTH), (unsigned)a->batch);
        VMB_CUDA(launch_pdl(ssim_tile_kernel, grid, dim3(kThreads), smem, s, *a, OH, OW));
    }
    VMB_CUDA(launch_pdl(ssim_final_kernel, dim3((unsigned)a->batch), dim3(kThreads), 0, s, *a, tiles, (int64_t)OH * OW));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
