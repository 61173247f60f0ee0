// The Real-ESRGAN degradation operators of basicsr (filter2D, USMSharp, DiffJPEG(differentiable=False), the Gaussian and Poisson
// noise of random_add_*_noise_pt) as fp32 NCHW kernels, for synthesising training pairs on the device (vmambair_b200.degradations).
// Nothing here reads the host: per-image JPEG quality, noise levels and draws are device tensors, so a whole degradation chain is
// launched without a synchronisation.  Reflect and zero pads are index arithmetic; every tile and its halo is staged in shared memory.
#include <math.h>

#include "common.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxK = 51;

// torch's 'reflect' pad of index i in [0, n) (valid for a pad < n), then clamped: taps beyond the pad only meet zero weights, and
// outputs beyond the image are not stored
__device__ __forceinline__ int reflect_idx(int i, int n) {
    i = i < 0 ? -i : i;
    i = i >= n ? 2 * (n - 1) - i : i;
    return min(max(i, 0), n - 1);
}

// torch's CUDA division of a float32 tensor by a Python number: a multiplication by the float32 reciprocal
constexpr float kInv255 = 1.f / 255.f, kInv100 = 1.f / 100.f;

// torch.clamp((v * 255.0).round(), 0, 255) / 255. in float32, rounding half to even
__device__ __forceinline__ float quant255(float v) { return __fmul_rn(fminf(fmaxf(rintf(__fmul_rn(v, 255.f)), 0.f), 255.f), kInv255); }

// ---- filter2D: k x k cross-correlation, reflect pads of k / 2 ----
// One CTA: a 64 x 16 output tile of one plane; each thread 4 horizontally adjacent outputs.  The kernel rows are zero-padded to kp (a
// multiple of 4), so a row is kp / 4 float4 weights and the thread slides an 8-value window of float4 tile loads along it.
constexpr int kFW = 64, kFH = 16;

size_t filter2d_smem_bytes(int k, int kp) { return (size_t)(k * kp + (kFH + k - 1) * (kFW + kp)) * sizeof(float); }

__global__ void __launch_bounds__(kThreads) filter2d_kernel(const vmb_filter2d_args a, int kp) {
    extern __shared__ float4 smem4[];
    pdl_trigger();
    pdl_wait();
    const int k = a.k, r = k / 2, sw = kFW + kp, sh = kFH + k - 1;
    float* ks = reinterpret_cast<float*>(smem4);  // [k][kp]
    float* tile = ks + k * kp;                    // [sh][sw]
    const int plane = blockIdx.z, b = plane / a.channels;
    const float* kern = a.kernel + (a.per_image ? (int64_t)b * k * k : 0);
    for (int i = threadIdx.x; i < k * kp; i += kThreads) {
        const int row = i / kp, col = i % kp;
        ks[i] = col < k ? kern[row * k + col] : 0.f;
    }
    const int x0 = blockIdx.x * kFW - r, y0 = blockIdx.y * kFH - r;
    const float* src = a.img + (int64_t)plane * a.H * a.W;
    for (int i = threadIdx.x; i < sh * sw; i += kThreads) {
        const int ty = i / sw, tx = i % sw;
        tile[i] = __ldg(src + (int64_t)reflect_idx(y0 + ty, a.H) * a.W + reflect_idx(x0 + tx, a.W));
    }
    __syncthreads();
    const int tx = (threadIdx.x % (kFW / 4)) * 4, ty = threadIdx.x / (kFW / 4);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < k; ++i) {
        const float4* row = reinterpret_cast<const float4*>(tile + (ty + i) * sw + tx);
        const float4* kr = reinterpret_cast<const float4*>(ks + i * kp);
        float4 cur = row[0];
        for (int jc = 0; jc < kp / 4; ++jc) {
            const float4 nxt = row[jc + 1], w4 = kr[jc];
            const float win[8] = {cur.x, cur.y, cur.z, cur.w, nxt.x, nxt.y, nxt.z, nxt.w};
            const float w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[q] = fmaf(win[q + jj], w[jj], acc[q]);
            cur = nxt;
        }
    }
    const int gy = blockIdx.y * kFH + ty;
    if (gy >= a.H) return;
    float* dst = a.out + (int64_t)plane * a.H * a.W + (int64_t)gy * a.W;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int gx = blockIdx.x * kFW + tx + q;
        if (gx < a.W) dst[gx] = a.quantize_out ? quant255(acc[q]) : acc[q];
    }
}

// ---- USMSharp: the separable Gaussian, a row pass then a column pass over a 32 x 32 tile and its halo ----
// pass 0: blur = G * img; residual = img - blur; workspace = (|residual| 255 > threshold); out = clip(img + weight residual, 0, 1)
// pass 1: soft = G * workspace; out = soft out + (1 - soft) img
constexpr int kUT = 32, kUIn = kUT + kMaxK - 1;

__global__ void __launch_bounds__(kThreads) usm_kernel(const vmb_usm_sharp_args a, int pass) {
    __shared__ float in[kUIn * kUIn];  // [kUT + k - 1][kUT + k - 1]
    __shared__ float hp[kUIn * kUT];   // [kUT + k - 1][kUT]: the row pass
    pdl_trigger();
    pdl_wait();
    const int k = a.k, r = k / 2, n = kUT + k - 1;
    const int64_t poff = (int64_t)blockIdx.z * a.H * a.W;
    const float* src = (pass == 0 ? a.img : a.workspace) + poff;
    const int x0 = blockIdx.x * kUT - r, y0 = blockIdx.y * kUT - r;
    for (int i = threadIdx.x; i < n * n; i += kThreads)
        in[i] = src[(int64_t)reflect_idx(y0 + i / n, a.H) * a.W + reflect_idx(x0 + i % n, a.W)];
    __syncthreads();
    for (int i = threadIdx.x; i < n * kUT; i += kThreads) {
        const int row = i / kUT, col = i % kUT;
        float s = 0.f;
        for (int j = 0; j < k; ++j) s = fmaf(in[row * n + col + j], a.taps[j], s);
        hp[i] = s;
    }
    __syncthreads();
    const int tx = threadIdx.x % kUT, ty = (threadIdx.x / kUT) * 4, gx = blockIdx.x * kUT + tx;
    if (gx >= a.W) return;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int gy = blockIdx.y * kUT + ty + q;
        if (gy >= a.H) break;
        float s = 0.f;
        for (int i = 0; i < k; ++i) s = fmaf(hp[(ty + q + i) * kUT + tx], a.taps[i], s);
        const int64_t o = poff + (int64_t)gy * a.W + gx;
        const float x = a.img[o];
        if (pass == 0) {
            const float res = __fsub_rn(x, s);
            a.workspace[o] = __fmul_rn(fabsf(res), 255.f) > a.threshold ? 1.f : 0.f;
            a.out[o] = fminf(fmaxf(__fadd_rn(x, __fmul_rn(a.weight, res)), 0.f), 1.f);
        } else {
            a.out[o] = __fadd_rn(__fmul_rn(s, a.out[o]), __fmul_rn(__fsub_rn(1.f, s), x));
        }
    }
}

// ---- DiffJPEG(differentiable=False) ----
// One CTA: a 16 x 64 strip of four 16 x 16 MCUs of one image (zero beyond H x W, as the reference's bottom / right pad).  Its 24 8 x 8
// blocks (16 Y, 4 Cb, 4 Cr) live in shared memory through colour conversion, 4:2:0 averaging, the separable DCT, quantisation, the
// inverse DCT and the conversion back; the strip is read once and written once.
constexpr int kJW = 64, kJH = 16, kJBlocks = 24;

// ITU-T T.81 Annex K tables K.1 (luma) and K.2's top-left 4 x 4 (chroma, 99 elsewhere), as printed: row v, column u.  basicsr stores
// both transposed (T[u][v] = Q[v][u], u the row frequency of the coefficient), and that is what is applied here.
__constant__ float kQY[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                              14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                              18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                              49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
__constant__ float kQC4[16] = {17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 99, 47, 66, 99, 99};

__device__ __forceinline__ float qtable(bool luma, int u, int v) {
    if (luma) return kQY[v * 8 + u];
    return u < 4 && v < 4 ? kQC4[v * 4 + u] : 99.f;
}

// quality_to_factor on a float32 element, as basicsr evaluates it on its quality tensor
__device__ __forceinline__ float jpeg_factor(float q) {
    return __fmul_rn(q < 50.f ? __fdiv_rn(5000.f, q) : __fsub_rn(200.f, __fmul_rn(q, 2.f)), kInv100);
}

__global__ void __launch_bounds__(kThreads) jpeg_kernel(const vmb_jpeg_args a) {
    __shared__ float blk[kJBlocks * 64];     // [block][row][col]: pixels - 128, then coefficients, then pixels - 128 again
    __shared__ float tmp[kJBlocks * 64];     // the separable passes' intermediate
    __shared__ float chroma[2][kJH][kJW];    // full-resolution Cb, Cr
    __shared__ float cosv[64];               // cosv[x * 8 + u] = alpha(u) / 2 cos((2x + 1) u pi / 16): D = C^T P C, P = C D C^T
    pdl_trigger();
    pdl_wait();
    const int tid = threadIdx.x, b = blockIdx.z;
    if (tid < 64) {
        const int x = tid / 8, u = tid % 8;
        cosv[tid] = (float)(cospi((2 * x + 1) * u / 16.0) * (u == 0 ? 0.35355339059327373 : 0.5));
    }
    const float factor = a.quality ? jpeg_factor(a.quality[b]) : a.factor;
    const int64_t hw = (int64_t)a.H * a.W;
    const float* src = a.img + (int64_t)b * 3 * hw;
    const int y0 = blockIdx.y * kJH, x0 = blockIdx.x * kJW;
    // load, x 255, RGB -> YCbCr
    for (int i = tid; i < kJH * kJW; i += kThreads) {
        const int row = i / kJW, col = i % kJW, gy = y0 + row, gx = x0 + col;
        float c[3] = {0.f, 0.f, 0.f};
        if (gy < a.H && gx < a.W) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                float v = src[ch * hw + (int64_t)gy * a.W + gx];
                if (a.clamp_in) v = fminf(fmaxf(v, 0.f), 1.f);
                c[ch] = v * 255.f;
            }
        }
        const float Y = 0.299f * c[0] + 0.587f * c[1] + 0.114f * c[2];
        chroma[0][row][col] = -0.168736f * c[0] - 0.331264f * c[1] + 0.5f * c[2] + 128.f;
        chroma[1][row][col] = 0.5f * c[0] - 0.418688f * c[1] - 0.081312f * c[2] + 128.f;
        blk[((row / 8) * 8 + col / 8) * 64 + (row % 8) * 8 + col % 8] = Y - 128.f;
    }
    __syncthreads();
    // 2 x 2 chroma averages -> blocks 16 + 4 c + j
    for (int i = tid; i < 2 * 8 * 32; i += kThreads) {
        const int c = i / 256, row = (i % 256) / 32, col = i % 32;
        const float s = chroma[c][2 * row][2 * col] + chroma[c][2 * row][2 * col + 1] + chroma[c][2 * row + 1][2 * col] +
                        chroma[c][2 * row + 1][2 * col + 1];
        blk[(16 + 4 * c + col / 8) * 64 + row * 8 + col % 8] = s * 0.25f - 128.f;
    }
    __syncthreads();
    // DCT: tmp[x][v] = sum_y P[x][y] C[y][v]; D[u][v] = sum_x C[x][u] tmp[x][v]; quantise and dequantise in place
    for (int i = tid; i < kJBlocks * 64; i += kThreads) {
        const float* p = blk + (i / 64) * 64 + (i % 64) / 8 * 8;
        const int v = i % 8;
        float s = 0.f;
#pragma unroll
        for (int y = 0; y < 8; ++y) s = fmaf(p[y], cosv[y * 8 + v], s);
        tmp[i] = s;
    }
    __syncthreads();
    for (int i = tid; i < kJBlocks * 64; i += kThreads) {
        const int bi = i / 64, u = (i % 64) / 8, v = i % 8;
        const float* t = tmp + bi * 64 + v;
        float d = 0.f;
#pragma unroll
        for (int x = 0; x < 8; ++x) d = fmaf(cosv[x * 8 + u], t[x * 8], d);
        const float step = qtable(bi < 16, u, v) * factor;
        // a zero step (quality 100) is the lossless limit of rint(d / step) step
        blk[i] = step != 0.f ? rintf(d / step) * step : d;
    }
    __syncthreads();
    // inverse DCT: tmp[x][v] = sum_u C[x][u] D[u][v]; P[x][y] = sum_v tmp[x][v] C[y][v]
    for (int i = tid; i < kJBlocks * 64; i += kThreads) {
        const int bi = i / 64, x = (i % 64) / 8, v = i % 8;
        const float* d = blk + bi * 64 + v;
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) s = fmaf(cosv[x * 8 + u], d[u * 8], s);
        tmp[i] = s;
    }
    __syncthreads();
    for (int i = tid; i < kJBlocks * 64; i += kThreads) {
        const float* t = tmp + (i / 64) * 64 + (i % 64) / 8 * 8;
        const int y = i % 8;
        float s = 0.f;
#pragma unroll
        for (int v = 0; v < 8; ++v) s = fmaf(t[v], cosv[y * 8 + v], s);
        blk[i] = s;
    }
    __syncthreads();
    // YCbCr -> RGB (chroma repeated 2 x 2), clamp to [0, 255], / 255, crop
    float* dst = a.out + (int64_t)b * 3 * hw;
    for (int i = tid; i < kJH * kJW; i += kThreads) {
        const int row = i / kJW, col = i % kJW, gy = y0 + row, gx = x0 + col;
        if (gy >= a.H || gx >= a.W) continue;
        const float Y = blk[((row / 8) * 8 + col / 8) * 64 + (row % 8) * 8 + col % 8] + 128.f;
        const int ci = (col / 16) * 64 + (row / 2) * 8 + (col / 2) % 8;
        const float cb = blk[16 * 64 + ci], cr = blk[20 * 64 + ci];  // (Cb + 128) - 128
        const float rgb[3] = {Y + 1.402f * cr, Y - 0.344136f * cb - 0.714136f * cr, Y + 1.772f * cb};
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            float v = __fmul_rn(fminf(fmaxf(rgb[ch], 0.f), 255.f), kInv255);
            dst[ch * hw + (int64_t)gy * a.W + gx] = a.quantize_out ? quant255(v) : v;
        }
    }
}

// ---- noise ----
// the level (0..255) of clamp(rint(v 255), 0, 255), and torchvision's rgb_to_grayscale with torch's separate float32 roundings
__device__ __forceinline__ float gray_of(float r, float g, float b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}
__device__ __forceinline__ int level_of(float v) { return (int)fminf(fmaxf(rintf(__fmul_rn(v, 255.f)), 0.f), 255.f); }
// 2^ceil(log2(count)) of the levels present in a 256-bit mask
__device__ __forceinline__ float vals_of(const uint32_t* mask) {
    int n = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) n += __popc(mask[w]);
    return n <= 1 ? 1.f : (float)(1u << (32 - __clz(n - 1)));
}

// masks[b][0 | 1][8]: the levels present in image b (RGB | gray), OR-ed per CTA in shared memory, then into global memory
__global__ void __launch_bounds__(kThreads) levels_kernel(const vmb_noise_levels_args a) {
    __shared__ uint32_t m[16];
    pdl_trigger();
    pdl_wait();
    if (threadIdx.x < 16) m[threadIdx.x] = 0u;
    __syncthreads();
    const int b = blockIdx.y;
    const int64_t hw = (int64_t)a.H * a.W;
    const float* src = a.img + (int64_t)b * 3 * hw;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < hw; i += (int64_t)gridDim.x * kThreads) {
        const float r = src[i], g = src[hw + i], bl = src[2 * hw + i];
        const int lr = level_of(r), lg = level_of(g), lb = level_of(bl), ly = level_of(gray_of(r, g, bl));
        atomicOr(&m[lr / 32], 1u << (lr % 32));
        atomicOr(&m[lg / 32], 1u << (lg % 32));
        atomicOr(&m[lb / 32], 1u << (lb % 32));
        atomicOr(&m[8 + ly / 32], 1u << (ly % 32));
    }
    __syncthreads();
    uint32_t* masks = reinterpret_cast<uint32_t*>(a.workspace) + 16 * b;
    if (threadIdx.x < 16 && m[threadIdx.x]) atomicOr(&masks[threadIdx.x], m[threadIdx.x]);
}

// rates = q vals, rates_gray = q_gray vals_gray; vals[b], vals_gray[b]
__global__ void __launch_bounds__(kThreads) rates_kernel(const vmb_noise_levels_args a) {
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.y;
    const uint32_t* masks = reinterpret_cast<const uint32_t*>(a.workspace) + 16 * b;
    const float vals = vals_of(masks), valsg = vals_of(masks + 8);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.vals[b] = vals;
        a.vals_gray[b] = valsg;
    }
    const int64_t hw = (int64_t)a.H * a.W;
    const float* src = a.img + (int64_t)b * 3 * hw;
    float* rates = a.rates + (int64_t)b * 3 * hw;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < hw; i += (int64_t)gridDim.x * kThreads) {
        const float r = src[i], g = src[hw + i], bl = src[2 * hw + i];
        rates[i] = __fmul_rn(quant255(r), vals);
        rates[hw + i] = __fmul_rn(quant255(g), vals);
        rates[2 * hw + i] = __fmul_rn(quant255(bl), vals);
        a.rates_gray[(int64_t)b * hw + i] = __fmul_rn(quant255(gray_of(r, g, bl)), valsg);
    }
}

__global__ void __launch_bounds__(kThreads) noise_apply_kernel(const vmb_noise_apply_args a) {
    pdl_trigger();
    pdl_wait();
    const int64_t hw = (int64_t)a.H * a.W, chw = a.channels * hw, n = a.batch * chw;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const int b = (int)(i / chw);
        const int64_t p = i % hw;
        const float param = __fadd_rn(__fmul_rn(a.u_param[b], a.param_span), a.param_lo);
        const float g = a.u_gray[b] < a.gray_prob ? 1.f : 0.f;
        const float x = a.img[i];
        float noise, noise_g;
        if (a.kind == VMB_NOISE_GAUSSIAN) {  // randn sigma / 255
            noise = __fmul_rn(__fmul_rn(a.noise[i], param), kInv255);
            noise_g = __fmul_rn(__fmul_rn(a.noise_gray[p], param), kInv255);
        } else {                             // poisson(q vals) / vals - q, RGB and gray
            const float* px = a.img + (int64_t)b * chw + p;
            noise = __fsub_rn(__fdiv_rn(a.noise[i], a.vals[b]), quant255(x));
            noise_g = __fsub_rn(__fdiv_rn(a.noise_gray[(int64_t)b * hw + p], a.vals_gray[b]), quant255(gray_of(px[0], px[hw], px[2 * hw])));
        }
        float v = __fadd_rn(__fmul_rn(noise, __fsub_rn(1.f, g)), __fmul_rn(noise_g, g));
        if (a.kind == VMB_NOISE_POISSON) v = __fmul_rn(v, param);
        v = __fadd_rn(x, v);
        if (a.clip && a.rounds) v = quant255(v);
        else if (a.clip) v = fminf(fmaxf(v, 0.f), 1.f);
        else if (a.rounds) v = __fmul_rn(rintf(__fmul_rn(v, 255.f)), kInv255);
        a.out[i] = v;
    }
}

unsigned grid_1d(int64_t n, int64_t cap) {
    const int64_t g = (n + kThreads - 1) / kThreads;
    return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace

}  // namespace vmb

using namespace vmb;

static int check_planes(const float* img, const float* out, int batch, int channels, int H, int W, const char* who) {
    VMB_CHECK(img && out, "%s: null image or output", who);
    VMB_CHECK(batch > 0 && channels > 0 && (int64_t)batch * channels < 65536 && H > 0 && W > 0,
              "%s: bad batch %d, channels %d or size %d x %d", who, batch, channels, H, W);
    return VMB_OK;
}

static int check_taps(int k, int H, int W, const char* who) {
    VMB_CHECK(k % 2 == 1 && k >= 1 && k <= kMaxK, "%s: kernel size %d must be odd and at most %d", who, k, kMaxK);
    VMB_CHECK(H > k / 2 && W > k / 2, "%s: a %d x %d image is too small for the reflect pad %d of a %d x %d kernel", who, H, W, k / 2, k, k);
    return VMB_OK;
}

extern "C" int vmb_filter2d(const vmb_filter2d_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->kernel, "filter2d: null pointer");
    int st = check_planes(a->img, a->out, a->batch, a->channels, a->H, a->W, "filter2d");
    if (st == VMB_OK) st = check_taps(a->k, a->H, a->W, "filter2d");
    if (st != VMB_OK) return st;
    const int kp = (a->k + 3) / 4 * 4;
    const dim3 grid((unsigned)cdiv(a->W, kFW), (unsigned)cdiv(a->H, kFH), (unsigned)(a->batch * a->channels));
    VMB_CHECK(grid.y < 65536, "filter2d: image too tall (%d rows)", a->H);
    VMB_CUDA(launch_pdl(filter2d_kernel, grid, dim3(kThreads), filter2d_smem_bytes(a->k, kp), static_cast<cudaStream_t>(stream), *a, kp));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_usm_sharp(const vmb_usm_sharp_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->workspace, "usm_sharp: null pointer");
    int st = check_planes(a->img, a->out, a->batch, a->channels, a->H, a->W, "usm_sharp");
    if (st == VMB_OK) st = check_taps(a->k, a->H, a->W, "usm_sharp");
    if (st != VMB_OK) return st;
    VMB_CHECK(a->out != a->img && a->workspace != a->img && a->workspace != a->out, "usm_sharp: img, out and workspace must not alias");
    const dim3 grid((unsigned)cdiv(a->W, kUT), (unsigned)cdiv(a->H, kUT), (unsigned)(a->batch * a->channels));
    VMB_CHECK(grid.y < 65536, "usm_sharp: image too tall (%d rows)", a->H);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    VMB_CUDA(launch_pdl(usm_kernel, grid, dim3(kThreads), 0, s, *a, 0));
    VMB_CUDA(launch_pdl(usm_kernel, grid, dim3(kThreads), 0, s, *a, 1));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_jpeg(const vmb_jpeg_args* a, void* stream) {
    VMB_CHECK(a != nullptr, "jpeg: null pointer");
    const int st = check_planes(a->img, a->out, a->batch, 3, a->H, a->W, "jpeg");
    if (st != VMB_OK) return st;
    const dim3 grid((unsigned)cdiv(a->W, kJW), (unsigned)cdiv(a->H, kJH), (unsigned)a->batch);
    VMB_CHECK(grid.y < 65536, "jpeg: image too tall (%d rows)", a->H);
    VMB_CUDA(launch_pdl(jpeg_kernel, grid, dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_noise_levels(const vmb_noise_levels_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->rates && a->rates_gray && a->vals && a->vals_gray && a->workspace, "noise_levels: null pointer");
    const int st = check_planes(a->img, a->rates, a->batch, 3, a->H, a->W, "noise_levels");
    if (st != VMB_OK) return st;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d((int64_t)a->H * a->W, 2 * num_sms()), (unsigned)a->batch);
    VMB_CUDA(cudaMemsetAsync(a->workspace, 0, (size_t)a->batch * 16 * sizeof(uint32_t), s));
    VMB_CUDA(launch_pdl(levels_kernel, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(launch_pdl(rates_kernel, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_noise_apply(const vmb_noise_apply_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->noise && a->noise_gray && a->u_param && a->u_gray, "noise_apply: null pointer");
    VMB_CHECK(a->kind == VMB_NOISE_GAUSSIAN || a->kind == VMB_NOISE_POISSON, "noise_apply: unknown kind %d", a->kind);
    VMB_CHECK(a->kind == VMB_NOISE_GAUSSIAN || (a->channels == 3 && a->vals && a->vals_gray),
              "noise_apply: Poisson noise takes 3 channels and the levels of vmb_noise_levels");
    const int st = check_planes(a->img, a->out, a->batch, a->channels, a->H, a->W, "noise_apply");
    if (st != VMB_OK) return st;
    const int64_t n = (int64_t)a->batch * a->channels * a->H * a->W;
    VMB_CUDA(launch_pdl(noise_apply_kernel, dim3(grid_1d(n, 8 * num_sms())), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
