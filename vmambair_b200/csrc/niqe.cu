// NIQE of the reference (Deraining/basicsr/metrics/niqe.py: calculate_niqe, niqe, compute_feature, estimate_aggd_param) on the
// device, in three launches per call (plus one per device that builds the r(gamma) table):
//   prep      the float32 plane (Y, gray or the value itself) cut to whole 96 x 96 blocks, and its float32 2 x 2 mean;
//   features  one CTA per block and scale: the MSCN values (7 x 7 filters summed in fp64, rounded once to float32, as scipy.ndimage
//             stores them), fp64 sums of the five distributions, the AGGD fits against the table, 18 features;
//   score     one CTA per image: column nanmean, covariance of the NaN-free rows, Cholesky solve with the pristine model.
// Every reduction runs in a fixed order (shuffle tree, then the warps in index order; the score's sums in block order), no atomics:
// results are bitwise reproducible and independent of the batch they are computed in.
#include <math.h>

#include "metric_src.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;
constexpr int kBlock = VMB_NIQE_BLOCK;  // block side at scale 1; kBlock / 2 at scale 2
constexpr int kR = 3;                   // the 7 x 7 window's radius
constexpr int kStats = 5;               // per distribution: negative count, sum x^2 over x < 0, positive count, sum x^2 over x > 0, sum |x|
constexpr int kDists = 5;               // the block, and its products with the block rolled by [0,1], [1,0], [1,1], [1,-1]
constexpr int kNF = VMB_NIQE_FEATURES;  // 36: 18 per scale
constexpr int kTable = VMB_NIQE_TABLE;

__host__ __device__ constexpr size_t feature_smem_bytes() {
    return ((kBlock + 2 * kR) * (kBlock + 2 * kR) + kBlock * kBlock) * sizeof(float);
}

// gam[i] of np.arange(0.2, 10.001, 0.001): numpy fills start + i * delta with delta = (start + step) - start
__device__ __forceinline__ double gam_at(int i) { return __dadd_rn(0.2, __dmul_rn((double)i, __dsub_rn(__dadd_rn(0.2, 0.001), 0.2))); }

// r_gam = gamma(2 / g)^2 / (gamma(1 / g) gamma(3 / g)) (estimate_aggd_param), one entry per thread
__global__ void __launch_bounds__(kThreads) niqe_table_kernel(double* table) {
    pdl_trigger();
    pdl_wait();
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= kTable) return;
    const double rec = __ddiv_rn(1.0, gam_at(i)), g2 = tgamma(__dmul_rn(rec, 2.0));
    table[i] = __ddiv_rn(__dmul_rn(g2, g2), __dmul_rn(tgamma(rec), tgamma(__dmul_rn(rec, 3.0))));
}

// the plane value of pixel (b, y, x) for the conversion `convert` (calculate_niqe's float32 cast, then to_y_channel, cv2's
// BGR2GRAY of img / 255. times 255., or nothing)
__device__ __forceinline__ float plane_val(const vmb_niqe_prep_args& a, int b, int y, int x) {
    if (a.convert == VMB_NIQE_PLANE) return __double2float_rn(load_val(a.src, b, y, x, 0));
    if (a.convert == VMB_NIQE_Y)
        return a.channels == 1 ? y_gray(load_val(a.src, b, y, x, 0))
                               : y_bgr(load_val(a.src, b, y, x, 0), load_val(a.src, b, y, x, 1), load_val(a.src, b, y, x, 2));
    const float xb = __fdiv_rn(__double2float_rn(load_val(a.src, b, y, x, 0)), 255.f),
                xg = __fdiv_rn(__double2float_rn(load_val(a.src, b, y, x, 1)), 255.f),
                xr = __fdiv_rn(__double2float_rn(load_val(a.src, b, y, x, 2)), 255.f);
    const float g = __fadd_rn(__fadd_rn(__fmul_rn(xb, 0.114f), __fmul_rn(xg, 0.587f)), __fmul_rn(xr, 0.299f));
    return __fmul_rn(g, 255.f);
}

// one thread per 2 x 2 quad: the four plane values, and the half plane's cv2.resize(img / 255., (w // 2, h // 2)) * 255. as the
// float32 mean ((q00 + q01) + (q10 + q11)) * 0.25 of q = v / 255
__global__ void __launch_bounds__(kThreads) niqe_prep_kernel(const vmb_niqe_prep_args a) {
    pdl_trigger();
    pdl_wait();
    const int hh = a.H / 2, hw = a.W / 2, b = blockIdx.y;
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= (int64_t)hh * hw) return;
    const int qy = (int)(i / hw), qx = (int)(i % hw);
    float q[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int y = 2 * qy + k / 2, x = 2 * qx + k % 2;
        const float v = plane_val(a, b, y, x);
        a.plane[((int64_t)b * a.H + y) * a.W + x] = v;
        q[k] = __fdiv_rn(v, 255.f);
    }
    const float m = __fmul_rn(__fadd_rn(__fadd_rn(q[0], q[1]), __fadd_rn(q[2], q[3])), 0.25f);
    a.half[((int64_t)b * hh + qy) * hw + qx] = __fmul_rn(m, 255.f);
}

// estimate_aggd_param from the fp64 sums s of one distribution of n values, and compute_feature's outputs for it:
// d == 0: [alpha, (beta_l + beta_r) / 2]; d > 0: [alpha, (beta_r - beta_l) gamma(2 / alpha) / gamma(1 / alpha), beta_l, beta_r].
// An empty side makes rhatnorm NaN; np.argmin of the all-NaN distances is 0, so alpha is then 0.2 and the betas NaN.
__device__ void aggd_features(const double* s, double n, const double* __restrict__ table, int d, double* out) {
    const double left = sqrt(s[1] / s[0]), right = sqrt(s[3] / s[2]);  // 0 / 0: NaN, as numpy's mean of an empty selection
    const double gh = left / right, m1 = s[4] / n;
    const double rhat = (m1 * m1) / ((s[1] + s[3]) / n);
    const double rhatnorm = (rhat * (gh * gh * gh + 1.0) * (gh + 1.0)) / ((gh * gh + 1.0) * (gh * gh + 1.0));
    int idx = 0;
    if (!isnan(rhatnorm)) {  // r_gam is strictly increasing: the argmin is the first entry >= rhatnorm or the one before it
        int lo = 0, hi = kTable;
        while (lo < hi) {
            const int mid = (lo + hi) / 2;
            if (table[mid] < rhatnorm) lo = mid + 1; else hi = mid;
        }
        idx = lo < kTable ? lo : kTable - 1;
        if (lo > 0) {
            const double e0 = table[lo - 1] - rhatnorm, e1 = idx == lo ? table[lo] - rhatnorm : INFINITY;
            if (__dmul_rn(e0, e0) <= __dmul_rn(e1, e1)) idx = lo - 1;  // a tie goes to the lower index, as np.argmin's
        }
    }
    const double alpha = gam_at(idx), g1 = tgamma(1.0 / alpha);
    const double r = sqrt(g1 / tgamma(3.0 / alpha)), bl = left * r, br = right * r;
    if (d == 0) {
        out[0] = alpha;
        out[1] = (bl + br) / 2.0;
    } else {
        out[0] = alpha;
        out[1] = (br - bl) * (tgamma(2.0 / alpha) / g1);
        out[2] = bl;
        out[3] = br;
    }
}

// One CTA: block blockIdx.x (reference order: block (h, w) is w * nbh + h) of image blockIdx.z at scale blockIdx.y + 1.  The block
// and its 3-pixel halo, clamped to the plane (scipy's mode='nearest' on the cut plane), go to shared memory; then the MSCN values
// (img - mu) / (sigma + 1), sigma = sqrt(|conv(img^2) - mu^2|), every step float32 and each 49-tap sum in fp64, rounded once.
__global__ void __launch_bounds__(kThreads) niqe_features_kernel(const vmb_niqe_features_args a) {
    extern __shared__ float smem[];
    __shared__ double red[kThreads / 32][kDists * kStats];
    __shared__ double tot[kDists * kStats];
    pdl_trigger();
    pdl_wait();
    const int scale = blockIdx.y, b = blockIdx.z, bs = kBlock >> scale, in_w = bs + 2 * kR;
    const int H = a.H >> scale, W = a.W >> scale, nbh = a.H / kBlock, nb = nbh * (a.W / kBlock);
    const int by = (blockIdx.x % nbh) * bs, bx = (blockIdx.x / nbh) * bs;
    const float* img = (scale ? a.half : a.plane) + (int64_t)b * H * W;
    float* in = smem;                  // [in_w][in_w]
    float* nrm = smem + in_w * in_w;   // [bs][bs]
    for (int i = threadIdx.x; i < in_w * in_w; i += kThreads) {
        const int y = min(max(by - kR + i / in_w, 0), H - 1), x = min(max(bx - kR + i % in_w, 0), W - 1);
        in[i] = img[(int64_t)y * W + x];
    }
    __syncthreads();
    float* mscn_out = scale ? a.mscn_half : a.mscn;
    for (int p = threadIdx.x; p < bs * bs; p += kThreads) {
        const int r = p / bs, c = p % bs;
        double mu = 0.0, sq = 0.0;
#pragma unroll
        for (int i = 0; i < 2 * kR + 1; ++i)
#pragma unroll
            for (int j = 0; j < 2 * kR + 1; ++j) {  // convolution: window tap (i, j) meets pixel (r + 3 - i, c + 3 - j)
                const float v = in[(r + 2 * kR - i) * in_w + c + 2 * kR - j];
                const double w = a.window[i * (2 * kR + 1) + j];
                mu = fma(w, (double)v, mu);
                sq = fma(w, (double)__fmul_rn(v, v), sq);
            }
        const float muf = __double2float_rn(mu), v = in[(r + kR) * in_w + c + kR];
        const float sigma = __fsqrt_rn(fabsf(__fsub_rn(__double2float_rn(sq), __fmul_rn(muf, muf))));
        const float n = __fdiv_rn(__fsub_rn(v, muf), __fadd_rn(sigma, 1.f));
        nrm[p] = n;
        if (mscn_out) mscn_out[((int64_t)b * H + by + r) * W + bx + c] = n;
    }
    __syncthreads();
    double s[kDists * kStats];
#pragma unroll
    for (int k = 0; k < kDists * kStats; ++k) s[k] = 0.0;
    for (int p = threadIdx.x; p < bs * bs; p += kThreads) {
        const int r = p / bs, c = p % bs, ru = (r + bs - 1) % bs, cl = (c + bs - 1) % bs, cr = (c + 1) % bs;
        const float x = nrm[p];
        // np.roll(block, shift, axis=(0, 1))[r, c] = block[r - shift[0], c - shift[1]], circular within the block
        const float v[kDists] = {x, __fmul_rn(x, nrm[r * bs + cl]), __fmul_rn(x, nrm[ru * bs + c]), __fmul_rn(x, nrm[ru * bs + cl]),
                                 __fmul_rn(x, nrm[ru * bs + cr])};
#pragma unroll
        for (int d = 0; d < kDists; ++d) {
            const double u = v[d], u2 = u * u;  // exact: a float32 square fits a double
            s[d * kStats + 0] += u < 0.0 ? 1.0 : 0.0;
            s[d * kStats + 1] += u < 0.0 ? u2 : 0.0;
            s[d * kStats + 2] += u > 0.0 ? 1.0 : 0.0;
            s[d * kStats + 3] += u > 0.0 ? u2 : 0.0;
            s[d * kStats + 4] += fabs(u);
        }
    }
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32;
#pragma unroll
    for (int k = 0; k < kDists * kStats; ++k) {
        double t = s[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
        if (lane == 0) red[warp][k] = t;
    }
    __syncthreads();
    if (threadIdx.x < kDists * kStats) {
        double t = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) t += red[w][threadIdx.x];
        tot[threadIdx.x] = t;
    }
    __syncthreads();
    if (threadIdx.x < kDists) {
        const int d = threadIdx.x;
        double* f = a.features + ((int64_t)b * nb + blockIdx.x) * kNF + scale * (kNF / 2) + (d == 0 ? 0 : 4 * d - 2);
        aggd_features(tot + d * kStats, (double)(bs * bs), a.table, d, f);
    }
}

// One CTA per image: mu_d = np.nanmean(features, axis=0); cov_d = np.cov of the rows without a NaN (ddof 1, about their own mean);
// score = sqrt(d^T ((cov_p + cov_d) / 2)^-1 d), d = mu_p - mu_d, by a Cholesky factorisation and one forward substitution.
// NaN where the reference raises (fewer than two NaN-free rows, no block) or the matrix is not positive definite.
__global__ void __launch_bounds__(kThreads) niqe_score_kernel(const vmb_niqe_score_args a) {
    extern __shared__ unsigned char valid[];  // [blocks]
    __shared__ double mu[kNF], mean[kNF], L[kNF][kNF];
    __shared__ int nvalid, ok;
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, nb = a.blocks;
    const double* F = a.features + (int64_t)b * nb * kNF;
    for (int r = threadIdx.x; r < nb; r += kThreads) {
        bool v = true;
        for (int c = 0; c < kNF; ++c) v = v && !isnan(F[(int64_t)r * kNF + c]);
        valid[r] = v;
    }
    __syncthreads();
    if (threadIdx.x < kNF) {
        const int c = threadIdx.x;
        double s = 0.0, sv = 0.0;
        int n = 0, nv = 0;
        for (int r = 0; r < nb; ++r) {
            const double v = F[(int64_t)r * kNF + c];
            if (!isnan(v)) { s += v; ++n; }
            if (valid[r]) { sv += v; ++nv; }
        }
        mu[c] = s / n;
        mean[c] = sv / nv;
        if (c == 0) {
            nvalid = nv;
            ok = nv >= 2;
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kNF * kNF; e += kThreads) {
        const int i = e / kNF, j = e % kNF;
        double s = 0.0;
        for (int r = 0; r < nb; ++r)
            if (valid[r]) s += (F[(int64_t)r * kNF + i] - mean[i]) * (F[(int64_t)r * kNF + j] - mean[j]);
        L[i][j] = (a.cov_pris[e] + s / (nvalid - 1)) / 2.0;
    }
    // in place: L's lower triangle becomes the Cholesky factor, column by column
    for (int k = 0; k < kNF; ++k) {
        __syncthreads();
        if (threadIdx.x == 0) {
            double d = L[k][k];
            for (int j = 0; j < k; ++j) d -= L[k][j] * L[k][j];
            if (!(d > 0.0)) ok = 0;
            L[k][k] = sqrt(d);
        }
        __syncthreads();
        const int i = k + 1 + threadIdx.x;
        if (i < kNF) {
            double d = L[i][k];
            for (int j = 0; j < k; ++j) d -= L[i][j] * L[k][j];
            L[i][k] = d / L[k][k];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double y[kNF], q = 0.0;
        for (int i = 0; i < kNF; ++i) {
            double d = a.mu_pris[i] - mu[i];
            for (int j = 0; j < i; ++j) d -= L[i][j] * y[j];
            y[i] = d / L[i][i];
            q += y[i] * y[i];
        }
        a.score[b] = ok ? sqrt(q) : NAN;
    }
}

}  // namespace

}  // namespace vmb

using namespace vmb;

// shared-memory bytes of the score kernel's row flags: up to this many blocks per image (a 40000 x 40000 image has 173,056)
static constexpr int kMaxScoreBlocks = 200 * 1024;

extern "C" int vmb_niqe_table(double* table, void* stream) {
    VMB_CHECK(table != nullptr, "niqe_table: null pointer");
    VMB_CUDA(launch_pdl(niqe_table_kernel, dim3(cdiv(kTable, kThreads)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), table));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

static int check_blocks(int batch, int H, int W, const char* who) {
    VMB_CHECK(batch > 0 && batch < 65536 && H > 0 && W > 0 && H % kBlock == 0 && W % kBlock == 0,
              "%s: bad batch %d or size %d x %d (positive multiples of %d)", who, batch, H, W, kBlock);
    VMB_CHECK((int64_t)(H / kBlock) * (W / kBlock) <= kMaxScoreBlocks, "%s: %d x %d has more than %d blocks", who, H, W, kMaxScoreBlocks);
    return VMB_OK;
}

extern "C" int vmb_niqe_prep(const vmb_niqe_prep_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->plane && a->half && metric_src_ok(a->src), "niqe_prep: null pointer or unknown source dtype");
    const int st = check_blocks(a->batch, a->H, a->W, "niqe_prep");
    if (st != VMB_OK) return st;
    VMB_CHECK((a->convert == VMB_NIQE_Y && (a->channels == 1 || a->channels == 3)) || (a->convert == VMB_NIQE_GRAY && a->channels == 3) ||
              (a->convert == VMB_NIQE_PLANE && a->channels == 1),
              "niqe_prep: conversion %d does not take %d channels (Y: 1 or 3, GRAY: 3, PLANE: 1)", a->convert, a->channels);
    const int64_t quads = (int64_t)(a->H / 2) * (a->W / 2);
    const dim3 grid((unsigned)((quads + kThreads - 1) / kThreads), (unsigned)a->batch);
    VMB_CUDA(launch_pdl(niqe_prep_kernel, grid, dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_niqe_features(const vmb_niqe_features_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->plane && a->half && a->table && a->features, "niqe_features: null pointer");
    const int st = check_blocks(a->batch, a->H, a->W, "niqe_features");
    if (st != VMB_OK) return st;
    VMB_CUDA(cudaFuncSetAttribute(niqe_features_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)feature_smem_bytes()));
    const dim3 grid((unsigned)((a->H / kBlock) * (a->W / kBlock)), 2u, (unsigned)a->batch);
    VMB_CUDA(launch_pdl(niqe_features_kernel, grid, dim3(kThreads), feature_smem_bytes(), static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_niqe_score(const vmb_niqe_score_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->mu_pris && a->cov_pris && a->score && (a->features || a->blocks == 0), "niqe_score: null pointer");
    VMB_CHECK(a->batch > 0 && a->batch < (1 << 30) && a->blocks >= 0 && a->blocks <= kMaxScoreBlocks,
              "niqe_score: bad batch %d or block count %d (at most %d)", a->batch, a->blocks, kMaxScoreBlocks);
    VMB_CUDA(cudaFuncSetAttribute(niqe_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxScoreBlocks));
    VMB_CUDA(launch_pdl(niqe_score_kernel, dim3((unsigned)a->batch), dim3(kThreads), (size_t)a->blocks, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
