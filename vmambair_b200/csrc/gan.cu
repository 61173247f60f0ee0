// The GAN stage's discriminator (UNetDiscriminatorSN) between its convolutions, and the vanilla GAN loss (vmambair_b200.gan):
// spectral normalisation of all SN layers of a call in a fixed number of launches, the decoder junction up2(leaky(pre) [+ skip])
// and its adjoint as a gather, the encoder's leaky ReLU with a two-gradient backward, and BCE-with-logits as a two-level sum.
// Every reduction has one fixed order and there are no atomics, so a forward + backward is bitwise reproducible; all math is fp32,
// activations are fp32 or bf16 (VMB_F32 / VMB_BF16).  Nothing reads the host.
#include <math.h>

#include "common.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;
constexpr float kSlope = 0.2f;  // F.leaky_relu(negative_slope=0.2) of every activation of the discriminator

template <typename T> __device__ __forceinline__ float ld(const void* p, int64_t i) { return to_f32<T>(static_cast<const T*>(p)[i]); }
template <typename T> __device__ __forceinline__ void st(void* p, int64_t i, float v) { static_cast<T*>(p)[i] = from_f32<T>(v); }
__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : x * kSlope; }
// leaky'(pre) from pre or from leaky(pre) alike (same sign); torch's in-place backward takes the slope at 0 too
__device__ __forceinline__ float dleaky(float r) { return r > 0.f ? 1.f : kSlope; }

// sum of v over the CTA in one fixed order (butterfly within each warp, then warp 0 adds the warp sums in index order); every thread
// gets the result.  `red` holds kThreads / 32 + 1 floats.
__device__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    __syncthreads();  // red may still be read from a previous call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < (int)blockDim.x / 32; ++w) s += red[w];
        red[kThreads / 32] = s;
    }
    __syncthreads();
    return red[kThreads / 32];
}

// sum of p[0..n) in index order (n is small: a few hundred per-CTA partials at most)
__device__ __forceinline__ float serial_sum(const float* p, int n) {
    float s = 0.f;
    for (int i = 0; i < n; ++i) s += p[i];
    return s;
}

// ---- spectral norm ----
// Layer l is the (rows, cols) matrix W_orig.view(out, -1).  Workspace per layer (floats, offsets in SnPlan):
//   p1 [nrb1][cols]  partial W^T u over 32-row blocks          vraw [cols]  W^T u
//   vnp [ncb]        sum vraw^2 per 256-column block           wv [rows]    W v
//   wnp [nrb3]       sum wv^2 per 8-row block
constexpr int kRB1 = 32;           // rows per CTA of the W^T u partials
constexpr int kRB3 = kThreads / 32;  // rows per CTA of W v (one warp per row)
constexpr int kEl4 = 4096;         // elements per CTA of the scaling and of the backward passes

struct SnLayerPlan {
    int64_t p1, vraw, vnp, wv, wnp;   // workspace offsets (floats)
    int nrb1, ncb, nrb3, nel;         // row blocks, column blocks, row blocks of W v, element chunks
    int b[4];                         // first CTA of the layer in each phase's grid (W^T u, v, W v, elements)
};
struct SnPlan {
    SnLayerPlan l[VMB_SN_MAX_LAYERS + 1];  // l[layers].b = each grid's size
    int64_t floats;
};

SnPlan sn_plan(int layers, const int* rows, const int* cols) {
    SnPlan p = {};
    int64_t off = 0;
    int b1 = 0, b2 = 0, b3 = 0, b4 = 0;
    for (int i = 0; i < layers; ++i) {
        SnLayerPlan& q = p.l[i];
        q.nrb1 = cdiv(rows[i], kRB1);
        q.ncb = cdiv(cols[i], kThreads);
        q.nrb3 = cdiv(rows[i], kRB3);
        q.nel = (int)(((int64_t)rows[i] * cols[i] + kEl4 - 1) / kEl4);
        q.p1 = off; off += (int64_t)q.nrb1 * cols[i];
        q.vraw = off; off += cols[i];
        q.vnp = off; off += q.ncb;
        q.wv = off; off += rows[i];
        q.wnp = off; off += q.nrb3;
        q.b[0] = b1; b1 += q.nrb1 * q.ncb;
        q.b[1] = b2; b2 += q.ncb;
        q.b[2] = b3; b3 += q.nrb3;
        q.b[3] = b4; b4 += q.nel;
    }
    p.l[layers].b[0] = b1; p.l[layers].b[1] = b2; p.l[layers].b[2] = b3; p.l[layers].b[3] = b4;
    p.floats = off;
    return p;
}

// which layer CTA `b` of phase F's grid belongs to
template <int F>
__device__ __forceinline__ int layer_of(const SnPlan& p, int layers, int b) {
    int l = 0;
    while (l + 1 < layers && b >= p.l[l + 1].b[F]) ++l;
    return l;
}

__device__ __forceinline__ float normalize_den(float sumsq, float eps) { return fmaxf(sqrtf(sumsq), eps); }

// phase 1 (train): p1[rb][k] = sum_{m in row block rb} W[m][k] u[m], one column per thread, rows in ascending order
__global__ void __launch_bounds__(kThreads) sn_wtu_kernel(const vmb_sn_fwd_args a, const SnPlan p) {
    pdl_trigger();
    pdl_wait();
    const int l = layer_of<0>(p, a.layers, blockIdx.x);
    const SnLayerPlan& q = p.l[l];
    const int b = blockIdx.x - q.b[0], rb = b / q.ncb, cb = b % q.ncb;
    const int K = a.cols[l], R = a.rows[l], k = cb * kThreads + threadIdx.x;
    if (k >= K) return;
    const float* w = a.w[l];
    const float* u = a.u[l];
    const int m1 = min(R, (rb + 1) * kRB1);
    float s = 0.f;
    for (int m = rb * kRB1; m < m1; ++m) s = fmaf(__ldg(w + (int64_t)m * K + k), __ldg(u + m), s);
    static_cast<float*>(a.workspace)[q.p1 + (int64_t)rb * K + k] = s;
}

// phase 2 (train): vraw = W^T u (row-block partials in order), and the column block's sum of vraw^2
__global__ void __launch_bounds__(kThreads) sn_v_kernel(const vmb_sn_fwd_args a, const SnPlan p) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    const int l = layer_of<1>(p, a.layers, blockIdx.x);
    const SnLayerPlan& q = p.l[l];
    const int cb = blockIdx.x - q.b[1], K = a.cols[l], k = cb * kThreads + threadIdx.x;
    float* ws = static_cast<float*>(a.workspace);
    float s = 0.f;
    if (k < K) {
        for (int rb = 0; rb < q.nrb1; ++rb) s += ws[q.p1 + (int64_t)rb * K + k];
        ws[q.vraw + k] = s;
    }
    const float ss = block_sum(s * s, red);
    if (threadIdx.x == 0) ws[q.vnp + cb] = ss;
}

// phase 3: wv = W v, one warp per row, with v = normalize(vraw) (train) or the stored v (eval) staged in shared memory; and the
// row block's sum of wv^2
__global__ void __launch_bounds__(kThreads) sn_wv_kernel(const vmb_sn_fwd_args a, const SnPlan p) {
    extern __shared__ float vs[];
    __shared__ float red[kRB3];
    pdl_trigger();
    pdl_wait();
    const int l = layer_of<2>(p, a.layers, blockIdx.x);
    const SnLayerPlan& q = p.l[l];
    const int K = a.cols[l], R = a.rows[l];
    float* ws = static_cast<float*>(a.workspace);
    if (a.train) {
        const float den = normalize_den(serial_sum(ws + q.vnp, q.ncb), a.eps);
        for (int k = threadIdx.x; k < K; k += kThreads) vs[k] = __fdiv_rn(ws[q.vraw + k], den);
    } else {
        for (int k = threadIdx.x; k < K; k += kThreads) vs[k] = a.v[l][k];
    }
    __syncthreads();
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, m = (blockIdx.x - q.b[2]) * kRB3 + warp;
    float s = 0.f;
    if (m < R) {
        const float* w = a.w[l] + (int64_t)m * K;
        for (int k = lane; k < K; k += 32) s = fmaf(__ldg(w + k), vs[k], s);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) ws[q.wv + m] = s;
    }
    if (lane == 0) red[warp] = m < R ? s * s : 0.f;
    __syncthreads();
    if (threadIdx.x == 0) ws[q.wnp + (blockIdx.x - q.b[2])] = serial_sum(red, kRB3);
}

// phase 4: u = normalize(wv) (train) or the stored u (eval), sigma = u . wv, Wn = W / sigma; the layer's first CTA writes sigma, the
// u and v the backward uses, and (train) advances the stored u and v
template <typename T>
__global__ void __launch_bounds__(kThreads) sn_scale_kernel(const vmb_sn_fwd_args a, const SnPlan p) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    const int l = layer_of<3>(p, a.layers, blockIdx.x);
    const SnLayerPlan& q = p.l[l];
    const int K = a.cols[l], R = a.rows[l], chunk = blockIdx.x - q.b[3];
    const bool train = a.train;
    const float* ws = static_cast<const float*>(a.workspace);
    const float* wv = ws + q.wv;
    float* u = a.u[l];
    const float den_u = train ? normalize_den(serial_sum(ws + q.wnp, q.nrb3), a.eps) : 1.f;
    float s = 0.f;
    for (int m = threadIdx.x; m < R; m += kThreads) s = fmaf(train ? __fdiv_rn(wv[m], den_u) : u[m], wv[m], s);
    const float sigma = block_sum(s, red);
    const float* w = a.w[l];
    void* wn = a.wn[l];
    const int64_t n = (int64_t)R * K, i0 = (int64_t)chunk * kEl4, i1 = min(n, i0 + kEl4);
    for (int64_t i = i0 + threadIdx.x; i < i1; i += kThreads) st<T>(wn, i, __fdiv_rn(__ldg(w + i), sigma));
    if (chunk != 0) return;
    if (threadIdx.x == 0) a.sigma[l] = sigma;
    // every thread reads its own elements before writing them: the stored u / v may be overwritten in place
    float* us = a.u_save[l];
    for (int m = threadIdx.x; m < R; m += kThreads) {
        const float um = train ? __fdiv_rn(wv[m], den_u) : u[m];
        us[m] = um;
        if (train) u[m] = um;
    }
    const float* vraw = ws + q.vraw;
    float* v = a.v[l];
    float* vsv = a.v_save[l];
    const float den_v = train ? normalize_den(serial_sum(ws + q.vnp, q.ncb), a.eps) : 1.f;
    for (int k = threadIdx.x; k < K; k += kThreads) {
        const float vk = train ? __fdiv_rn(vraw[k], den_v) : v[k];
        vsv[k] = vk;
        if (train) v[k] = vk;
    }
}

// backward, pass 1: per 4096-element chunk, sum of G * W_orig
template <typename T>
__global__ void __launch_bounds__(kThreads) sn_bwd_dot_kernel(const vmb_sn_bwd_args a, const SnPlan p) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    const int l = layer_of<3>(p, a.layers, blockIdx.x);
    const SnLayerPlan& q = p.l[l];
    const int chunk = blockIdx.x - q.b[3];
    const int64_t n = (int64_t)a.rows[l] * a.cols[l], i0 = (int64_t)chunk * kEl4, i1 = min(n, i0 + kEl4);
    float s = 0.f;
    for (int64_t i = i0 + threadIdx.x; i < i1; i += kThreads) s = fmaf(ld<T>(a.g[l], i), __ldg(a.w[l] + i), s);
    s = block_sum(s, red);
    if (threadIdx.x == 0) static_cast<float*>(a.workspace)[q.b[3] + chunk] = s;
}

// backward, pass 2: dW_orig = G / sigma - (<G, W_orig> / sigma^2) u v^T, written or added to grad
template <typename T>
__global__ void __launch_bounds__(kThreads) sn_bwd_apply_kernel(const vmb_sn_bwd_args a, const SnPlan p) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    const int l = layer_of<3>(p, a.layers, blockIdx.x);
    const SnLayerPlan& q = p.l[l];
    const int chunk = blockIdx.x - q.b[3], K = a.cols[l];
    const float* part = static_cast<const float*>(a.workspace) + q.b[3];
    float s = 0.f;
    for (int i = threadIdx.x; i < q.nel; i += kThreads) s += part[i];
    const float dot = block_sum(s, red);
    const float sigma = a.sigma[l], inv = __fdiv_rn(1.f, sigma), c = __fdiv_rn(dot, sigma * sigma);
    const int64_t n = (int64_t)a.rows[l] * K, i0 = (int64_t)chunk * kEl4, i1 = min(n, i0 + kEl4);
    float* grad = a.grad[l];
    for (int64_t i = i0 + threadIdx.x; i < i1; i += kThreads) {
        const int m = (int)(i / K), k = (int)(i - (int64_t)m * K);
        const float d = ld<T>(a.g[l], i) * inv - c * a.u[l][m] * a.v[l][k];
        grad[i] = a.accumulate[l] ? grad[i] + d : d;
    }
}

// ---- decoder junction: out = up2(leaky(pre) [+ skip]), bilinear x2, align_corners=False ----
// Output row Y reads input rows (r0, r1) with weights (h0, h1) exactly as torch's upsample_bilinear2d: Y = 2i -> (i - 1, i),
// (0.25, 0.75); Y = 2i + 1 -> (i, i + 1), (0.75, 0.25); clamped at the borders (row 0 reads row 0 alone).
__device__ __forceinline__ void src_pair(int Y, int n, int& r0, int& r1, float& h0, float& h1) {
    const int i = Y >> 1;
    if (Y & 1) {
        r0 = i; r1 = min(i + 1, n - 1); h0 = 0.75f; h1 = 0.25f;
    } else if (i == 0) {
        r0 = 0; r1 = 0; h0 = 1.f; h1 = 0.f;
    } else {
        r0 = i - 1; r1 = i; h0 = 0.25f; h1 = 0.75f;
    }
}

template <typename T>
__device__ __forceinline__ float x_at(const vmb_gan_up_args& a, int64_t o) { return leaky(ld<T>(a.pre, o)) + (a.skip ? ld<T>(a.skip, o) : 0.f); }

// one thread: output row Y, input column j -> outputs (Y, 2j) and (Y, 2j + 1)
template <typename T>
__global__ void __launch_bounds__(kThreads) up_kernel(const vmb_gan_up_args a) {
    pdl_trigger();
    pdl_wait();
    const int H = a.H, W = a.W;
    const int64_t n = (int64_t)a.planes * 2 * H * W;
    for (int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x; t < n; t += (int64_t)gridDim.x * kThreads) {
        const int j = (int)(t % W);
        const int64_t py = t / W;
        const int Y = (int)(py % (2 * H));
        const int64_t pl = py / (2 * H), base = pl * H * W;
        int r0, r1;
        float h0, h1;
        src_pair(Y, H, r0, r1, h0, h1);
        const int cl = max(j - 1, 0), cr = min(j + 1, W - 1);
        const int64_t o0 = base + (int64_t)r0 * W, o1 = base + (int64_t)r1 * W;
        const float a0l = x_at<T>(a, o0 + cl), a0c = x_at<T>(a, o0 + j), a0r = x_at<T>(a, o0 + cr);
        const float a1l = x_at<T>(a, o1 + cl), a1c = x_at<T>(a, o1 + j), a1r = x_at<T>(a, o1 + cr);
        // X = 2j reads columns (j - 1, j) with (0.25, 0.75), at j = 0 column 0 alone; X = 2j + 1 reads (j, j + 1) with (0.75, 0.25)
        const float w0 = j == 0 ? 1.f : 0.25f, w1 = j == 0 ? 0.f : 0.75f;
        float o2[2];
        o2[0] = h0 * (w0 * a0l + w1 * a0c) + h1 * (w0 * a1l + w1 * a1c);
        o2[1] = h0 * (0.75f * a0c + 0.25f * a0r) + h1 * (0.75f * a1c + 0.25f * a1r);
        const int64_t o = (pl * 2 * H + Y) * (int64_t)(2 * W) + 2 * j;
        st<T>(a.out, o, o2[0]);
        st<T>(a.out, o + 1, o2[1]);
    }
}

// taps of the adjoint of up2 along one axis at input index i of n: output indices 2i - 1 .. 2i + 2 with weights
// (0.25, 0.75, 0.75, 0.25), the clamped border taps folded into their neighbour (weight 0 marks a tap outside the output)
__device__ __forceinline__ void adj_taps(int i, int n, float* w) {
    w[0] = i > 0 ? 0.25f : 0.f;
    w[1] = i > 0 ? 0.75f : 1.f;
    w[2] = i < n - 1 ? 0.75f : 1.f;
    w[3] = i < n - 1 ? 0.25f : 0.f;
}

// one thread per input element: adj = up2^T(dout) gathered from its 4 x 4 output neighbourhood, rows then columns in order;
// dskip = adj, dpre = adj leaky'(pre)
template <typename T>
__global__ void __launch_bounds__(kThreads) up_bwd_kernel(const vmb_gan_up_bwd_args a) {
    pdl_trigger();
    pdl_wait();
    const int H = a.H, W = a.W, W2 = 2 * W;
    const int64_t n = (int64_t)a.planes * H * W;
    for (int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x; t < n; t += (int64_t)gridDim.x * kThreads) {
        const int j = (int)(t % W), i = (int)((t / W) % H);
        const int64_t pl = t / ((int64_t)H * W);
        float wy[4], wx[4];
        adj_taps(i, H, wy);
        adj_taps(j, W, wx);
        const int64_t base = pl * 4 * H * W;
        float adj = 0.f;
#pragma unroll
        for (int y = 0; y < 4; ++y) {
            if (wy[y] == 0.f) continue;
            const int64_t row = base + (int64_t)(2 * i - 1 + y) * W2;
            float r = 0.f;
#pragma unroll
            for (int x = 0; x < 4; ++x)
                if (wx[x] != 0.f) r = fmaf(wx[x], ld<T>(a.dout, row + 2 * j - 1 + x), r);
            adj = fmaf(wy[y], r, adj);
        }
        if (a.dskip) st<T>(a.dskip, t, adj);
        st<T>(a.dpre, t, adj * dleaky(ld<T>(a.pre, t)));
    }
}

// ---- activation: out = leaky(x) [+ skip]; backward dx = (g [+ g2]) leaky'(ref) ----
template <typename T>
__global__ void __launch_bounds__(kThreads) act_kernel(const vmb_gan_act_args a) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads)
        st<T>(a.out, i, leaky(ld<T>(a.x, i)) + (a.skip ? ld<T>(a.skip, i) : 0.f));
}

template <typename T>
__global__ void __launch_bounds__(kThreads) act_bwd_kernel(const vmb_gan_act_bwd_args a) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads) {
        const float g = a.g2 ? ld<T>(a.g, i) + ld<T>(a.g2, i) : ld<T>(a.g, i);
        st<T>(a.dx, i, g * dleaky(ld<T>(a.ref, i)));
    }
}

// ---- vanilla GAN loss: mean BCE-with-logits against a constant target ----
constexpr int kBceMaxCtas = 512;  // partials; the second pass adds them in one CTA

unsigned grid_1d(int64_t n, int64_t cap) {
    const int64_t g = (n + kThreads - 1) / kThreads;
    return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) bce_partial_kernel(const vmb_bce_logits_args a) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    float s = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads) {
        const float x = ld<T>(a.x, i);
        s += fmaxf(x, 0.f) - x * a.target + log1pf(expf(-fabsf(x)));  // stable for any |x|
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) static_cast<float*>(a.workspace)[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) bce_final_kernel(const vmb_bce_logits_args a, int parts) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    const float* ws = static_cast<const float*>(a.workspace);
    float s = 0.f;
    for (int i = threadIdx.x; i < parts; i += kThreads) s += ws[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) *a.loss = __fdiv_rn(s, (float)a.n) * a.weight;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) bce_bwd_kernel(const vmb_bce_logits_bwd_args a) {
    pdl_trigger();
    pdl_wait();
    const float scale = __fdiv_rn(*a.grad_loss * a.weight, (float)a.n);
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads) {
        const float x = ld<T>(a.x, i);
        st<T>(a.grad_x, i, scale * (__fdiv_rn(1.f, 1.f + expf(-x)) - a.target));
    }
}

bool gan_dtype_ok(int dt) { return dt == VMB_F32 || dt == VMB_BF16; }

int check_sn_layers(int layers, const int* rows, const int* cols, const char* what) {
    VMB_CHECK(layers >= 1 && layers <= VMB_SN_MAX_LAYERS, "%s: layers %d not in 1..%d", what, layers, VMB_SN_MAX_LAYERS);
    for (int i = 0; i < layers; ++i)
        VMB_CHECK(rows[i] >= 1 && cols[i] >= 1 && (int64_t)rows[i] * cols[i] < ((int64_t)1 << 31),
                  "%s: layer %d has a %d x %d matrix", what, i, rows[i], cols[i]);
    return VMB_OK;
}

}  // namespace

}  // namespace vmb

using namespace vmb;

extern "C" int64_t vmb_sn_workspace_bytes(int layers, const int* rows, const int* cols) {
    if (layers < 1 || layers > VMB_SN_MAX_LAYERS) return -1;
    return sn_plan(layers, rows, cols).floats * (int64_t)sizeof(float);
}

extern "C" int vmb_sn_fwd(const vmb_sn_fwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->workspace && a->sigma, "sn_fwd: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "sn_fwd: dtype %d is not fp32 or bf16", a->dtype);
    const int st0 = check_sn_layers(a->layers, a->rows, a->cols, "sn_fwd");
    if (st0 != VMB_OK) return st0;
    int max_cols = 0;
    for (int i = 0; i < a->layers; ++i) {
        VMB_CHECK(a->w[i] && a->wn[i] && a->u[i] && a->v[i] && a->u_save[i] && a->v_save[i], "sn_fwd: null pointer in layer %d", i);
        max_cols = max(max_cols, a->cols[i]);
    }
    const SnPlan p = sn_plan(a->layers, a->rows, a->cols);
    const SnLayerPlan& g = p.l[a->layers];
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t vbytes = (size_t)max_cols * sizeof(float);
    VMB_CHECK(vbytes <= 227 * 1024, "sn_fwd: %d columns do not fit in shared memory", max_cols);
    VMB_CUDA(cudaFuncSetAttribute(sn_wv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vbytes));
    if (a->train) {
        VMB_CUDA(launch_pdl(sn_wtu_kernel, dim3(g.b[0]), dim3(kThreads), 0, s, *a, p));
        VMB_CUDA(launch_pdl(sn_v_kernel, dim3(g.b[1]), dim3(kThreads), 0, s, *a, p));
    }
    VMB_CUDA(launch_pdl(sn_wv_kernel, dim3(g.b[2]), dim3(kThreads), vbytes, s, *a, p));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(sn_scale_kernel<float>, dim3(g.b[3]), dim3(kThreads), 0, s, *a, p));
    else
        VMB_CUDA(launch_pdl(sn_scale_kernel<__nv_bfloat16>, dim3(g.b[3]), dim3(kThreads), 0, s, *a, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_sn_bwd(const vmb_sn_bwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->workspace && a->sigma, "sn_bwd: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "sn_bwd: dtype %d is not fp32 or bf16", a->dtype);
    const int st0 = check_sn_layers(a->layers, a->rows, a->cols, "sn_bwd");
    if (st0 != VMB_OK) return st0;
    for (int i = 0; i < a->layers; ++i)
        VMB_CHECK(a->g[i] && a->w[i] && a->u[i] && a->v[i] && a->grad[i], "sn_bwd: null pointer in layer %d", i);
    const SnPlan p = sn_plan(a->layers, a->rows, a->cols);
    const unsigned grid = (unsigned)p.l[a->layers].b[3];
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (a->dtype == VMB_F32) {
        VMB_CUDA(launch_pdl(sn_bwd_dot_kernel<float>, dim3(grid), dim3(kThreads), 0, s, *a, p));
        VMB_CUDA(launch_pdl(sn_bwd_apply_kernel<float>, dim3(grid), dim3(kThreads), 0, s, *a, p));
    } else {
        VMB_CUDA(launch_pdl(sn_bwd_dot_kernel<__nv_bfloat16>, dim3(grid), dim3(kThreads), 0, s, *a, p));
        VMB_CUDA(launch_pdl(sn_bwd_apply_kernel<__nv_bfloat16>, dim3(grid), dim3(kThreads), 0, s, *a, p));
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int64_t vmb_sn_bwd_workspace_bytes(int layers, const int* rows, const int* cols) {
    if (layers < 1 || layers > VMB_SN_MAX_LAYERS) return -1;
    return (int64_t)sn_plan(layers, rows, cols).l[layers].b[3] * (int64_t)sizeof(float);
}

extern "C" int vmb_gan_up(const vmb_gan_up_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->pre && a->out, "gan_up: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "gan_up: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->planes >= 1 && a->H >= 1 && a->W >= 1, "gan_up: empty input (%d planes of %d x %d)", a->planes, a->H, a->W);
    const int64_t n = (int64_t)a->planes * 2 * a->H * a->W;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(n, 16 * num_sms()));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(up_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(up_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_gan_up_bwd(const vmb_gan_up_bwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->dout && a->pre && a->dpre, "gan_up_bwd: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "gan_up_bwd: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->planes >= 1 && a->H >= 1 && a->W >= 1, "gan_up_bwd: empty input (%d planes of %d x %d)", a->planes, a->H, a->W);
    const int64_t n = (int64_t)a->planes * a->H * a->W;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(n, 16 * num_sms()));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(up_bwd_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(up_bwd_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_gan_act(const vmb_gan_act_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->x && a->out, "gan_act: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "gan_act: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->n >= 1, "gan_act: empty input");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(a->n, 16 * num_sms()));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(act_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(act_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_gan_act_bwd(const vmb_gan_act_bwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->g && a->ref && a->dx, "gan_act_bwd: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "gan_act_bwd: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->n >= 1, "gan_act_bwd: empty input");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(a->n, 16 * num_sms()));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(act_bwd_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(act_bwd_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int64_t vmb_bce_logits_workspace_bytes(int64_t n) { return (int64_t)grid_1d(n, kBceMaxCtas) * (int64_t)sizeof(float); }

extern "C" int vmb_bce_logits(const vmb_bce_logits_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->x && a->loss && a->workspace, "bce_logits: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "bce_logits: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->n >= 1, "bce_logits: empty input");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned parts = grid_1d(a->n, kBceMaxCtas);
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(bce_partial_kernel<float>, dim3(parts), dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(bce_partial_kernel<__nv_bfloat16>, dim3(parts), dim3(kThreads), 0, s, *a));
    VMB_CUDA(launch_pdl(bce_final_kernel, dim3(1), dim3(kThreads), 0, s, *a, (int)parts));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_bce_logits_bwd(const vmb_bce_logits_bwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->x && a->grad_loss && a->grad_x, "bce_logits_bwd: null pointer");
    VMB_CHECK(gan_dtype_ok(a->dtype), "bce_logits_bwd: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->n >= 1, "bce_logits_bwd: empty input");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(a->n, 16 * num_sms()));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(bce_bwd_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(bce_bwd_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
