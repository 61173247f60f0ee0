// basicsr's PerceptualLoss (VGG features, vmambair_b200.perceptual) between its convolutions: the input normalisation of output and
// ground truth into one 2B batch, one stage kernel per convolution (in-place ReLU fused with the following 2 x 2 max-pool, the
// criterion's per-CTA partials at the layers that are features, and the few bits the backward needs), the loss in one CTA, and on
// the way back one kernel per stage that builds the gradient at the convolution's output from those bits.
// Every reduction has one fixed order and there are no atomics, so a forward + backward is bitwise reproducible; all math is fp32,
// activations are fp32 or bf16 (VMB_F32 / VMB_BF16).  Nothing reads the host.
#include <math.h>

#include "common.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxCtas = 2048;  // stage grid cap: its partials are added by one CTA

template <typename T> __device__ __forceinline__ float ld(const void* p, int64_t i) { return to_f32<T>(static_cast<const T*>(p)[i]); }
template <typename T> __device__ __forceinline__ void st(void* p, int64_t i, float v) { static_cast<T*>(p)[i] = from_f32<T>(v); }

// sum of v over the CTA in one fixed order (butterfly within each warp, then thread 0 adds the warp sums in index order); the result
// is valid in thread 0.  `red` holds kThreads / 32 floats.
__device__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // red may still be read from a previous call
    if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = v;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < kThreads / 32; ++w) s += red[w];
    return s;
}

__device__ __forceinline__ float crit_term(float d, int crit) { return crit == VMB_PERCEP_L1 ? fabsf(d) : d * d; }
// the l1 sign code of one element: bit 0 d > 0, bit 1 d < 0 (torch's sign, 0 at 0)
__device__ __forceinline__ uint32_t sign_code(float d) { return (d > 0.f ? 1u : 0u) | (d < 0.f ? 2u : 0u); }
__device__ __forceinline__ float sign_of(uint32_t c) { return (c & 1u) ? 1.f : ((c & 2u) ? -1.f : 0.f); }

unsigned stage_ctas(int B, int C, int H, int W) {
    const int64_t cells = (int64_t)B * C * ((H + 1) / 2) * ((W + 1) / 2);
    const int64_t g = (cells + kThreads - 1) / kThreads;
    return (unsigned)(g < kMaxCtas ? (g > 0 ? g : 1) : kMaxCtas);
}

// ---- input: out[0:B] = norm(x), out[B:2B] = norm(gt), norm(v) = ((v + 1) / 2 - mean) / std with each step optional ----
template <typename T>
__global__ void __launch_bounds__(kThreads) norm_kernel(const vmb_percep_norm_args a) {
    pdl_trigger();
    pdl_wait();
    const int H = a.H, W = a.W;
    const int64_t n = (int64_t)a.B * 3 * H * W;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < 2 * n; i += (int64_t)gridDim.x * kThreads) {
        const bool g = i >= n;
        const int64_t j = g ? i - n : i;
        const int w = (int)(j % W), h = (int)((j / W) % H), c = (int)((j / ((int64_t)H * W)) % 3);
        const int64_t b = j / (3 * (int64_t)H * W);
        const int64_t o = g ? b * a.gt_stride[0] + c * a.gt_stride[1] + h * a.gt_stride[2] + w * a.gt_stride[3]
                            : b * a.x_stride[0] + c * a.x_stride[1] + h * a.x_stride[2] + w * a.x_stride[3];
        float v = (g ? a.gt : a.x)[o];
        if (a.range_norm) v = __fdiv_rn(v + 1.f, 2.f);
        if (a.mean) v = __fdiv_rn(v - a.mean[c], a.std[c]);
        st<T>(a.out, i, v);
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) norm_bwd_kernel(const vmb_percep_norm_bwd_args a) {
    pdl_trigger();
    pdl_wait();
    const int64_t hw = (int64_t)a.H * a.W, n = (int64_t)a.B * 3 * hw;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        float g = ld<T>(a.g, i);
        if (a.std) g = __fdiv_rn(g, a.std[(i / hw) % 3]);
        if (a.range_norm) g = __fdiv_rn(g, 2.f);
        a.dx[i] = g;
    }
}

// ---- one stage: the conv output y (2B, C, H, W) in 2 x 2 cells, one thread per cell of the x half and its gt twin ----
// Cells tile ceil(H / 2) x ceil(W / 2); a cell past an odd border has fewer than 4 elements and pools nothing (floor sizes).
template <typename T>
__global__ void __launch_bounds__(kThreads) stage_kernel(const vmb_percep_stage_args a) {
    __shared__ float red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    const int H = a.H, W = a.W, Hc = (H + 1) / 2, Wc = (W + 1) / 2, Hp = H / 2, Wp = W / 2, crit = a.crit;
    const int64_t cells = (int64_t)a.B * a.C * Hc * Wc, half = (int64_t)a.B * a.C * H * W, halfp = (int64_t)a.B * a.C * Hp * Wp;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x; t < cells; t += (int64_t)gridDim.x * kThreads) {
        const int cj = (int)(t % Wc);
        const int64_t r = t / Wc;
        const int ci = (int)(r % Hc);
        const int64_t pl = r / Hc;
        float vx[4], vg[4];
        bool in[4];
        int64_t idx[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int y = 2 * ci + e / 2, x = 2 * cj + e % 2;
            in[e] = y < H && x < W;
            idx[e] = (pl * H + y) * W + x;
            vx[e] = in[e] ? ld<T>(a.y, idx[e]) : 0.f;
            vg[e] = in[e] ? ld<T>(a.y, idx[e] + half) : 0.f;
        }
        uint32_t code = 0, c0 = 0, c1 = 0;
        if (a.feat[0]) {  // conv feature: before the ReLU
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (!in[e]) continue;
                const float d = vx[e] - vg[e];
                s0 += crit_term(d, crit);
                c0 |= sign_code(d) << (2 * e);
                if (crit != VMB_PERCEP_L1 && a.save[0]) static_cast<float*>(a.save[0])[idx[e]] = d;
            }
        }
        if (a.relu) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                code |= (vx[e] > 0.f ? 1u : 0u) << e;
                vx[e] = vx[e] > 0.f ? vx[e] : 0.f;
                vg[e] = vg[e] > 0.f ? vg[e] : 0.f;
                if (in[e] && !a.pool) {  // with a pool after it, only the pooled tensor is read again
                    st<T>(a.y, idx[e], vx[e]);
                    st<T>(a.y, idx[e] + half, vg[e]);
                }
            }
        }
        if (a.feat[1]) {  // relu feature
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (!in[e]) continue;
                const float d = vx[e] - vg[e];
                s1 += crit_term(d, crit);
                c1 |= sign_code(d) << (2 * e);
                if (crit != VMB_PERCEP_L1 && a.save[1]) static_cast<float*>(a.save[1])[idx[e]] = d;
            }
        }
        if (a.pool && in[3]) {  // complete cell: max over the window in row-major order, the first maximum wins (torch)
            int am = 0;
            float mx = vx[0], mg = vg[0];
#pragma unroll
            for (int e = 1; e < 4; ++e) {
                if (vx[e] > mx) { mx = vx[e]; am = e; }
                mg = vg[e] > mg ? vg[e] : mg;
            }
            code |= (uint32_t)am << 4;
            const int64_t p = (pl * Hp + ci) * Wp + cj;
            st<T>(a.pooled, p, mx);
            st<T>(a.pooled, p + halfp, mg);
            if (a.feat[2]) {  // pool feature, at the pooled element
                const float d = mx - mg;
                s2 += crit_term(d, crit);
                if (a.save[2]) {
                    if (crit == VMB_PERCEP_L1) static_cast<uint8_t*>(a.save[2])[p] = (uint8_t)sign_code(d);
                    else static_cast<float*>(a.save[2])[p] = d;
                }
            }
        }
        if (a.code) a.code[t] = (uint8_t)code;
        if (crit == VMB_PERCEP_L1) {
            if (a.feat[0] && a.save[0]) static_cast<uint8_t*>(a.save[0])[t] = (uint8_t)c0;
            if (a.feat[1] && a.save[1]) static_cast<uint8_t*>(a.save[1])[t] = (uint8_t)c1;
        }
    }
    float* const part[3] = {a.partial[0], a.partial[1], a.partial[2]};
    const float sums[3] = {s0, s1, s2};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (!a.feat[k]) continue;
        const float v = block_sum(sums[k], red);
        if (threadIdx.x == 0) part[k][blockIdx.x] = v;
    }
}

// ---- the loss: per feature, its partials added in order, then the mean or the Frobenius norm, times w_k, summed in order ----
__global__ void __launch_bounds__(kThreads) loss_kernel(const vmb_percep_loss_args a) {
    __shared__ float red[kThreads / 32];
    pdl_trigger();
    pdl_wait();
    float acc = 0.f;
    for (int k = 0; k < a.feats; ++k) {
        float s = 0.f;
        for (int i = a.offset[k] + threadIdx.x; i < a.offset[k + 1]; i += kThreads) s += a.partial[i];
        s = block_sum(s, red);
        if (threadIdx.x == 0) {
            const float v = a.crit == VMB_PERCEP_FRO ? sqrtf(s) : __fdiv_rn(s, (float)a.numel[k]);
            a.value[k] = v;
            acc += v * a.weight[k];
        }
    }
    if (threadIdx.x == 0) *a.loss = acc * a.perceptual_weight;
}

// ---- backward of one stage, x half only: dpre = [pre > 0] (pool adjoint of g_in, or g_in, + relu-feature term) + conv-feature term
template <typename T>
__global__ void __launch_bounds__(kThreads) stage_bwd_kernel(const vmb_percep_stage_bwd_args a) {
    pdl_trigger();
    pdl_wait();
    const int H = a.H, W = a.W, Hc = (H + 1) / 2, Wc = (W + 1) / 2, Hp = H / 2, Wp = W / 2, crit = a.crit;
    const int64_t cells = (int64_t)a.B * a.C * Hc * Wc;
    // the loss gradient's factor at each site: g pw w_k / N_k (l1), 2 g pw w_k / N_k (l2), g pw w_k / |d|_F (fro; 0 where |d| = 0)
    float cf[3];
    const float g = *a.grad_loss;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        cf[k] = 0.f;
        if (!a.feat[k]) continue;
        cf[k] = g * a.scale[k];
        if (crit == VMB_PERCEP_FRO) {
            const float nrm = a.value[a.feat_index[k]];
            cf[k] = nrm > 0.f ? __fdiv_rn(cf[k], nrm) : 0.f;
        }
    }
    for (int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x; t < cells; t += (int64_t)gridDim.x * kThreads) {
        const int cj = (int)(t % Wc);
        const int64_t r = t / Wc;
        const int ci = (int)(r % Hc);
        const int64_t pl = r / Hc;
        bool in[4];
        int64_t idx[4];
        float dp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int y = 2 * ci + e / 2, x = 2 * cj + e % 2;
            in[e] = y < H && x < W;
            idx[e] = (pl * H + y) * W + x;
        }
        const uint32_t code = a.relu ? a.code[t] : 0xfu;
        if (a.pool) {
            if (in[3]) {  // the pooled element's gradient goes to the window's argmax
                const int64_t p = (pl * Hp + ci) * Wp + cj;
                float d = a.g_in ? ld<T>(a.g_in, p) : 0.f;
                if (a.feat[2])
                    d += cf[2] * (crit == VMB_PERCEP_L1 ? sign_of(static_cast<const uint8_t*>(a.save[2])[p])
                                                        : static_cast<const float*>(a.save[2])[p]);
                const uint32_t am = (code >> 4) & 3u;
#pragma unroll
                for (int e = 0; e < 4; ++e) dp[e] = am == (uint32_t)e ? d : 0.f;
            }
        } else if (a.g_in) {
#pragma unroll
            for (int e = 0; e < 4; ++e) dp[e] = in[e] ? ld<T>(a.g_in, idx[e]) : 0.f;
        }
        const uint32_t c0 = a.feat[0] && crit == VMB_PERCEP_L1 ? static_cast<const uint8_t*>(a.save[0])[t] : 0u;
        const uint32_t c1 = a.feat[1] && crit == VMB_PERCEP_L1 ? static_cast<const uint8_t*>(a.save[1])[t] : 0u;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            if (!in[e]) continue;
            float d = dp[e];
            if (a.feat[1])
                d += cf[1] * (crit == VMB_PERCEP_L1 ? sign_of(c1 >> (2 * e)) : static_cast<const float*>(a.save[1])[idx[e]]);
            d = (code >> e) & 1u ? d : 0.f;
            if (a.feat[0])
                d += cf[0] * (crit == VMB_PERCEP_L1 ? sign_of(c0 >> (2 * e)) : static_cast<const float*>(a.save[0])[idx[e]]);
            st<T>(a.g_out, idx[e], d);
        }
    }
}

bool percep_dtype_ok(int dt) { return dt == VMB_F32 || dt == VMB_BF16; }
bool crit_ok(int c) { return c == VMB_PERCEP_L1 || c == VMB_PERCEP_L2 || c == VMB_PERCEP_FRO; }

unsigned grid_1d(int64_t n) {
    const int64_t g = (n + kThreads - 1) / kThreads, cap = 16 * (int64_t)num_sms();
    return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace

}  // namespace vmb

using namespace vmb;

extern "C" int vmb_percep_norm(const vmb_percep_norm_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->x && a->gt && a->out, "percep_norm: null pointer");
    VMB_CHECK(percep_dtype_ok(a->dtype), "percep_norm: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->B >= 1 && a->H >= 1 && a->W >= 1, "percep_norm: empty input (%d x 3 x %d x %d)", a->B, a->H, a->W);
    VMB_CHECK((a->mean == nullptr) == (a->std == nullptr), "percep_norm: mean and std go together");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(2 * (int64_t)a->B * 3 * a->H * a->W));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(norm_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(norm_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_percep_norm_bwd(const vmb_percep_norm_bwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->g && a->dx, "percep_norm_bwd: null pointer");
    VMB_CHECK(percep_dtype_ok(a->dtype), "percep_norm_bwd: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->B >= 1 && a->H >= 1 && a->W >= 1, "percep_norm_bwd: empty input (%d x 3 x %d x %d)", a->B, a->H, a->W);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d((int64_t)a->B * 3 * a->H * a->W));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(norm_bwd_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(norm_bwd_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_percep_stage_ctas(int B, int C, int H, int W) {
    if (B < 1 || C < 1 || H < 1 || W < 1) return -1;
    return (int)stage_ctas(B, C, H, W);
}

extern "C" int vmb_percep_stage(const vmb_percep_stage_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->y, "percep_stage: null pointer");
    VMB_CHECK(percep_dtype_ok(a->dtype), "percep_stage: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(crit_ok(a->crit), "percep_stage: criterion %d", a->crit);
    VMB_CHECK(a->B >= 1 && a->C >= 1 && a->H >= 1 && a->W >= 1, "percep_stage: empty input");
    VMB_CHECK(!a->pool || (a->relu && a->pooled && a->H >= 2 && a->W >= 2), "percep_stage: a pool needs a ReLU, an output and 2 x 2");
    VMB_CHECK(!a->feat[1] || a->relu, "percep_stage: a relu feature without the ReLU");
    VMB_CHECK(!a->feat[2] || a->pool, "percep_stage: a pool feature without the pool");
    for (int k = 0; k < 3; ++k) VMB_CHECK(!a->feat[k] || a->partial[k], "percep_stage: feature %d has no partials", k);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(stage_ctas(a->B, a->C, a->H, a->W));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(stage_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(stage_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_percep_loss(const vmb_percep_loss_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->partial && a->loss && a->value, "percep_loss: null pointer");
    VMB_CHECK(crit_ok(a->crit), "percep_loss: criterion %d", a->crit);
    VMB_CHECK(a->feats >= 1 && a->feats <= VMB_PERCEP_MAX_FEATS, "percep_loss: %d features not in 1..%d", a->feats,
              VMB_PERCEP_MAX_FEATS);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    VMB_CUDA(launch_pdl(loss_kernel, dim3(1), dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_percep_stage_bwd(const vmb_percep_stage_bwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->g_out && a->grad_loss, "percep_stage_bwd: null pointer");
    VMB_CHECK(percep_dtype_ok(a->dtype), "percep_stage_bwd: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(crit_ok(a->crit), "percep_stage_bwd: criterion %d", a->crit);
    VMB_CHECK(a->B >= 1 && a->C >= 1 && a->H >= 1 && a->W >= 1, "percep_stage_bwd: empty input");
    VMB_CHECK(!a->relu || a->code, "percep_stage_bwd: a ReLU needs its codes");
    VMB_CHECK(!a->pool || a->relu, "percep_stage_bwd: a pool needs a ReLU");
    VMB_CHECK(!a->feat[1] || a->relu, "percep_stage_bwd: a relu feature without the ReLU");
    VMB_CHECK(!a->feat[2] || a->pool, "percep_stage_bwd: a pool feature without the pool");
    for (int k = 0; k < 3; ++k) {
        VMB_CHECK(!a->feat[k] || a->save[k], "percep_stage_bwd: feature %d has nothing saved", k);
        VMB_CHECK(!a->feat[k] || a->crit != VMB_PERCEP_FRO || (a->value && a->feat_index[k] >= 0 &&
                  a->feat_index[k] < VMB_PERCEP_MAX_FEATS), "percep_stage_bwd: feature %d has no norm", k);
    }
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d((int64_t)a->B * a->C * ((a->H + 1) / 2) * ((a->W + 1) / 2)));
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(stage_bwd_kernel<float>, grid, dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(stage_bwd_kernel<__nv_bfloat16>, grid, dim3(kThreads), 0, s, *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
