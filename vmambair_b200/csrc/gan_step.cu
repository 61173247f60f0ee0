// The GAN training step's own kernels (vmambair_b200.gan_train): the pixel loss and the logit means as a two-level sum, the
// generator's output-gradient junction of its three losses, the learning-rate schedule of both optimizers from the device's
// iteration counter (step decay and MultiStepLR, or cosine annealing with restarts for vmambair_b200.restore_train), and the EMA
// for iterations that skip the generator's optimizer step.  Every reduction has one fixed order (the grid depends on n alone) and
// there are no atomics, so the results are bitwise repeatable; all math is fp32, tensors are fp32 or bf16 (VMB_F32 / VMB_BF16).
// Nothing reads the host, so the step can be captured in a CUDA graph.
#include <math.h>

#include "common.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxCtas = 512;  // partials of the two-level sum; the second pass adds them in one CTA

template <typename T> __device__ __forceinline__ float ld(const void* p, int64_t i) { return to_f32<T>(static_cast<const T*>(p)[i]); }

// sum of v over the CTA in one fixed order (butterfly within each warp, then thread 0 adds the warp sums in index order); every
// thread gets the result.  `red` holds kThreads / 32 + 1 floats.
__device__ float block_sum(float v, float* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kThreads / 32; ++w) s += red[w];
        red[kThreads / 32] = s;
    }
    __syncthreads();
    return red[kThreads / 32];
}

unsigned grid_1d(int64_t n, int64_t cap) {
    const int64_t g = (n + kThreads - 1) / kThreads;
    return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

bool dtype_ok(int dt) { return dt == VMB_F32 || dt == VMB_BF16; }

// ---- weight mean(|x - y|) or weight mean(x) ----
template <typename T>
__global__ void __launch_bounds__(kThreads) mean_partial_kernel(const vmb_mean_loss_args a) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    float s = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads)
        s += a.y ? fabsf(ld<T>(a.x, i) - ld<T>(a.y, i)) : ld<T>(a.x, i);
    s = block_sum(s, red);
    if (threadIdx.x == 0) static_cast<float*>(a.workspace)[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kThreads) mean_final_kernel(const vmb_mean_loss_args a, int parts) {
    __shared__ float red[kThreads / 32 + 1];
    pdl_trigger();
    pdl_wait();
    const float* ws = static_cast<const float*>(a.workspace);
    float s = 0.f;
    for (int i = threadIdx.x; i < parts; i += kThreads) s += ws[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) *a.out = __fdiv_rn(s, (float)a.n) * a.weight;
}

// ---- dout = w_pix sign(out - gt) / n + g_percep + g_gan ----
template <typename Tin, typename Tout>
__global__ void __launch_bounds__(kThreads) out_grad_kernel(const vmb_gan_out_grad_args a) {
    pdl_trigger();
    pdl_wait();
    const float scale = __fdiv_rn(a.w_pix, (float)a.n);
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kThreads) {
        const float d = ld<Tin>(a.out, i) - ld<Tin>(a.gt, i);
        float g = d > 0.f ? scale : (d < 0.f ? -scale : 0.f);
        if (a.g_percep) g += a.g_percep[i];
        if (a.g_gan) g += a.g_gan[i];
        static_cast<Tout*>(a.dout)[i] = from_f32<Tout>(g);
    }
}

template <typename Tin>
int out_grad_launch(const vmb_gan_out_grad_args& a, dim3 grid, cudaStream_t s) {
    if (a.out_dtype == VMB_F32)
        VMB_CUDA(launch_pdl(out_grad_kernel<Tin, float>, grid, dim3(kThreads), 0, s, a));
    else
        VMB_CUDA(launch_pdl(out_grad_kernel<Tin, __nv_bfloat16>, grid, dim3(kThreads), 0, s, a));
    return VMB_OK;
}

// ---- learning-rate schedule ----
// basicsr's cosine annealing with restarts at last_epoch e (lr_scheduler.py:115-235), in Python's order of evaluation: no
// contraction into fma, so the double result is the host's up to cos()'s last bit
__device__ float cosine_lr(const vmb_lr_rule& r, int64_t e) {
    int64_t start = 0;
    for (int j = 0; j < r.n_periods; ++j) {
        if (e <= start + r.periods[j]) {
            const double eta = r.eta_mins[j];
            const double t = __ddiv_rn((double)(e - start), (double)r.periods[j]);
            const double c = __dadd_rn(1.0, cos(__dmul_rn(M_PI, t)));
            return (float)__dadd_rn(eta, __dmul_rn(__dmul_rn(__dmul_rn(r.restart_weights[j], 0.5), __dadd_rn(r.base, -eta)), c));
        }
        start += r.periods[j];
    }
    return __int_as_float(0x7fc00000);  // past the last period: the reference has no lr
}

__device__ float rule_lr(const vmb_lr_rule& r, int64_t it) {
    if (r.n_periods > 0) return cosine_lr(r, it - 1);
    double lr = r.base;
    if (r.step_size > 0) lr *= pow(r.step_gamma, (double)(it / r.step_size));
    int passed = 0;
    for (int k = 0; k < r.n_milestones; ++k) passed += r.milestones[k] <= it - 1;
    if (passed) lr *= pow(r.milestone_gamma, (double)passed);
    return (float)lr;
}

__global__ void lr_schedule_kernel(const vmb_lr_schedule_args a) {
    pdl_trigger();
    pdl_wait();
    const int64_t it = *a.iter + 1;
    *a.iter = it;
    for (int k = 0; k < a.n_rules; ++k) a.lr[k] = rule_lr(a.rule[k], it);
}

// ---- EMA alone, vmb_fused_adam's formula ----
__global__ void __launch_bounds__(kThreads) ema_kernel(float* __restrict__ ema, const float* __restrict__ param, int64_t n, float decay) {
    pdl_trigger();
    pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
        ema[i] = fmaf(decay, ema[i], (1.f - decay) * param[i]);
}

}  // namespace

}  // namespace vmb

using namespace vmb;

extern "C" int64_t vmb_mean_loss_workspace_bytes(int64_t n) { return (int64_t)grid_1d(n, kMaxCtas) * (int64_t)sizeof(float); }

extern "C" int vmb_mean_loss(const vmb_mean_loss_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->x && a->out && a->workspace, "mean_loss: null pointer");
    VMB_CHECK(dtype_ok(a->dtype), "mean_loss: dtype %d is not fp32 or bf16", a->dtype);
    VMB_CHECK(a->n >= 1, "mean_loss: empty input");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned parts = grid_1d(a->n, kMaxCtas);
    if (a->dtype == VMB_F32)
        VMB_CUDA(launch_pdl(mean_partial_kernel<float>, dim3(parts), dim3(kThreads), 0, s, *a));
    else
        VMB_CUDA(launch_pdl(mean_partial_kernel<__nv_bfloat16>, dim3(parts), dim3(kThreads), 0, s, *a));
    VMB_CUDA(launch_pdl(mean_final_kernel, dim3(1), dim3(kThreads), 0, s, *a, (int)parts));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_gan_out_grad(const vmb_gan_out_grad_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->out && a->gt && a->dout, "gan_out_grad: null pointer");
    VMB_CHECK(dtype_ok(a->in_dtype) && dtype_ok(a->out_dtype), "gan_out_grad: dtypes %d, %d are not fp32 or bf16", a->in_dtype,
              a->out_dtype);
    VMB_CHECK(a->n >= 1, "gan_out_grad: empty input");
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const dim3 grid(grid_1d(a->n, 16 * num_sms()));
    const int st = a->in_dtype == VMB_F32 ? out_grad_launch<float>(*a, grid, s) : out_grad_launch<__nv_bfloat16>(*a, grid, s);
    if (st != VMB_OK) return st;
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_lr_schedule(const vmb_lr_schedule_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->iter && a->lr, "lr_schedule: null pointer");
    VMB_CHECK(a->n_rules >= 1 && a->n_rules <= 2, "lr_schedule: %d rules, not 1 or 2", a->n_rules);
    for (int k = 0; k < a->n_rules; ++k)
        VMB_CHECK(a->rule[k].base >= 0.f && a->rule[k].n_milestones >= 0 && a->rule[k].n_milestones <= VMB_LR_MAX_MILESTONES,
                  "lr_schedule: rule %d has base %g and %d milestones (at most %d)", k, a->rule[k].base,
                  a->rule[k].n_milestones, VMB_LR_MAX_MILESTONES);
    for (int k = 0; k < a->n_rules; ++k) {
        VMB_CHECK(a->rule[k].n_periods >= 0 && a->rule[k].n_periods <= VMB_LR_MAX_PERIODS, "lr_schedule: rule %d has %d periods (at most %d)",
                  k, a->rule[k].n_periods, VMB_LR_MAX_PERIODS);
        for (int j = 0; j < a->rule[k].n_periods; ++j)
            VMB_CHECK(a->rule[k].periods[j] >= 1, "lr_schedule: rule %d period %d is %lld", k, j, (long long)a->rule[k].periods[j]);
    }
    VMB_CUDA(launch_pdl(lr_schedule_kernel, dim3(1), dim3(1), 0, static_cast<cudaStream_t>(stream), *a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

extern "C" int vmb_ema_update(float* ema, const float* param, int64_t n, float decay, void* stream) {
    VMB_CHECK(ema && param, "ema_update: null pointer");
    VMB_CHECK(n >= 1 && decay >= 0.f && decay <= 1.f, "ema_update: n %lld, decay %g", (long long)n, (double)decay);
    VMB_CUDA(launch_pdl(ema_kernel, dim3(grid_1d(n, 8 * num_sms())), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), ema, param,
                        n, decay));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
