// The restoration training step's input preparation (vmambair_b200.restore_train): Restormer's progressive subset and crop and
// ImageCleanModel's mixup, for lq and gt in one launch, written straight into the step's (or its CUDA graph's) input buffers.
// Every draw is made on the host; the indices, window origins and lam travel in the argument struct, so nothing reads the host.
#include "common.cuh"

namespace vmb {

namespace {

constexpr int kThreads = 256;

// one thread per output element of both tensors; the element's tensor, image, channel, row and column follow from its linear index
__global__ void __launch_bounds__(kThreads) crop_mix_kernel(const vmb_batch_crop_mix_args a, int64_t n0, int64_t n_all) {
    pdl_trigger();
    pdl_wait();
    for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < n_all; e += (int64_t)gridDim.x * kThreads) {
        const int k = e >= n0;
        const vmb_crop_mix_tensor& t = a.t[k];
        int64_t r = k ? e - n0 : e;
        const int x = (int)(r % t.w);
        r /= t.w;
        const int y = (int)(r % t.h);
        r /= t.h;
        const int c = (int)(r % t.c);
        const int i = (int)(r / t.c);
        const int64_t pix = (int64_t)c * t.stride_c + (int64_t)(t.row0 + y) * t.stride_h + (int64_t)(t.col0 + x) * t.stride_w;
        float v = t.src[(int64_t)a.idx[i] * t.stride_n + pix];
        if (a.mix) {
            // torch: lam * s (fp32 product), (1 - lam) * s[perm] (fp32 product), then their fp32 sum -- no fma
            const float b = t.src[(int64_t)a.idx[a.perm[i]] * t.stride_n + pix];
            v = __fadd_rn(__fmul_rn(a.lam, v), __fmul_rn(a.one_minus_lam, b));
        }
        t.dst[(k ? e - n0 : e)] = v;
    }
}

}  // namespace

}  // namespace vmb

using namespace vmb;

extern "C" int vmb_batch_crop_mix(const vmb_batch_crop_mix_args* a, void* stream) {
    VMB_CHECK(a != nullptr, "batch_crop_mix: null arguments");
    VMB_CHECK(a->n_tensors >= 1 && a->n_tensors <= 2, "batch_crop_mix: %d tensors, not 1 or 2", a->n_tensors);
    VMB_CHECK(a->batch >= 1 && a->batch <= VMB_CROP_MIX_MAX_IMAGES, "batch_crop_mix: batch %d, 1 to %d", a->batch,
              VMB_CROP_MIX_MAX_IMAGES);
    for (int i = 0; i < a->batch; ++i)
        VMB_CHECK(a->idx[i] >= 0 && a->perm[i] >= 0 && a->perm[i] < a->batch, "batch_crop_mix: image %d has idx %d, perm %d", i,
                  a->idx[i], a->perm[i]);
    int64_t n[2] = {0, 0};
    for (int k = 0; k < a->n_tensors; ++k) {
        const vmb_crop_mix_tensor& t = a->t[k];
        VMB_CHECK(t.src && t.dst, "batch_crop_mix: tensor %d has a null pointer", k);
        VMB_CHECK(t.c >= 1 && t.h >= 1 && t.w >= 1 && t.row0 >= 0 && t.col0 >= 0, "batch_crop_mix: tensor %d window %dx%dx%d at (%d, %d)",
                  k, t.c, t.h, t.w, t.row0, t.col0);
        n[k] = (int64_t)a->batch * t.c * t.h * t.w;
    }
    const int64_t n_all = n[0] + n[1];
    const int64_t g = (n_all + kThreads - 1) / kThreads, cap = 16 * (int64_t)num_sms();
    VMB_CUDA(launch_pdl(crop_mix_kernel, dim3((unsigned)(g < cap ? g : cap)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), *a,
                        n[0], n_all));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
