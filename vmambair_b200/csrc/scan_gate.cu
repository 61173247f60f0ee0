// Backward of the z gate of the gated selective-scan forward (vmb_scan_gate_bwd; mamba_ssm's selective_scan_cuda.bwd evaluates the
// same terms inside its scan backward kernel).  Element-wise, fp32 math: with s = sigmoid(z),
//   dout_eff = dout * z * s   (fp32: the scan backward reads it without rounding, dout_f32)
//   dz       = dout * out * s * (1 + z (1 - s))
//   out_z    = out * z * s    (optional: the reference's recompute_out_z)
// Thread = 8 consecutive positions of one row, 16 B vectors where the rows allow them.
#include "scan_common.cuh"

namespace vmb {

constexpr int kGateEpt = 8;  // positions per thread

template <typename T>
__device__ __forceinline__ void load8(const T* p, float* f, int valid, bool ok) {
    constexpr int V = Vec<T>::N;
#pragma unroll
    for (int v = 0; v < kGateEpt / V; ++v) load_vec<T>(p + v * V, f + v * V, valid - v * V, ok);
}
template <typename T>
__device__ __forceinline__ void store8(T* p, const float* f, int valid, bool ok) {
    constexpr int V = Vec<T>::N;
#pragma unroll
    for (int v = 0; v < kGateEpt / V; ++v) store_vec<T>(p + v * V, f + v * V, valid - v * V, ok);
}

template <typename in_t>
__global__ void __launch_bounds__(256) scan_gate_bwd_kernel(const vmb_scan_gate_args a, bool vec_ok) {
    pdl_trigger();
    pdl_wait();
    const int cpr = (a.seqlen + kGateEpt - 1) / kGateEpt;  // thread items per row
    const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (item >= (int64_t)a.batch * a.dim * cpr) return;
    const int row = (int)(item / cpr), l0 = (int)(item % cpr) * kGateEpt;
    const int b = row / a.dim, d = row % a.dim;
    const int valid = a.seqlen - l0;
    float g[kGateEpt], o[kGateEpt], z[kGateEpt], de[kGateEpt], dz[kGateEpt];
    load8<in_t>(reinterpret_cast<const in_t*>(a.dout) + (int64_t)b * a.dout_bs + (int64_t)d * a.dout_ds + l0, g, valid, vec_ok);
    load8<in_t>(reinterpret_cast<const in_t*>(a.out) + (int64_t)b * a.out_bs + (int64_t)d * a.out_ds + l0, o, valid, vec_ok);
    load8<in_t>(reinterpret_cast<const in_t*>(a.z) + (int64_t)b * a.z_bs + (int64_t)d * a.z_ds + l0, z, valid, vec_ok);
#pragma unroll
    for (int i = 0; i < kGateEpt; ++i) {
        const float s = 1.f / (1.f + __expf(-z[i]));
        const float silu = silu_gate(z[i]);
        de[i] = g[i] * silu;
        dz[i] = g[i] * o[i] * s * (1.f + z[i] * (1.f - s));
        o[i] = o[i] * silu;
    }
    store8<float>(a.dout_eff + (int64_t)row * a.seqlen + l0, de, valid, vec_ok);
    store8<in_t>(reinterpret_cast<in_t*>(a.dz) + (int64_t)b * a.dz_bs + (int64_t)d * a.dz_ds + l0, dz, valid, vec_ok);
    if (a.out_z)
        store8<in_t>(reinterpret_cast<in_t*>(a.out_z) + (int64_t)b * a.out_z_bs + (int64_t)d * a.out_z_ds + l0, o, valid, vec_ok);
}

int scan_gate_bwd_launch(const vmb_scan_gate_args& a, bool vec_ok, cudaStream_t stream) {
    const int64_t items = (int64_t)a.batch * a.dim * ((a.seqlen + kGateEpt - 1) / kGateEpt);
    const int64_t blocks = (items + 255) / 256;
    VMB_CHECK(blocks < (1LL << 31), "scan_gate_bwd: too many elements");
    switch (a.dtype) {
        case VMB_F32: VMB_CUDA(launch_pdl(scan_gate_bwd_kernel<float>, dim3((unsigned)blocks), dim3(256), 0, stream, a, vec_ok)); break;
        case VMB_BF16: VMB_CUDA(launch_pdl(scan_gate_bwd_kernel<__nv_bfloat16>, dim3((unsigned)blocks), dim3(256), 0, stream, a, vec_ok)); break;
        case VMB_F16: VMB_CUDA(launch_pdl(scan_gate_bwd_kernel<__half>, dim3((unsigned)blocks), dim3(256), 0, stream, a, vec_ok)); break;
        default: set_error("scan_gate_bwd: unsupported dtype %d", a.dtype); return VMB_ERR_INVALID;
    }
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb
