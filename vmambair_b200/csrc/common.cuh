// Shared device helpers for the vmambair_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vmambair_b200.h"

namespace vmb {

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// ---- error plumbing (thread-local message, returned through vmb_last_error()) ----
void set_error(const char* fmt, ...);
#define VMB_CHECK(cond, ...)                         \
    do {                                             \
        if (!(cond)) {                               \
            ::vmb::set_error(__VA_ARGS__);           \
            return VMB_ERR_INVALID;                  \
        }                                            \
    } while (0)
#define VMB_CUDA(expr)                                                           \
    do {                                                                         \
        cudaError_t e_ = (expr);                                                 \
        if (e_ != cudaSuccess) {                                                 \
            ::vmb::set_error("%s failed: %s", #expr, cudaGetErrorString(e_));    \
            return VMB_ERR_CUDA;                                                 \
        }                                                                        \
    } while (0)

// ---- programmatic dependent launch (PDL) ----
// Every kernel of the library starts with pdl_trigger(); pdl_wait();  -- the next kernel of the stream / graph may become
// resident while this one drains (its launch latency and whatever it does before its own pdl_wait() overlap our tail);
// pdl_wait() returns once the preceding kernel has completed and its writes are visible, so nothing that depends on it
// (and no global store) may precede the wait.  Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
int num_sms();  // SMs of the current device, read once (launch heuristics size their grids by it)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ---- scalar conversions ----
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// ---- math ----
__device__ __forceinline__ float ex2(float x) {  // MUFU.EX2, 2 ulp, flushes denormals
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float lg2(float x) {
    float y;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// softplus with the reference's threshold (fwd kernel :117: x<=20 ? log1p(exp(x)) : x).
// e=exp(x) by MUFU; log1p(e) by a degree-6 series when e is small (keeps full relative
// precision for the tiny dt's the model initialises to), else ln2*lg2(1+e).
__device__ __forceinline__ float softplus_f(float x) {
    const float e = ex2(x * kLog2e);
    float small = e * (1.f + e * (-0.5f + e * (0.33333334f + e * (-0.25f + e * (0.2f + e * (-0.16666667f))))));
    float big = kLn2 * lg2(1.f + e);
    float r = e < 0.03125f ? small : big;
    return x <= 20.f ? r : x;
}
__device__ __forceinline__ float sigmoid_f(float x) { return rcp_approx(1.f + ex2(-x * kLog2e)); }

// two-lane helpers: sm_90 has no packed f32x2 FMA, so each lane is one round-to-nearest FFMA / FMUL / FADD
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

__device__ __forceinline__ float2 shfl_up2(float2 v, int delta) {
    return make_float2(__shfl_up_sync(0xffffffffu, v.x, delta), __shfl_up_sync(0xffffffffu, v.y, delta));
}
__device__ __forceinline__ float2 shfl_down2(float2 v, int delta) {
    return make_float2(__shfl_down_sync(0xffffffffu, v.x, delta), __shfl_down_sync(0xffffffffu, v.y, delta));
}

// ---- vector global access (read-only / streaming) ----
__device__ __forceinline__ uint4 ldg128(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void stg128(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }

// unpack 8 16-bit elements (one uint4) to fp32
template <typename T> __device__ __forceinline__ void unpack8(uint4 v, float* f);
template <> __device__ __forceinline__ void unpack8<__nv_bfloat16>(uint4 v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        f[2 * i] = __uint_as_float(w[i] << 16);
        f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
}
template <> __device__ __forceinline__ void unpack8<__half>(uint4 v, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
    __half2 t = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
}

// Load `n` (<= VEC) consecutive elements starting at p into f[]; vectorised when allowed.
// VEC = 16/sizeof(T) elements per 128-bit access.
template <typename T> struct Vec { static constexpr int N = 16 / sizeof(T); };

template <typename T>
__device__ __forceinline__ void load_vec(const T* __restrict__ p, float* f, int valid, bool aligned) {
    constexpr int V = Vec<T>::N;
    if (aligned && valid >= V) {
        uint4 v = ldg128(p);
        if constexpr (sizeof(T) == 4) {
            f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
            f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
        } else {
            unpack8<T>(v, f);
        }
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i) f[i] = i < valid ? to_f32<T>(p[i]) : 0.f;
    }
}
// same, from shared memory (always 16 B aligned, always full)
template <typename T>
__device__ __forceinline__ void load_vec_smem(const T* p, float* f) {
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    if constexpr (sizeof(T) == 4) {
        f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
        f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
    } else {
        unpack8<T>(v, f);
    }
}
template <typename T>
__device__ __forceinline__ void store_vec(T* __restrict__ p, const float* f, int valid, bool aligned) {
    constexpr int V = Vec<T>::N;
    if (aligned && valid >= V) {
        uint4 v;
        if constexpr (sizeof(T) == 4) {
            v.x = __float_as_uint(f[0]); v.y = __float_as_uint(f[1]);
            v.z = __float_as_uint(f[2]); v.w = __float_as_uint(f[3]);
        } else {
            v.x = pack2<T>(f[0], f[1]); v.y = pack2<T>(f[2], f[3]);
            v.z = pack2<T>(f[4], f[5]); v.w = pack2<T>(f[6], f[7]);
        }
        stg128(p, v);
    } else {
#pragma unroll
        for (int i = 0; i < V; ++i)
            if (i < valid) p[i] = from_f32<T>(f[i]);
    }
}

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

}  // namespace vmb
