// TMA (cp.async.bulk.tensor) + mbarrier helpers for sm_90a, and the host-side tensor-map encoder.
// The library links only cudart: cuTensorMapEncodeTiled is fetched at run time through cudaGetDriverEntryPoint
// (the library builds on hosts without a driver; where it runs, the driver is present).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace vmb {

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbarrier_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarrier_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbarrier_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarrier_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(smem_addr(bar)),
        "r"(parity)
        : "memory");
}
// generic-proxy accesses of shared memory (LDS/STS) ordered before subsequent async-proxy (TMA) accesses
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 4-D tiled box load: coordinates innermost first (c0 = contiguous dimension); out-of-bounds elements are zero-filled
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_addr(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---- host ----
inline int dtype_to_tmap(int dtype, CUtensorMapDataType* out) {
    switch (dtype) {
        case VMB_F32: *out = CU_TENSOR_MAP_DATA_TYPE_FLOAT32; return VMB_OK;
        case VMB_BF16: *out = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; return VMB_OK;
        case VMB_F16: *out = CU_TENSOR_MAP_DATA_TYPE_FLOAT16; return VMB_OK;
    }
    return VMB_ERR_INVALID;
}

// 4-D tensor (d0 contiguous).  stride_k = element stride of dimension k (k = 1..3), box_k = box extent.  Dimensions of extent 1 may
// carry any stride.  Requires a 16 B-aligned base and byte strides that are multiples of 16 (the caller checked: vec_ok).
// swizzle: 0 none, 1 / 2 / 3 = CU_TENSOR_MAP_SWIZZLE_32B / 64B / 128B (the box's innermost extent must span at most that many bytes).
int make_tmap_4d(CUtensorMap* map, int dtype, const void* base, const uint64_t dims[4], const int64_t strides_elts[3],
                 const uint32_t box[4], int swizzle = 0);

}  // namespace vmb
