// tma.cuh -- bulk async copies (TMA engine, SASS UBLKCP) + mbarrier helpers, inline PTX for sm_90a.
// 1-D copies stage whole image-observation rows through shared memory: global -> shared (mbarrier complete_tx),
// shared -> global (bulk_group).  Addresses and sizes must be multiples of 16 bytes.  2-D copies move boxes of a tensor
// map; pb_tma_map_128 builds the map of the fp32 [rows][128] matrices that the wgmma kernels tile.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "pb_common.cuh"

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: try_wait suspends for a HW-defined interval per call; if the phase has not completed after ~4M
// attempts (seconds) something is broken (bad address, wrong byte count) -- trap instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
#pragma unroll 1
    for (uint32_t spins = 0; spins < (1u << 22); ++spins) {
        uint32_t ok;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(addr), "r"(parity)
            : "memory");
        if (ok) return;
    }
    __trap();
}
// global -> shared, completion signalled on an mbarrier (transaction bytes)
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global, tracked by the bulk async-group of the issuing thread
__device__ __forceinline__ void tma_store_1d(void* dst_gmem, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)),
                 "r"(bytes)
                 : "memory");
}
// global -> shared: the box of `map` at coordinates (c0 innermost, c1), completion signalled on an mbarrier
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
// shared -> global: one box of `map`, tracked by the bulk async-group of the issuing thread
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                     reinterpret_cast<uint64_t>(map)),
                 "r"(c0), "r"(c1), "r"(smem_u32(src))
                 : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_wait_read() {  // shared-memory sources of all but the N newest groups are free
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_wait_all() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// make generic-proxy writes to shared memory visible to the async proxy (before a bulk store reads them)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Host: the 2-D tensor map of a [rows][128] fp32 matrix whose rows are row_stride floats apart, in boxes of [box_rows][32
// floats] with the 128-byte swizzle (the K-major SWIZZLE_128B tiles of wgmma.cuh).  PB_OK, or PB_ERR_CUDA with the message
// set when the driver entry point is missing or refuses the map.
inline int pb_tma_map_128(CUtensorMap* map, const float* base, int64_t rows, int64_t row_stride, int box_rows) {
    typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    PB_REQUIRE(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) == cudaSuccess && fn &&
                   qr == cudaDriverEntryPointSuccess,
               PB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    const cuuint64_t dims[2] = {128, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)row_stride * 4};
    const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = ((EncodeTiledFn)fn)(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides,
                                           box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_REQUIRE(r == CUDA_SUCCESS, PB_ERR_CUDA, "cuTensorMapEncodeTiled failed: %d", (int)r);
    return PB_OK;
}
