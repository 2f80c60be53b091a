// pb_common.cuh -- shared helpers for libpuffer_b200.so (sm_90a only; no other arch is supported).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "pufferlib_b200.h"

void pb_set_error(const char* fmt, ...);

#define PB_CUDA(expr)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            pb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));    \
            return PB_ERR_CUDA;                                                                    \
        }                                                                                          \
    } while (0)

#define PB_REQUIRE(cond, code, ...)      \
    do {                                 \
        if (!(cond)) {                   \
            pb_set_error(__VA_ARGS__);   \
            return (code);               \
        }                                \
    } while (0)

extern unsigned long long g_pb_launches;  // kernels launched by this library (host-side count)
#define PB_LAUNCH_CHECK()            \
    do {                             \
        ++g_pb_launches;             \
        PB_CUDA(cudaGetLastError()); \
    } while (0)

static inline int64_t pb_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
#ifdef __CUDACC__
__device__ __forceinline__ int64_t pb_ceil_div_dev(int64_t a, int64_t b) { return (a + b - 1) / b; }
#endif

// SM count of the current device (H100 SXM: 132), queried once per device; grids are sized in multiples of it
int pb_num_sms();
#define PB_NUM_SMS (pb_num_sms())

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t pb_ld_acquire(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void pb_st_release(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// streaming (evict-first) stores for write-once rollout data
__device__ __forceinline__ void pb_st_cs(float* p, float v) { __stcs(p, v); }
__device__ __forceinline__ void pb_st_cs(float4* p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ void pb_st_cs(uint4* p, uint4 v) { __stcs(p, v); }

// splitmix64 finaliser: the counter-based RNG of the builder-specified envs (oracle/SPEC.md §rng)
__host__ __device__ __forceinline__ uint32_t pb_mix32(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return (uint32_t)(x >> 32);
}
#endif
