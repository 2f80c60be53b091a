// reduce_partials.cuh -- the deterministic second stage of the kernels that split a row reduction across CTAs into fp32
// partial rows (mlp_tail.cu, nature_conv1.cu).
#pragma once
#include <stdint.h>

namespace {

// out[j] = sum over blocks of partials[b][j], j < n (n <= pstride, the distance between partial rows).  One warp per
// output element: lane l sums blocks l, l+32, ... in order, then a fixed shuffle tree combines the 32 lane sums (same
// order every run).
__global__ void __launch_bounds__(256) k_reduce_partials(const float* __restrict__ partials, int n_blocks, int pstride,
                                                        int n, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= n) return;
    float s = 0.f;
    for (int b = lane; b < n_blocks; b += 32) s += partials[(int64_t)b * pstride + j];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) out[j] = s;
}

}  // namespace
