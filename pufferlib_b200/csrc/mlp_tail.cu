// mlp_tail.cu -- backward of the policy's "tail" (ReLU -> action/value heads) in one pass over the hidden layer (sm_90a).
//
// The configured policy is models.Default (reference pufferlib/models.py:12-62): Linear(obs->H)+ReLU, then two
// heads H->n_act and H->1.  In train (clean_pufferl.py:193-244) the backward of everything after the encoder GEMM is
// memory-bound work on [M, H] tensors that ATen runs as five launches, each re-reading 268 MB at M = 524288:
//   dHidden = dOut @ W_heads           (skinny GEMM, 8 columns)         dW_heads = dOut^T @ hidden   (skinny GEMM)
//   db_heads = sum_rows dOut           dPre = dHidden * (hidden > 0)    db_enc = sum_rows dPre
// This kernel does all five reading `hidden` ONCE and writing dPre once (2 * 4H + 32 B per row).  The dense H x H
// encoder GEMMs (forward, and dW_enc = dPre^T @ obs) stay on cuBLAS tensor cores.
// A warp owns rows; lane l owns columns 4l..4l+3 (one float4 per row per lane, 512 B coalesced for H = 128); the
// head weights live in registers (NO x 4 per lane); per-lane accumulators (dW: NO x 4, db_enc: 4) are reduced over
// the block's warps in shared memory and written as ONE partial row per block; a second tiny kernel sums the
// partials in a fixed order (deterministic, no atomics).
#include "pb_common.cuh"
#include "tma.cuh"

namespace {

constexpr int NO = 8;          // padded number of head outputs (n_act + 1 <= 8)
constexpr int MT_THREADS = 256;
constexpr int MT_WARPS = MT_THREADS / 32;
constexpr int ROWS_PER_BLOCK = 512;

// partial layout per block: [NO*H] dW_heads | [H] db_enc | [NO] db_heads
template <int H>
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd(const float* __restrict__ dout, int64_t dout_stride,
                                                            const float* __restrict__ w_heads,   // [NO][H]
                                                            const float* __restrict__ hidden,    // [M][H] post-ReLU
                                                            float* __restrict__ dpre,            // [M][H]
                                                            float* __restrict__ partials, int64_t m) {
    static_assert(H % 128 == 0, "H must be a multiple of 128 (one or more float4 per lane)");
    constexpr int Q = H / 128;                  // float4s per lane per row
    constexpr int PSTRIDE = NO * H + H + NO;
    __shared__ float s_red[MT_WARPS][PSTRIDE > 2048 ? 1 : PSTRIDE];   // H = 128: 8 x 1160 floats = 37 KB
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    float4 w[NO][Q];
#pragma unroll
    for (int k = 0; k < NO; ++k)
#pragma unroll
        for (int q = 0; q < Q; ++q) w[k][q] = *reinterpret_cast<const float4*>(w_heads + (int64_t)k * H + 128 * q + 4 * lane);

    float4 acc_w[NO][Q], acc_b[Q];
    float acc_o[NO];
#pragma unroll
    for (int k = 0; k < NO; ++k) {
        acc_o[k] = 0.f;
#pragma unroll
        for (int q = 0; q < Q; ++q) acc_w[k][q] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) acc_b[q] = make_float4(0.f, 0.f, 0.f, 0.f);

    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
#pragma unroll 2
    for (int64_t r = row0 + warp; r < row_end; r += MT_WARPS) {
        // the row's 8 head gradients: every lane reads the same 32 bytes (broadcast)
        const float4 d0 = *reinterpret_cast<const float4*>(dout + r * dout_stride);
        const float4 d1 = *reinterpret_cast<const float4*>(dout + r * dout_stride + 4);
        const float d[NO] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
#pragma unroll
        for (int k = 0; k < NO; ++k) acc_o[k] += d[k];
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const float4 h = __ldcs(reinterpret_cast<const float4*>(hidden + r * H + 128 * q + 4 * lane));
            float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < NO; ++k) {
                g.x = fmaf(d[k], w[k][q].x, g.x); g.y = fmaf(d[k], w[k][q].y, g.y);
                g.z = fmaf(d[k], w[k][q].z, g.z); g.w = fmaf(d[k], w[k][q].w, g.w);
                acc_w[k][q].x = fmaf(d[k], h.x, acc_w[k][q].x); acc_w[k][q].y = fmaf(d[k], h.y, acc_w[k][q].y);
                acc_w[k][q].z = fmaf(d[k], h.z, acc_w[k][q].z); acc_w[k][q].w = fmaf(d[k], h.w, acc_w[k][q].w);
            }
            // ReLU backward (threshold_backward: gradient passes where the activation is > 0)
            g.x = h.x > 0.f ? g.x : 0.f; g.y = h.y > 0.f ? g.y : 0.f;
            g.z = h.z > 0.f ? g.z : 0.f; g.w = h.w > 0.f ? g.w : 0.f;
            acc_b[q].x += g.x; acc_b[q].y += g.y; acc_b[q].z += g.z; acc_b[q].w += g.w;
            __stcs(reinterpret_cast<float4*>(dpre + r * H + 128 * q + 4 * lane), g);
        }
    }
    // ---- block reduction: every warp deposits its partial, then the block sums the 8 deposits column-wise
    float* mine = s_red[warp];
#pragma unroll
    for (int k = 0; k < NO; ++k)
#pragma unroll
        for (int q = 0; q < Q; ++q) *reinterpret_cast<float4*>(mine + k * H + 128 * q + 4 * lane) = acc_w[k][q];
#pragma unroll
    for (int q = 0; q < Q; ++q) *reinterpret_cast<float4*>(mine + NO * H + 128 * q + 4 * lane) = acc_b[q];
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NO; ++k) mine[NO * H + H + k] = acc_o[k];
    __syncthreads();
    float* out = partials + (int64_t)blockIdx.x * PSTRIDE;
    for (int j = threadIdx.x; j < PSTRIDE; j += MT_THREADS) {
        float s = 0.f;
#pragma unroll
        for (int wq = 0; wq < MT_WARPS; ++wq) s += s_red[wq][j];
        out[j] = s;
    }
}

// TMA-staged variant (dout contiguous [M][8]): the hidden rows and their head gradients are pulled into a 4-stage
// shared-memory ring by cp.async.bulk (one elected thread, mbarrier complete_tx), 32 rows = 16 KiB + 1 KiB per stage,
// so ~64 KiB per CTA is in flight independently of the register budget; the warps consume from shared memory
// (conflict-free LDS.128) and stream dPre straight back to HBM.
constexpr int TT_STAGES = 4;
constexpr int TT_CHUNK = 32;   // rows per stage

template <int H>
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd_tma(const float* __restrict__ dout,      // [M][NO]
                                                                const float* __restrict__ w_heads,   // [NO][H]
                                                                const float* __restrict__ hidden,    // [M][H] post-ReLU
                                                                float* __restrict__ dpre,            // [M][H]
                                                                float* __restrict__ partials, int64_t m) {
    static_assert(H == 128, "one float4 per lane per row");
    constexpr int PSTRIDE = NO * H + H + NO;
    constexpr uint32_t H_BYTES = TT_CHUNK * H * 4, D_BYTES = TT_CHUNK * NO * 4;
    extern __shared__ __align__(128) unsigned char dyn[];
    float* s_h = reinterpret_cast<float*>(dyn);                                   // [STAGES][CHUNK][H]
    float* s_d = reinterpret_cast<float*>(dyn + (size_t)TT_STAGES * H_BYTES);     // [STAGES][CHUNK][NO]
    float* s_red = reinterpret_cast<float*>(dyn + (size_t)TT_STAGES * (H_BYTES + D_BYTES));   // [WARPS][PSTRIDE]
    __shared__ uint64_t bars[TT_STAGES];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
    const int n_chunks = (int)((row_end - row0 + TT_CHUNK - 1) / TT_CHUNK);
    auto issue = [&](int c) {   // thread 0
        const int st = c % TT_STAGES;
        const int64_t r = row0 + (int64_t)c * TT_CHUNK;
        const uint32_t rows = (uint32_t)min((int64_t)TT_CHUNK, row_end - r);
        mbar_expect_tx(&bars[st], rows * (H * 4 + NO * 4));
        tma_load_1d(s_h + (size_t)st * TT_CHUNK * H, hidden + r * H, rows * H * 4, &bars[st]);
        tma_load_1d(s_d + (size_t)st * TT_CHUNK * NO, dout + r * NO, rows * NO * 4, &bars[st]);
    };
    if (threadIdx.x == 0) {
        for (int st = 0; st < TT_STAGES; ++st) mbar_init(&bars[st], 1);
        mbar_fence_init();
        for (int c = 0; c < TT_STAGES && c < n_chunks; ++c) issue(c);
    }

    float4 w[NO];
#pragma unroll
    for (int k = 0; k < NO; ++k) w[k] = *reinterpret_cast<const float4*>(w_heads + (int64_t)k * H + 4 * lane);
    float4 acc_w[NO], acc_b = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc_o[NO];
#pragma unroll
    for (int k = 0; k < NO; ++k) { acc_o[k] = 0.f; acc_w[k] = make_float4(0.f, 0.f, 0.f, 0.f); }
    __syncthreads();   // barriers initialised before anyone waits on them

    for (int c = 0; c < n_chunks; ++c) {
        const int st = c % TT_STAGES;
        mbar_wait(&bars[st], (uint32_t)((c / TT_STAGES) & 1));
        const int64_t r0 = row0 + (int64_t)c * TT_CHUNK;
        const int rows = (int)min((int64_t)TT_CHUNK, row_end - r0);
        const float* ch = s_h + (size_t)st * TT_CHUNK * H;
        const float* cd = s_d + (size_t)st * TT_CHUNK * NO;
#pragma unroll
        for (int i = 0; i < TT_CHUNK / MT_WARPS; ++i) {
            const int rl = warp + i * MT_WARPS;
            if (rl < rows) {
                const float4 d0 = *reinterpret_cast<const float4*>(cd + rl * NO);
                const float4 d1 = *reinterpret_cast<const float4*>(cd + rl * NO + 4);
                const float d[NO] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
                const float4 h = *reinterpret_cast<const float4*>(ch + rl * H + 4 * lane);
                float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int k = 0; k < NO; ++k) {
                    acc_o[k] += d[k];
                    g.x = fmaf(d[k], w[k].x, g.x); g.y = fmaf(d[k], w[k].y, g.y);
                    g.z = fmaf(d[k], w[k].z, g.z); g.w = fmaf(d[k], w[k].w, g.w);
                    acc_w[k].x = fmaf(d[k], h.x, acc_w[k].x); acc_w[k].y = fmaf(d[k], h.y, acc_w[k].y);
                    acc_w[k].z = fmaf(d[k], h.z, acc_w[k].z); acc_w[k].w = fmaf(d[k], h.w, acc_w[k].w);
                }
                g.x = h.x > 0.f ? g.x : 0.f; g.y = h.y > 0.f ? g.y : 0.f;
                g.z = h.z > 0.f ? g.z : 0.f; g.w = h.w > 0.f ? g.w : 0.f;
                acc_b.x += g.x; acc_b.y += g.y; acc_b.z += g.z; acc_b.w += g.w;
                __stcs(reinterpret_cast<float4*>(dpre + (r0 + rl) * H + 4 * lane), g);
            }
        }
        __syncthreads();                                   // everyone is done reading stage st
        if (threadIdx.x == 0 && c + TT_STAGES < n_chunks) issue(c + TT_STAGES);
    }
    // ---- block reduction (same as the LDG variant)
    float* mine = s_red + (size_t)warp * PSTRIDE;
#pragma unroll
    for (int k = 0; k < NO; ++k) *reinterpret_cast<float4*>(mine + k * H + 4 * lane) = acc_w[k];
    *reinterpret_cast<float4*>(mine + NO * H + 4 * lane) = acc_b;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NO; ++k) mine[NO * H + H + k] = acc_o[k];
    __syncthreads();
    float* out = partials + (int64_t)blockIdx.x * PSTRIDE;
    for (int j = threadIdx.x; j < PSTRIDE; j += MT_THREADS) {
        float sum = 0.f;
#pragma unroll
        for (int wq = 0; wq < MT_WARPS; ++wq) sum += s_red[(size_t)wq * PSTRIDE + j];
        out[j] = sum;
    }
}

// deterministic second stage: out[j] = sum over blocks of partials[b][j].  One warp per output element: lane l sums
// blocks l, l+32, ... in order, then a fixed shuffle tree combines the 32 lane sums (same order every run).
__global__ void __launch_bounds__(256) k_reduce_partials(const float* __restrict__ partials, int n_blocks, int pstride,
                                                        float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= pstride) return;
    float s = 0.f;
    for (int b = lane; b < n_blocks; b += 32) s += partials[(int64_t)b * pstride + j];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) out[j] = s;
}

}  // namespace

extern "C" size_t pb_mlp_tail_workspace_bytes(int64_t m, int32_t hidden) {
    if (m <= 0 || hidden <= 0) return 16;
    const int64_t blocks = pb_ceil_div(m, ROWS_PER_BLOCK);
    return (size_t)blocks * (size_t)(NO * hidden + hidden + NO) * sizeof(float);
}

extern "C" int pb_mlp_tail_backward(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden,
                                    int64_t m, int32_t hidden_size, float* dpre, float* grads_out, void* workspace,
                                    size_t workspace_bytes, void* stream) {
    PB_REQUIRE(m >= 1, PB_ERR_INVALID, "pb_mlp_tail_backward: m must be positive");
    PB_REQUIRE(hidden_size == 128, PB_ERR_UNSUPPORTED, "pb_mlp_tail_backward: hidden size %d (only 128 is built)",
               hidden_size);
    PB_REQUIRE(dout && w_heads && hidden && dpre && grads_out && workspace, PB_ERR_INVALID,
               "pb_mlp_tail_backward: null pointer");
    PB_REQUIRE(dout_stride >= NO && dout_stride % 4 == 0 && ((uintptr_t)dout & 15) == 0 && ((uintptr_t)hidden & 15) == 0 &&
                   ((uintptr_t)dpre & 15) == 0 && ((uintptr_t)w_heads & 15) == 0,
               PB_ERR_INVALID, "pb_mlp_tail_backward: dout needs 8 padded columns; pointers must be 16-byte aligned");
    PB_REQUIRE(workspace_bytes >= pb_mlp_tail_workspace_bytes(m, hidden_size), PB_ERR_INVALID,
               "pb_mlp_tail_backward: workspace too small");
    const int blocks = (int)pb_ceil_div(m, ROWS_PER_BLOCK);
    const int pstride = NO * hidden_size + hidden_size + NO;
    cudaStream_t s = (cudaStream_t)stream;
    if (dout_stride == NO) {   // contiguous head gradients: TMA-staged pipeline
        const size_t smem = (size_t)TT_STAGES * (TT_CHUNK * 128 * 4 + TT_CHUNK * NO * 4) + (size_t)MT_WARPS * pstride * 4;
        PB_CUDA(cudaFuncSetAttribute(k_mlp_tail_bwd_tma<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_mlp_tail_bwd_tma<128><<<blocks, MT_THREADS, smem, s>>>(dout, w_heads, hidden, dpre, (float*)workspace, m);
    } else {
        k_mlp_tail_bwd<128><<<blocks, MT_THREADS, 0, s>>>(dout, dout_stride, w_heads, hidden, dpre, (float*)workspace, m);
    }
    PB_LAUNCH_CHECK();
    k_reduce_partials<<<(pstride * 32 + 255) / 256, 256, 0, s>>>((const float*)workspace, blocks, pstride, grads_out);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
