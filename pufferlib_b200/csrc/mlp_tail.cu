// mlp_tail.cu -- backward of the policy's "tail" (ReLU -> action/value heads) in one pass over the hidden layer (sm_90a).
//
// The configured policy is models.Default (reference pufferlib/models.py:12-62): Linear(obs->H)+ReLU, then two
// heads H->n_act and H->1.  In train (clean_pufferl.py:193-244) the backward of everything after the encoder GEMM is
// memory-bound work on [M, H] tensors that ATen runs as five launches, each re-reading 268 MB at M = 524288:
//   dHidden = dOut @ W_heads           (skinny GEMM, 8 columns)         dW_heads = dOut^T @ hidden   (skinny GEMM)
//   db_heads = sum_rows dOut           dPre = dHidden * (hidden > 0)    db_enc = sum_rows dPre
// This kernel does all five reading `hidden` ONCE and writing dPre once (2 * 4H + 4 NO B per row).  The dense H x H
// encoder GEMMs (forward, and dW_enc = dPre^T @ obs) stay on cuBLAS tensor cores.
// NO = the padded head rows: 8 for n_act <= 7, 16 for 8 <= n_act <= 15 (models.Default.head_matrix); both kernels are
// templates on it.  32 rows (16 <= n_act <= 31) take the half-width kernels further down (k_mlp_tail_bwd(_tma)_half).
// A warp owns rows; lane l owns columns 4l..4l+3 (one float4 per row per lane, 512 B coalesced for H = 128); the
// head weights live in registers (NO x 4 per lane); per-lane accumulators (dW: NO x 4, db_enc: 4) are reduced over
// the block's warps in shared memory and written as ONE partial row per block; a second tiny kernel sums the
// partials in a fixed order (deterministic, no atomics).
// Registers at NO = 16: the weights and the dW accumulators alone are 128 per thread, so the TMA kernel runs one
// 256-thread CTA per SM (its 4-stage ring still keeps 72 KB per SM in flight).  Moving W_heads to shared memory would
// add 16 LDS.128 per row and warp to the 5 the row needs, about the whole shared-memory bandwidth budget of a row at
// HBM speed, so the weights stay in registers.
#include "pb_common.cuh"
#include "tma.cuh"

namespace {

constexpr int MT_THREADS = 256;
constexpr int MT_WARPS = MT_THREADS / 32;
constexpr int ROWS_PER_BLOCK = 512;

// the row's NO head gradients from NO / 4 float4s (every lane of the warp reads the same bytes: a broadcast)
template <int NO>
__device__ __forceinline__ void tail_load_dout(const float* src, float (&d)[NO]) {
#pragma unroll
    for (int j = 0; j < NO / 4; ++j) {
        const float4 v = *reinterpret_cast<const float4*>(src + 4 * j);
        d[4 * j] = v.x; d[4 * j + 1] = v.y; d[4 * j + 2] = v.z; d[4 * j + 3] = v.w;
    }
}

// partial layout per block: [NO*H] dW_heads | [H] db_enc | [NO] db_heads
template <int H, int NO>
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd(const float* __restrict__ dout, int64_t dout_stride,
                                                            const float* __restrict__ w_heads,   // [NO][H]
                                                            const float* __restrict__ hidden,    // [M][H] post-ReLU
                                                            float* __restrict__ dpre,            // [M][H]
                                                            float* __restrict__ partials, int64_t m) {
    static_assert(H % 128 == 0, "H must be a multiple of 128 (one or more float4 per lane)");
    constexpr int Q = H / 128;                  // float4s per lane per row
    constexpr int PSTRIDE = NO * H + H + NO;
    // the block reduction goes through [WARPS][8 H + H + NO] floats (H = 128: 37 KB at NO = 8, 37.4 KB at NO = 16) in
    // NO / 8 passes of 8 dW_heads rows; the first pass also carries db_enc and db_heads.  NO = 8 is one pass over the
    // whole partial row.
    constexpr int RSTRIDE = 8 * H + H + NO;
    __shared__ float s_red[MT_WARPS][RSTRIDE];
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
        // the row's NO head gradients: every lane reads the same 4 NO bytes (broadcast)
        float d[NO];
        tail_load_dout<NO>(dout + r * dout_stride, d);
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
    float* out = partials + (int64_t)blockIdx.x * PSTRIDE;
    if constexpr (NO == 8) {   // the partial row fits: one pass, s_red row = partial row
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
        for (int j = threadIdx.x; j < PSTRIDE; j += MT_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int wq = 0; wq < MT_WARPS; ++wq) s += s_red[wq][j];
            out[j] = s;
        }
    } else {
        // pass p: dW_heads rows 8p..8p+7 at s_red[.][0, 8H); pass 0 also db_enc at [8H, 9H) and db_heads at [9H, 9H + NO)
#pragma unroll
        for (int pass = 0; pass < NO / 8; ++pass) {
            if (pass > 0) __syncthreads();   // the previous pass has been summed
#pragma unroll
            for (int k = 0; k < 8; ++k)
#pragma unroll
                for (int q = 0; q < Q; ++q)
                    *reinterpret_cast<float4*>(mine + k * H + 128 * q + 4 * lane) = acc_w[8 * pass + k][q];
            if (pass == 0) {
#pragma unroll
                for (int q = 0; q < Q; ++q) *reinterpret_cast<float4*>(mine + 8 * H + 128 * q + 4 * lane) = acc_b[q];
                if (lane == 0)
#pragma unroll
                    for (int k = 0; k < NO; ++k) mine[9 * H + k] = acc_o[k];
            }
            __syncthreads();
            const int n = pass == 0 ? RSTRIDE : 8 * H;
            for (int j = threadIdx.x; j < n; j += MT_THREADS) {
                float s = 0.f;
#pragma unroll
                for (int wq = 0; wq < MT_WARPS; ++wq) s += s_red[wq][j];
                // s_red column j -> partial column: dW rows of this pass, then (pass 0) db_enc | db_heads after all NO rows
                out[j < 8 * H ? 8 * pass * H + j : (NO - 8) * H + j] = s;
            }
        }
    }
}

// TMA-staged variant (dout contiguous [M][NO]): the hidden rows and their head gradients are pulled into a 4-stage
// shared-memory ring by cp.async.bulk (one elected thread, mbarrier complete_tx), 32 rows = 16 KiB + NO / 8 KiB per
// stage, so ~64 KiB per CTA is in flight independently of the register budget; the warps consume from shared memory
// (conflict-free LDS.128) and stream dPre straight back to HBM.  Dynamic shared memory: the ring plus the [WARPS][PSTRIDE]
// reduction buffer, 105 KB at NO = 8 (2 CTAs per SM), 140.5 KB at NO = 16.
constexpr int TT_STAGES = 4;
constexpr int TT_CHUNK = 32;   // rows per stage

template <int H, int NO>
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
                float d[NO];
                tail_load_dout<NO>(cd + rl * NO, d);
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

// ---- H = 256, 384, 512: the same per-row plan over 128-column slices of the hidden layer, slice s = blockIdx.y.
// Every output but db_heads is per hidden column, so a CTA of slice s reads columns [128s, 128s + 128) of its rows
// (row stride H), reads each row's dOut once, and writes its columns of the block's [NO*H | H | NO] partial row; slice 0
// also writes db_heads.  A slice's accumulators are those of the H = 128 kernels, so the registers, the reduction
// buffer and the dynamic shared memory are theirs too.  The H = 128 kernels above are kept as they are.

// index in the [NO*H | H | NO] partial row of entry j of a slice's [NO*128 | 128 | NO] accumulators
template <int NO>
__device__ __forceinline__ int64_t slice_partial_index(int j, int h, int col0) {
    if (j < NO * 128) return (int64_t)(j >> 7) * h + col0 + (j & 127);
    if (j < NO * 128 + 128) return (int64_t)NO * h + col0 + (j - NO * 128);
    return (int64_t)NO * h + h + (j - NO * 128 - 128);
}

template <int NO>
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd_slices(const float* __restrict__ dout, int64_t dout_stride,
                                                                   const float* __restrict__ w_heads,   // [NO][h]
                                                                   const float* __restrict__ hidden,    // [M][h]
                                                                   float* __restrict__ dpre,            // [M][h]
                                                                   float* __restrict__ partials, int64_t m, int h) {
    constexpr int RSTRIDE = 8 * 128 + 128 + NO;   // NO / 8 passes of 8 dW rows, as k_mlp_tail_bwd<128, NO>
    __shared__ float s_red[MT_WARPS][RSTRIDE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col0 = 128 * (int)blockIdx.y;
    const float* hcol = hidden + col0 + 4 * lane;
    float* dcol = dpre + col0 + 4 * lane;

    float4 w[NO], acc_w[NO], acc_b = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc_o[NO];
#pragma unroll
    for (int k = 0; k < NO; ++k) {
        w[k] = *reinterpret_cast<const float4*>(w_heads + (int64_t)k * h + col0 + 4 * lane);
        acc_w[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        acc_o[k] = 0.f;
    }
    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
#pragma unroll 2
    for (int64_t r = row0 + warp; r < row_end; r += MT_WARPS) {
        float d[NO];
        tail_load_dout<NO>(dout + r * dout_stride, d);
        const float4 hv = __ldcs(reinterpret_cast<const float4*>(hcol + r * h));
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < NO; ++k) {
            acc_o[k] += d[k];
            g.x = fmaf(d[k], w[k].x, g.x); g.y = fmaf(d[k], w[k].y, g.y);
            g.z = fmaf(d[k], w[k].z, g.z); g.w = fmaf(d[k], w[k].w, g.w);
            acc_w[k].x = fmaf(d[k], hv.x, acc_w[k].x); acc_w[k].y = fmaf(d[k], hv.y, acc_w[k].y);
            acc_w[k].z = fmaf(d[k], hv.z, acc_w[k].z); acc_w[k].w = fmaf(d[k], hv.w, acc_w[k].w);
        }
        g.x = hv.x > 0.f ? g.x : 0.f; g.y = hv.y > 0.f ? g.y : 0.f;
        g.z = hv.z > 0.f ? g.z : 0.f; g.w = hv.w > 0.f ? g.w : 0.f;
        acc_b.x += g.x; acc_b.y += g.y; acc_b.z += g.z; acc_b.w += g.w;
        __stcs(reinterpret_cast<float4*>(dcol + r * h), g);
    }
    // pass p: dW rows 8p..8p+7 at s_red[.][0, 1024); pass 0 also db_enc at [1024, 1152) and db_heads at [1152, 1152 + NO)
    float* mine = s_red[warp];
    float* out = partials + (int64_t)blockIdx.x * (NO * h + h + NO);
#pragma unroll
    for (int pass = 0; pass < NO / 8; ++pass) {
        if (pass > 0) __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; ++k) *reinterpret_cast<float4*>(mine + k * 128 + 4 * lane) = acc_w[8 * pass + k];
        if (pass == 0) {
            *reinterpret_cast<float4*>(mine + 8 * 128 + 4 * lane) = acc_b;
            if (lane == 0)
#pragma unroll
                for (int k = 0; k < NO; ++k) mine[9 * 128 + k] = acc_o[k];
        }
        __syncthreads();
        const int n = pass == 0 ? (blockIdx.y == 0 ? RSTRIDE : 9 * 128) : 8 * 128;
        for (int j = threadIdx.x; j < n; j += MT_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int wq = 0; wq < MT_WARPS; ++wq) s += s_red[wq][j];
            out[slice_partial_index<NO>(j < 8 * 128 ? 8 * 128 * pass + j : (NO - 8) * 128 + j, h, col0)] = s;
        }
    }
}

// TMA-staged slices (dout contiguous [M][NO]): the ring of k_mlp_tail_bwd_tma, filled with one 512-byte bulk copy per
// row (the slice's columns of the row; lane l of warp 0 copies row l of the chunk) plus the chunk's dOut rows.
template <int NO>
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd_tma_slices(const float* __restrict__ dout,      // [M][NO]
                                                                       const float* __restrict__ w_heads,   // [NO][h]
                                                                       const float* __restrict__ hidden,    // [M][h]
                                                                       float* __restrict__ dpre,            // [M][h]
                                                                       float* __restrict__ partials, int64_t m, int h) {
    constexpr int PS = NO * 128 + 128 + NO;   // a slice's accumulators
    constexpr uint32_t H_BYTES = TT_CHUNK * 128 * 4, D_BYTES = TT_CHUNK * NO * 4;
    extern __shared__ __align__(128) unsigned char dyn[];
    float* s_h = reinterpret_cast<float*>(dyn);                                   // [STAGES][CHUNK][128]
    float* s_d = reinterpret_cast<float*>(dyn + (size_t)TT_STAGES * H_BYTES);     // [STAGES][CHUNK][NO]
    float* s_red = reinterpret_cast<float*>(dyn + (size_t)TT_STAGES * (H_BYTES + D_BYTES));   // [WARPS][PS]
    __shared__ uint64_t bars[TT_STAGES];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col0 = 128 * (int)blockIdx.y;

    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
    const int n_chunks = (int)((row_end - row0 + TT_CHUNK - 1) / TT_CHUNK);
    auto issue = [&](int c) {   // warp 0; lane 0 arrives with the byte count before any lane copies
        const int st = c % TT_STAGES;
        const int64_t r = row0 + (int64_t)c * TT_CHUNK;
        const uint32_t rows = (uint32_t)min((int64_t)TT_CHUNK, row_end - r);
        if (lane == 0) {
            mbar_expect_tx(&bars[st], rows * (128 * 4 + NO * 4));
            tma_load_1d(s_d + (size_t)st * TT_CHUNK * NO, dout + r * NO, rows * NO * 4, &bars[st]);
        }
        __syncwarp();
        if ((uint32_t)lane < rows)
            tma_load_1d(s_h + ((size_t)st * TT_CHUNK + lane) * 128, hidden + (r + lane) * h + col0, 128 * 4, &bars[st]);
    };
    if (threadIdx.x == 0) {
        for (int st = 0; st < TT_STAGES; ++st) mbar_init(&bars[st], 1);
        mbar_fence_init();
    }
    __syncthreads();   // barriers initialised before warp 0 copies and anyone waits on them
    if (warp == 0)
        for (int c = 0; c < TT_STAGES && c < n_chunks; ++c) issue(c);

    float4 w[NO], acc_w[NO], acc_b = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc_o[NO];
#pragma unroll
    for (int k = 0; k < NO; ++k) {
        w[k] = *reinterpret_cast<const float4*>(w_heads + (int64_t)k * h + col0 + 4 * lane);
        acc_o[k] = 0.f;
        acc_w[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float* dcol = dpre + col0 + 4 * lane;

    for (int c = 0; c < n_chunks; ++c) {
        const int st = c % TT_STAGES;
        mbar_wait(&bars[st], (uint32_t)((c / TT_STAGES) & 1));
        const int64_t r0 = row0 + (int64_t)c * TT_CHUNK;
        const int rows = (int)min((int64_t)TT_CHUNK, row_end - r0);
        const float* ch = s_h + (size_t)st * TT_CHUNK * 128;
        const float* cd = s_d + (size_t)st * TT_CHUNK * NO;
#pragma unroll
        for (int i = 0; i < TT_CHUNK / MT_WARPS; ++i) {
            const int rl = warp + i * MT_WARPS;
            if (rl < rows) {
                float d[NO];
                tail_load_dout<NO>(cd + rl * NO, d);
                const float4 hv = *reinterpret_cast<const float4*>(ch + rl * 128 + 4 * lane);
                float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int k = 0; k < NO; ++k) {
                    acc_o[k] += d[k];
                    g.x = fmaf(d[k], w[k].x, g.x); g.y = fmaf(d[k], w[k].y, g.y);
                    g.z = fmaf(d[k], w[k].z, g.z); g.w = fmaf(d[k], w[k].w, g.w);
                    acc_w[k].x = fmaf(d[k], hv.x, acc_w[k].x); acc_w[k].y = fmaf(d[k], hv.y, acc_w[k].y);
                    acc_w[k].z = fmaf(d[k], hv.z, acc_w[k].z); acc_w[k].w = fmaf(d[k], hv.w, acc_w[k].w);
                }
                g.x = hv.x > 0.f ? g.x : 0.f; g.y = hv.y > 0.f ? g.y : 0.f;
                g.z = hv.z > 0.f ? g.z : 0.f; g.w = hv.w > 0.f ? g.w : 0.f;
                acc_b.x += g.x; acc_b.y += g.y; acc_b.z += g.z; acc_b.w += g.w;
                __stcs(reinterpret_cast<float4*>(dcol + (r0 + rl) * h), g);
            }
        }
        __syncthreads();                                   // everyone is done reading stage st
        if (warp == 0 && c + TT_STAGES < n_chunks) issue(c + TT_STAGES);
    }
    float* mine = s_red + (size_t)warp * PS;
#pragma unroll
    for (int k = 0; k < NO; ++k) *reinterpret_cast<float4*>(mine + k * 128 + 4 * lane) = acc_w[k];
    *reinterpret_cast<float4*>(mine + NO * 128 + 4 * lane) = acc_b;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NO; ++k) mine[NO * 128 + 128 + k] = acc_o[k];
    __syncthreads();
    float* out = partials + (int64_t)blockIdx.x * (NO * h + h + NO);
    const int n = blockIdx.y == 0 ? PS : NO * 128 + 128;
    for (int j = threadIdx.x; j < n; j += MT_THREADS) {
        float sum = 0.f;
#pragma unroll
        for (int wq = 0; wq < MT_WARPS; ++wq) sum += s_red[(size_t)wq * PS + j];
        out[slice_partial_index<NO>(j, h, col0)] = sum;
    }
}

// ---- 32 head rows (16 <= n_act <= 31), any H = 128 k.  With one float4 per lane the head weights and dW accumulators
// alone would take 256 registers per lane, so here a lane owns ONE float2 of a row: a warp covers 64 columns and the grid
// runs over 64-column slices of the hidden layer, slice s = blockIdx.y (H / 64 of them, 2 at H = 128).  w and acc_w are
// then 64 registers each.  `hidden` is still read once and dPre written once; every slice re-reads the row's 128-byte
// dOut (+12 % bytes at H = 128).  db_heads: lane l sums column l of dOut (one 4-byte load per row and lane) instead of
// holding 32 sums; slice 0 writes it.  The partial row, k_reduce_partials and the workspace are those of the kernels above.
constexpr int HS_W = 64;                           // columns per slice
constexpr int HS_NO = 32;                          // head rows
constexpr int HS_RSTRIDE = 8 * HS_W + HS_W + HS_NO;   // reduction row: 8 dW rows | db_enc | db_heads (4 passes)

// one row of a slice: dPre's two columns of the lane (returned), and the lane's accumulators
__device__ __forceinline__ float2 half_slice_row(const float (&d)[HS_NO], float2 hv, const float2 (&w)[HS_NO],
                                                 float2 (&acc_w)[HS_NO], float2& acc_b) {
    float2 g = make_float2(0.f, 0.f);
#pragma unroll
    for (int k = 0; k < HS_NO; ++k) {
        g.x = fmaf(d[k], w[k].x, g.x); g.y = fmaf(d[k], w[k].y, g.y);
        acc_w[k].x = fmaf(d[k], hv.x, acc_w[k].x); acc_w[k].y = fmaf(d[k], hv.y, acc_w[k].y);
    }
    g.x = hv.x > 0.f ? g.x : 0.f; g.y = hv.y > 0.f ? g.y : 0.f;
    acc_b.x += g.x; acc_b.y += g.y;
    return g;
}

// the block's sum of every warp's accumulators into its [32 H | H | 32] partial row, in 4 passes of 8 dW rows through
// s_red [WARPS][HS_RSTRIDE]; pass 0 also carries db_enc and (slice 0) db_heads
__device__ __forceinline__ void half_slice_reduce(const float2 (&acc_w)[HS_NO], float2 acc_b, float acc_o,
                                                  float (*s_red)[HS_RSTRIDE], float* out, int h, int col0) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* mine = s_red[warp];
#pragma unroll
    for (int pass = 0; pass < HS_NO / 8; ++pass) {
        if (pass > 0) __syncthreads();   // the previous pass has been summed
#pragma unroll
        for (int k = 0; k < 8; ++k) *reinterpret_cast<float2*>(mine + k * HS_W + 2 * lane) = acc_w[8 * pass + k];
        if (pass == 0) {
            *reinterpret_cast<float2*>(mine + 8 * HS_W + 2 * lane) = acc_b;
            mine[9 * HS_W + lane] = acc_o;
        }
        __syncthreads();
        const int n = pass == 0 ? (col0 == 0 ? HS_RSTRIDE : 9 * HS_W) : 8 * HS_W;
        for (int j = threadIdx.x; j < n; j += MT_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int wq = 0; wq < MT_WARPS; ++wq) s += s_red[wq][j];
            int64_t idx;
            if (j < 8 * HS_W) idx = (int64_t)(8 * pass + j / HS_W) * h + col0 + j % HS_W;     // dW_heads
            else if (j < 9 * HS_W) idx = (int64_t)HS_NO * h + col0 + (j - 8 * HS_W);          // db_enc
            else idx = (int64_t)HS_NO * h + h + (j - 9 * HS_W);                               // db_heads
            out[idx] = s;
        }
    }
}

__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd_half(const float* __restrict__ dout, int64_t dout_stride,
                                                                 const float* __restrict__ w_heads,   // [32][h]
                                                                 const float* __restrict__ hidden,    // [M][h]
                                                                 float* __restrict__ dpre,            // [M][h]
                                                                 float* __restrict__ partials, int64_t m, int h) {
    __shared__ float s_red[MT_WARPS][HS_RSTRIDE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col0 = HS_W * (int)blockIdx.y;
    const float* hcol = hidden + col0 + 2 * lane;
    float* dcol = dpre + col0 + 2 * lane;

    float2 w[HS_NO], acc_w[HS_NO], acc_b = make_float2(0.f, 0.f);
    float acc_o = 0.f;
#pragma unroll
    for (int k = 0; k < HS_NO; ++k) {
        w[k] = *reinterpret_cast<const float2*>(w_heads + (int64_t)k * h + col0 + 2 * lane);
        acc_w[k] = make_float2(0.f, 0.f);
    }
    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
    for (int64_t r = row0 + warp; r < row_end; r += MT_WARPS) {
        const float* drow = dout + r * dout_stride;
        float d[HS_NO];
        tail_load_dout<HS_NO>(drow, d);
        acc_o += drow[lane];
        const float2 hv = __ldcs(reinterpret_cast<const float2*>(hcol + r * h));
        __stcs(reinterpret_cast<float2*>(dcol + r * h), half_slice_row(d, hv, w, acc_w, acc_b));
    }
    half_slice_reduce(acc_w, acc_b, acc_o, s_red, partials + (int64_t)blockIdx.x * (HS_NO * h + h + HS_NO), h, col0);
}

// TMA-staged (dout contiguous [M][32]): the 4-stage ring of k_mlp_tail_bwd_tma_slices, 32 rows per stage, filled with one
// 256-byte bulk copy per row (the slice's columns; lane l of warp 0 copies row l of the chunk) plus the chunk's dOut
// rows: 12 KB per stage, 48 KB of dynamic shared memory.
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd_tma_half(const float* __restrict__ dout,      // [M][32]
                                                                     const float* __restrict__ w_heads,   // [32][h]
                                                                     const float* __restrict__ hidden,    // [M][h]
                                                                     float* __restrict__ dpre,            // [M][h]
                                                                     float* __restrict__ partials, int64_t m, int h) {
    constexpr uint32_t H_BYTES = TT_CHUNK * HS_W * 4;
    extern __shared__ __align__(128) unsigned char dyn[];
    float* s_h = reinterpret_cast<float*>(dyn);                                   // [STAGES][CHUNK][64]
    float* s_d = reinterpret_cast<float*>(dyn + (size_t)TT_STAGES * H_BYTES);     // [STAGES][CHUNK][32]
    __shared__ float s_red[MT_WARPS][HS_RSTRIDE];
    __shared__ uint64_t bars[TT_STAGES];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col0 = HS_W * (int)blockIdx.y;

    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
    const int n_chunks = (int)((row_end - row0 + TT_CHUNK - 1) / TT_CHUNK);
    auto issue = [&](int c) {   // warp 0; lane 0 arrives with the byte count before any lane copies
        const int st = c % TT_STAGES;
        const int64_t r = row0 + (int64_t)c * TT_CHUNK;
        const uint32_t rows = (uint32_t)min((int64_t)TT_CHUNK, row_end - r);
        if (lane == 0) {
            mbar_expect_tx(&bars[st], rows * (HS_W * 4 + HS_NO * 4));
            tma_load_1d(s_d + (size_t)st * TT_CHUNK * HS_NO, dout + r * HS_NO, rows * HS_NO * 4, &bars[st]);
        }
        __syncwarp();
        if ((uint32_t)lane < rows)
            tma_load_1d(s_h + ((size_t)st * TT_CHUNK + lane) * HS_W, hidden + (r + lane) * h + col0, HS_W * 4, &bars[st]);
    };
    if (threadIdx.x == 0) {
        for (int st = 0; st < TT_STAGES; ++st) mbar_init(&bars[st], 1);
        mbar_fence_init();
    }
    __syncthreads();   // barriers initialised before warp 0 copies and anyone waits on them
    if (warp == 0)
        for (int c = 0; c < TT_STAGES && c < n_chunks; ++c) issue(c);

    float2 w[HS_NO], acc_w[HS_NO], acc_b = make_float2(0.f, 0.f);
    float acc_o = 0.f;
#pragma unroll
    for (int k = 0; k < HS_NO; ++k) {
        w[k] = *reinterpret_cast<const float2*>(w_heads + (int64_t)k * h + col0 + 2 * lane);
        acc_w[k] = make_float2(0.f, 0.f);
    }
    float* dcol = dpre + col0 + 2 * lane;

    for (int c = 0; c < n_chunks; ++c) {
        const int st = c % TT_STAGES;
        mbar_wait(&bars[st], (uint32_t)((c / TT_STAGES) & 1));
        const int64_t r0 = row0 + (int64_t)c * TT_CHUNK;
        const int rows = (int)min((int64_t)TT_CHUNK, row_end - r0);
        const float* ch = s_h + (size_t)st * TT_CHUNK * HS_W;
        const float* cd = s_d + (size_t)st * TT_CHUNK * HS_NO;
#pragma unroll
        for (int i = 0; i < TT_CHUNK / MT_WARPS; ++i) {
            const int rl = warp + i * MT_WARPS;
            if (rl < rows) {
                float d[HS_NO];
                tail_load_dout<HS_NO>(cd + rl * HS_NO, d);
                acc_o += cd[rl * HS_NO + lane];
                const float2 hv = *reinterpret_cast<const float2*>(ch + rl * HS_W + 2 * lane);
                __stcs(reinterpret_cast<float2*>(dcol + (r0 + rl) * h), half_slice_row(d, hv, w, acc_w, acc_b));
            }
        }
        __syncthreads();                                   // everyone is done reading stage st
        if (warp == 0 && c + TT_STAGES < n_chunks) issue(c + TT_STAGES);
    }
    half_slice_reduce(acc_w, acc_b, acc_o, s_red, partials + (int64_t)blockIdx.x * (HS_NO * h + h + HS_NO), h, col0);
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

template <int NO>
int launch_tail(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden, int64_t m, float* dpre,
                float* workspace, int blocks, cudaStream_t s) {
    const int pstride = NO * 128 + 128 + NO;
    if (dout_stride == NO) {   // contiguous head gradients: TMA-staged pipeline
        const size_t smem = (size_t)TT_STAGES * (TT_CHUNK * 128 * 4 + TT_CHUNK * NO * 4) + (size_t)MT_WARPS * pstride * 4;
        PB_CUDA(cudaFuncSetAttribute(k_mlp_tail_bwd_tma<128, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_mlp_tail_bwd_tma<128, NO><<<blocks, MT_THREADS, smem, s>>>(dout, w_heads, hidden, dpre, workspace, m);
    } else {
        k_mlp_tail_bwd<128, NO><<<blocks, MT_THREADS, 0, s>>>(dout, dout_stride, w_heads, hidden, dpre, workspace, m);
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

template <int NO>
int launch_tail_slices(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden, int64_t m, int h,
                       float* dpre, float* workspace, int blocks, cudaStream_t s) {
    const dim3 grid((unsigned)blocks, (unsigned)(h / 128));
    if (dout_stride == NO) {
        const size_t smem = (size_t)TT_STAGES * (TT_CHUNK * 128 * 4 + TT_CHUNK * NO * 4) + (size_t)MT_WARPS * (NO * 128 + 128 + NO) * 4;
        PB_CUDA(cudaFuncSetAttribute(k_mlp_tail_bwd_tma_slices<NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_mlp_tail_bwd_tma_slices<NO><<<grid, MT_THREADS, smem, s>>>(dout, w_heads, hidden, dpre, workspace, m, h);
    } else {
        k_mlp_tail_bwd_slices<NO><<<grid, MT_THREADS, 0, s>>>(dout, dout_stride, w_heads, hidden, dpre, workspace, m, h);
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int launch_tail_half(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden, int64_t m, int h,
                     float* dpre, float* workspace, int blocks, cudaStream_t s) {
    const dim3 grid((unsigned)blocks, (unsigned)(h / HS_W));
    if (dout_stride == HS_NO) {
        const size_t smem = (size_t)TT_STAGES * TT_CHUNK * (HS_W + HS_NO) * 4;
        PB_CUDA(cudaFuncSetAttribute(k_mlp_tail_bwd_tma_half, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_mlp_tail_bwd_tma_half<<<grid, MT_THREADS, smem, s>>>(dout, w_heads, hidden, dpre, workspace, m, h);
    } else {
        k_mlp_tail_bwd_half<<<grid, MT_THREADS, 0, s>>>(dout, dout_stride, w_heads, hidden, dpre, workspace, m, h);
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

}  // namespace

extern "C" size_t pb_mlp_tail_workspace_bytes_ex(int64_t m, int32_t hidden, int32_t head_rows) {
    if (m <= 0 || hidden <= 0 || (head_rows != 8 && head_rows != 16 && head_rows != 32)) return 16;
    const int64_t blocks = pb_ceil_div(m, ROWS_PER_BLOCK);
    return (size_t)blocks * (size_t)(head_rows * hidden + hidden + head_rows) * sizeof(float);
}

extern "C" size_t pb_mlp_tail_workspace_bytes(int64_t m, int32_t hidden) {
    return pb_mlp_tail_workspace_bytes_ex(m, hidden, 8);
}

extern "C" int pb_mlp_tail_backward_ex(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden,
                                       int64_t m, int32_t hidden_size, float* dpre, float* grads_out, void* workspace,
                                       size_t workspace_bytes, int32_t head_rows, void* stream) {
    PB_REQUIRE(m >= 1, PB_ERR_INVALID, "pb_mlp_tail_backward: m must be positive");
    PB_REQUIRE(hidden_size >= 128 && hidden_size <= 512 && hidden_size % 128 == 0, PB_ERR_UNSUPPORTED,
               "pb_mlp_tail_backward: hidden size %d (128, 256, 384 and 512 are built)", hidden_size);
    PB_REQUIRE(head_rows == 8 || head_rows == 16 || head_rows == 32, PB_ERR_UNSUPPORTED,
               "pb_mlp_tail_backward: head_rows %d (8, 16 and 32 are built)", head_rows);
    PB_REQUIRE(dout && w_heads && hidden && dpre && grads_out && workspace, PB_ERR_INVALID,
               "pb_mlp_tail_backward: null pointer");
    PB_REQUIRE(dout_stride >= head_rows && dout_stride % 4 == 0 && ((uintptr_t)dout & 15) == 0 &&
                   ((uintptr_t)hidden & 15) == 0 && ((uintptr_t)dpre & 15) == 0 && ((uintptr_t)w_heads & 15) == 0,
               PB_ERR_INVALID, "pb_mlp_tail_backward: dout needs %d padded columns; pointers must be 16-byte aligned",
               head_rows);
    PB_REQUIRE(workspace_bytes >= pb_mlp_tail_workspace_bytes_ex(m, hidden_size, head_rows), PB_ERR_INVALID,
               "pb_mlp_tail_backward: workspace too small");
    const int blocks = (int)pb_ceil_div(m, ROWS_PER_BLOCK);
    const int pstride = head_rows * hidden_size + hidden_size + head_rows;
    cudaStream_t s = (cudaStream_t)stream;
    float* ws = (float*)workspace;
    const int rc =
        head_rows == HS_NO ? launch_tail_half(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, ws, blocks, s)
        : hidden_size == 128
            ? (head_rows == 8 ? launch_tail<8>(dout, dout_stride, w_heads, hidden, m, dpre, ws, blocks, s)
                              : launch_tail<16>(dout, dout_stride, w_heads, hidden, m, dpre, ws, blocks, s))
            : (head_rows == 8 ? launch_tail_slices<8>(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, ws, blocks, s)
                              : launch_tail_slices<16>(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, ws, blocks, s));
    if (rc != PB_OK) return rc;
    k_reduce_partials<<<(pstride * 32 + 255) / 256, 256, 0, s>>>((const float*)workspace, blocks, pstride, grads_out);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_mlp_tail_backward(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden,
                                    int64_t m, int32_t hidden_size, float* dpre, float* grads_out, void* workspace,
                                    size_t workspace_bytes, void* stream) {
    return pb_mlp_tail_backward_ex(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, grads_out, workspace,
                                   workspace_bytes, 8, stream);
}
