// policy_mlp.cu -- the rollout-time forward of models.Default fused with the sampling epilogue, ONE launch per env step.
//
// Replaces, inside the evaluate loop (reference clean_pufferl.py:107-117), the chain
//   encoder Linear + ReLU -> action head + value head (pufferlib/models.py:12-62) -> sample_logits
//   (pufferlib/frameworks/cleanrl.py:25-47) -> Experience.store of value / logprob / action (clean_pufferl.py:443-446)
// which the library path runs as 2 GEMM launches + sampler + counter update.  At rollout time M = num_envs rows (16384),
// so the GEMMs are tiny (0.5 GFLOP) and launch/latency bound; here a CTA owns 64 rows:
//   * the 64x128 fp32 observation tile and the 128x128 encoder weights land in shared memory as 512-byte bulk copies
//     (cp.async.bulk, one per row, two mbarriers);
//   * hidden = relu(X W^T + b) on the tensor cores (mma.sync m16n8k8 TF32, fp32 accumulate; a warp owns 16 rows x 128
//     columns, accumulators stay in registers -- `hidden` is never written to memory);
//   * the two heads (n_act logits + value, padded to NC = 8 columns for n_act <= 7, 16 for n_act <= 15, 32 for
//     n_act <= 31) are a second mma whose A operand is the accumulator fragment itself (the k order of the second product
//     is permuted to match the C-fragment layout); NC = 16 and 32 are two and four n8 blocks on the same A fragments;
//   * a quad shuffle gathers each row's NC outputs, one lane per row does logsumexp / inverse-CDF sampling / logprob /
//     entropy and writes action, logprob, value straight into the rollout rows.
// Tensor-core path note: this is a 128x128x128 tile per CTA, far below the size where a wgmma pipeline pays; the large
// training GEMMs of the generic path stay on cuBLAS.
#include "pb_common.cuh"
#include "policy_sample.cuh"
#include "tma.cuh"

namespace {

constexpr int PM_K = 128;           // obs features
constexpr int PM_H = 128;           // hidden units
constexpr int PM_PITCH = PM_K + 8;  // shared row pitch in floats (544 B): conflict-free 64-bit fragment loads

struct PolicyParams {
    const float* obs; int64_t obs_stride;      // [M][128] fp32
    const float* w_enc; const float* b_enc;    // [128][128], [128]
    const float* w_heads; const float* b_heads;  // [NC][128], [NC]  (n_act logits | value | zero pad)
    int64_t m; int n_act;
    uint64_t seed; uint64_t* counter; unsigned int* ticket;
    int64_t* actions; float* logprobs; float* values; float* entropies;   // [M] each (entropies may be null)
};

// 64 rows per CTA, one warp per 16 rows: 128 threads, 104 KB shared (+ 4 KB more head rows at NC = 16) -> 2 CTAs per
// SM, 256 CTAs at 16384 rows.  NC = 32: a static [32][128] head copy (16 KB) would leave room for one CTA per SM only, so
// the head rows are read into registers (8 float4 per thread) before the hidden product and written over sW once every
// warp is done with W_enc: the shared memory, and the two CTAs per SM, stay those of NC = 16.
constexpr int PM_ROWS = 64;
constexpr int PM_THREADS = 2 * PM_ROWS;

template <int NC>
__global__ void __launch_bounds__(PM_THREADS) k_policy_mlp_sample(PolicyParams p) {
    constexpr bool HEADS_IN_SW = NC > 16;
    extern __shared__ __align__(128) float smem[];
    float* sX = smem;                              // [64][136]
    float* sW = smem + PM_ROWS * PM_PITCH;         // [128][136]  (row = hidden unit, col = input feature)
    __shared__ float sWh[HEADS_IN_SW ? 1 : NC][PM_H];
    __shared__ float sBe[PM_H];
    __shared__ float sBh[NC];
    __shared__ __align__(8) uint64_t bars[2];      // [0]: obs tile + W rows 0..63, [1]: W rows 64..127
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int64_t row0 = (int64_t)blockIdx.x * PM_ROWS;
    const int valid = (int)((p.m - row0) < PM_ROWS ? (p.m - row0) : PM_ROWS);
    const uint64_t offset = p.counter ? *p.counter : 0ull;   // every CTA reads it before taking its exit ticket

    // ---- stage the observation tile and the weights: one 512-byte bulk copy (TMA engine) per row, completion counted
    //      on two mbarriers so the first 8 n-tiles start while the second half of W is still in flight
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_fence_init();
        mbar_expect_tx(&bars[0], (uint32_t)(valid + 64) * PM_K * 4u);
        mbar_expect_tx(&bars[1], 64u * PM_K * 4u);
    }
    if (tid >= valid && tid < PM_ROWS) {           // rows past M: zeros
#pragma unroll 8
        for (int q = 0; q < PM_K / 4; ++q) *reinterpret_cast<float4*>(sX + tid * PM_PITCH + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float4 wh[HEADS_IN_SW ? NC * PM_H / 4 / PM_THREADS : 1];   // NC = 32: float4 i = tid + 128 j of w_heads
    if constexpr (HEADS_IN_SW) {
#pragma unroll
        for (int j = 0; j < NC * PM_H / 4 / PM_THREADS; ++j)
            wh[j] = *reinterpret_cast<const float4*>(p.w_heads + 4 * (tid + PM_THREADS * j));
    } else {
        for (int i = tid; i < NC * PM_H; i += PM_THREADS) sWh[i >> 7][i & 127] = p.w_heads[i];
    }
    if (tid < PM_H) sBe[tid] = p.b_enc[tid];
    if (tid < NC) sBh[tid] = p.b_heads[tid];
    __syncthreads();
    if (tid < valid) tma_load_1d(sX + tid * PM_PITCH, p.obs + (row0 + tid) * p.obs_stride, PM_K * 4u, &bars[0]);
    tma_load_1d(sW + tid * PM_PITCH, p.w_enc + (int64_t)tid * PM_K, PM_K * 4u, &bars[tid >> 6]);

    // ---- hidden tile: warp w owns rows 16w..16w+15, all 128 columns (16 n-tiles), K = 128 (16 k-steps).
    //      The sum over k is order-free, so k slots (t, t+4) of a k-step are mapped to the ADJACENT columns
    //      (8ks + 2t, 8ks + 2t + 1) for both operands: every fragment is one 64-bit shared load (pitch 136: conflict-free).
    //      A is rounded to TF32 here; W arrives pre-rounded (or is truncated by the tensor core, see the header).
    float acc[16][4];
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
    const float* xa = sX + (16 * warp + g) * PM_PITCH + 2 * t;
    const float* wbase = sW + g * PM_PITCH + 2 * t;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        mbar_wait(&bars[half], 0);
#pragma unroll 4
        for (int ks = 0; ks < 16; ++ks) {
            const float2 x0 = *reinterpret_cast<const float2*>(xa + 8 * ks);
            const float2 x1 = *reinterpret_cast<const float2*>(xa + 8 * PM_PITCH + 8 * ks);
            const uint32_t a[4] = {to_tf32(x0.x), to_tf32(x1.x), to_tf32(x0.y), to_tf32(x1.y)};
#pragma unroll
            for (int n8 = 0; n8 < 8; ++n8) {
                const int nt = 8 * half + n8;
                const float2 w = *reinterpret_cast<const float2*>(wbase + 8 * nt * PM_PITCH + 8 * ks);   // B[k][n] = W[n][k]
                mma_tf32(acc[nt], a, __float_as_uint(w.x), __float_as_uint(w.y));
            }
        }
    }
    if constexpr (HEADS_IN_SW) {   // every warp is done with W_enc: head row r -> sW row r (same 136-float pitch)
        __syncthreads();
#pragma unroll
        for (int j = 0; j < NC * PM_H / 4 / PM_THREADS; ++j) {
            const int i = tid + PM_THREADS * j;
            *reinterpret_cast<float4*>(sW + (i >> 5) * PM_PITCH + 4 * (i & 31)) = wh[j];
        }
        __syncthreads();
    }
    // ---- bias + ReLU on the accumulators; heads = hidden @ Wh^T as a second mma with A = the C fragments:
    //      C fragment of n-tile nt holds columns 8nt + {2t, 2t+1} of rows {g, g+8}; use them as k slots {t, t+4};
    //      head block q8 (columns 8q8..8q8+7) takes B from head rows 8q8 + g
    float out[NC / 8][4];
#pragma unroll
    for (int q8 = 0; q8 < NC / 8; ++q8) { out[q8][0] = out[q8][1] = out[q8][2] = out[q8][3] = 0.f; }
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
        const int c0 = 8 * nt + 2 * t;
        const float b0 = sBe[c0], b1 = sBe[c0 + 1];
        uint32_t a[4];
        a[0] = to_tf32(fmaxf(acc[nt][0] + b0, 0.f));      // (g,   col c0)   -> k slot t
        a[1] = to_tf32(fmaxf(acc[nt][2] + b0, 0.f));      // (g+8, col c0)   -> k slot t
        a[2] = to_tf32(fmaxf(acc[nt][1] + b1, 0.f));      // (g,   col c0+1) -> k slot t+4
        a[3] = to_tf32(fmaxf(acc[nt][3] + b1, 0.f));      // (g+8, col c0+1) -> k slot t+4
#pragma unroll
        for (int q8 = 0; q8 < NC / 8; ++q8) {   // B[k slot][n = g]
            if constexpr (HEADS_IN_SW) {
                const float2 hw = *reinterpret_cast<const float2*>(sW + (8 * q8 + g) * PM_PITCH + c0);
                mma_tf32(out[q8], a, to_tf32(hw.x), to_tf32(hw.y));
            } else {
                mma_tf32(out[q8], a, to_tf32(sWh[8 * q8 + g][c0]), to_tf32(sWh[8 * q8 + g][c0 + 1]));
            }
        }
    }
    // out[q8]: (row g, cols 8q8 + 2t, +1), (row g+8, same).  Gather the NC columns of a row across its quad.
    float rowv[2][NC];
#pragma unroll
    for (int q8 = 0; q8 < NC / 8; ++q8) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int src = (lane & ~3) | q, k = 8 * q8 + 2 * q;
            const float v0 = __shfl_sync(0xffffffffu, out[q8][0], src), v1 = __shfl_sync(0xffffffffu, out[q8][1], src);
            const float v2 = __shfl_sync(0xffffffffu, out[q8][2], src), v3 = __shfl_sync(0xffffffffu, out[q8][3], src);
            rowv[0][k] = v0 + sBh[k]; rowv[0][k + 1] = v1 + sBh[k + 1];
            rowv[1][k] = v2 + sBh[k]; rowv[1][k + 1] = v3 + sBh[k + 1];
        }
    }
    // lane t == 0 finishes row g, lane t == 1 finishes row g + 8
    if (t < 2) {
        const int64_t r = row0 + 16 * warp + g + 8 * t;
        if (r < p.m) {
            float z[NC];
#pragma unroll
            for (int k = 0; k < NC; ++k) z[k] = t ? rowv[1][k] : rowv[0][k];
            int a;
            float lp, ent, value;
            pb_sample_row<NC>(z, p.n_act, pb_policy_uniform(p.seed, offset, r), a, lp, ent, value);
            p.actions[r] = a;
            p.logprobs[r] = lp;
            p.values[r] = value;
            if (p.entropies) p.entropies[r] = ent;
        }
    }
    // ---- the last CTA to leave advances the stream counter (every CTA read it before its ticket): the host does not
    //      need a separate "counter += 1" launch per env step
    if (p.ticket) {
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            if (atomicAdd(p.ticket, 1u) == gridDim.x - 1) {
                *p.ticket = 0u;
                *p.counter = offset + 1ull;
                __threadfence();
            }
        }
    }
}

// ---- hidden = 256, 384, 512: the hidden layer in 128-unit chunks.  Chunk c is W_enc rows [128c, 128c + 128) (64 KB),
//      streamed by one 512-byte bulk copy per row into a two-stage ring on mbarriers; per chunk a warp computes its 16
//      rows x 128 hidden units with the fragments of k_policy_mlp_sample, applies bias, ReLU and cvt.rna, and adds the
//      chunk's share of the NC head columns into the same head accumulators (second mma).  The head bias is added once,
//      after the last chunk.  Shared memory: x tile 34 KB + ring 136 KB + heads / encoder bias up to 34 KB -> one
//      128-thread CTA per SM.
//      NC = 32: the whole [32][512] head matrix (64 KB) does not fit beside the ring, so each ring stage also carries
//      the chunk's 128 columns of the 32 head rows (one more 512-byte bulk copy per head row, 17 KB per stage): 204 KB
//      of dynamic shared memory.  A stage is then refilled after the chunk's head product, not before it.
constexpr int PW_HMAX = 512;

template <int NC>
__global__ void __launch_bounds__(PM_THREADS, 1) k_policy_mlp_sample_wide(PolicyParams p, int hid) {
    constexpr bool RING_HEADS = NC > 16;
    constexpr int STAGE_ROWS = RING_HEADS ? 128 + NC : 128;   // W_enc rows of the chunk (| its head columns)
    extern __shared__ __align__(128) float smem[];
    float* sX = smem;                              // [64][136]
    float* sW = smem + PM_ROWS * PM_PITCH;         // [2][STAGE_ROWS][136]: ring stage s holds chunk c with c % 2 == s
    __shared__ float sWh[RING_HEADS ? 1 : NC][PW_HMAX];
    __shared__ float sBe[PW_HMAX];
    __shared__ float sBh[NC];
    __shared__ __align__(8) uint64_t bars[3];      // [0]: obs tile, [1 + s]: ring stage s
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int n_chunks = hid >> 7;
    const int64_t row0 = (int64_t)blockIdx.x * PM_ROWS;
    const int valid = (int)((p.m - row0) < PM_ROWS ? (p.m - row0) : PM_ROWS);
    const uint64_t offset = p.counter ? *p.counter : 0ull;
    constexpr uint32_t CHUNK_BYTES = (uint32_t)STAGE_ROWS * PM_K * 4u;

    if (tid == 0) {
        for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
        mbar_fence_init();
        mbar_expect_tx(&bars[0], (uint32_t)valid * PM_K * 4u);
        mbar_expect_tx(&bars[1], CHUNK_BYTES);
        mbar_expect_tx(&bars[2], CHUNK_BYTES);      // n_chunks >= 2
    }
    if (tid >= valid && tid < PM_ROWS) {
#pragma unroll 8
        for (int q = 0; q < PM_K / 4; ++q) *reinterpret_cast<float4*>(sX + tid * PM_PITCH + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if constexpr (!RING_HEADS)
        for (int i = tid; i < NC * hid; i += PM_THREADS) sWh[i / hid][i % hid] = p.w_heads[i];
    for (int i = tid; i < hid; i += PM_THREADS) sBe[i] = p.b_enc[i];
    if (tid < NC) sBh[tid] = p.b_heads[tid];
    __syncthreads();
    if (tid < valid) tma_load_1d(sX + tid * PM_PITCH, p.obs + (row0 + tid) * p.obs_stride, PM_K * 4u, &bars[0]);
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        tma_load_1d(sW + (s * STAGE_ROWS + tid) * PM_PITCH, p.w_enc + (int64_t)(128 * s + tid) * PM_K, PM_K * 4u, &bars[1 + s]);
        if (RING_HEADS && tid < NC)
            tma_load_1d(sW + (s * STAGE_ROWS + 128 + tid) * PM_PITCH, p.w_heads + (int64_t)tid * hid + 128 * s, PM_H * 4u,
                        &bars[1 + s]);
    }

    float out[NC / 8][4];
#pragma unroll
    for (int q8 = 0; q8 < NC / 8; ++q8) { out[q8][0] = out[q8][1] = out[q8][2] = out[q8][3] = 0.f; }
    const float* xa = sX + (16 * warp + g) * PM_PITCH + 2 * t;
    mbar_wait(&bars[0], 0);
#pragma unroll 1
    for (int c = 0; c < n_chunks; ++c) {
        const int s = c & 1;
        mbar_wait(&bars[1 + s], (uint32_t)(c >> 1) & 1u);
        float acc[16][4];
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
        const float* wbase = sW + (s * STAGE_ROWS + g) * PM_PITCH + 2 * t;
#pragma unroll 4
        for (int ks = 0; ks < 16; ++ks) {
            const float2 x0 = *reinterpret_cast<const float2*>(xa + 8 * ks);
            const float2 x1 = *reinterpret_cast<const float2*>(xa + 8 * PM_PITCH + 8 * ks);
            const uint32_t a[4] = {to_tf32(x0.x), to_tf32(x1.x), to_tf32(x0.y), to_tf32(x1.y)};
#pragma unroll
            for (int nt = 0; nt < 16; ++nt) {
                const float2 w = *reinterpret_cast<const float2*>(wbase + 8 * nt * PM_PITCH + 8 * ks);
                mma_tf32(acc[nt], a, __float_as_uint(w.x), __float_as_uint(w.y));
            }
        }
        // stage s is free once every warp has read it: refill it with chunk c + 2 (tid 0 arrives with the byte count
        // before the barrier, so the copies can only complete the phase after it)
        if constexpr (!RING_HEADS) {
            if (c + 2 < n_chunks && tid == 0) mbar_expect_tx(&bars[1 + s], CHUNK_BYTES);
            __syncthreads();
            if (c + 2 < n_chunks)
                tma_load_1d(sW + (s * 128 + tid) * PM_PITCH, p.w_enc + (int64_t)(128 * (c + 2) + tid) * PM_K, PM_K * 4u,
                            &bars[1 + s]);
        }
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) {
            const int c0 = 128 * c + 8 * nt + 2 * t;
            const float b0 = sBe[c0], b1 = sBe[c0 + 1];
            uint32_t a[4];
            a[0] = to_tf32(fmaxf(acc[nt][0] + b0, 0.f));
            a[1] = to_tf32(fmaxf(acc[nt][2] + b0, 0.f));
            a[2] = to_tf32(fmaxf(acc[nt][1] + b1, 0.f));
            a[3] = to_tf32(fmaxf(acc[nt][3] + b1, 0.f));
#pragma unroll
            for (int q8 = 0; q8 < NC / 8; ++q8) {
                if constexpr (RING_HEADS) {   // the chunk's columns of head row 8 q8 + g, from the ring stage
                    const float2 hw = *reinterpret_cast<const float2*>(
                        sW + (s * STAGE_ROWS + 128 + 8 * q8 + g) * PM_PITCH + 8 * nt + 2 * t);
                    mma_tf32(out[q8], a, to_tf32(hw.x), to_tf32(hw.y));
                } else {
                    mma_tf32(out[q8], a, to_tf32(sWh[8 * q8 + g][c0]), to_tf32(sWh[8 * q8 + g][c0 + 1]));
                }
            }
        }
        if constexpr (RING_HEADS) {   // stage s (W_enc rows and head columns) is free: refill it with chunk c + 2
            if (c + 2 < n_chunks && tid == 0) mbar_expect_tx(&bars[1 + s], CHUNK_BYTES);
            __syncthreads();
            if (c + 2 < n_chunks) {
                tma_load_1d(sW + (s * STAGE_ROWS + tid) * PM_PITCH, p.w_enc + (int64_t)(128 * (c + 2) + tid) * PM_K,
                            PM_K * 4u, &bars[1 + s]);
                if (tid < NC)
                    tma_load_1d(sW + (s * STAGE_ROWS + 128 + tid) * PM_PITCH, p.w_heads + (int64_t)tid * hid + 128 * (c + 2),
                                PM_H * 4u, &bars[1 + s]);
            }
        }
    }
    float rowv[2][NC];
#pragma unroll
    for (int q8 = 0; q8 < NC / 8; ++q8) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int src = (lane & ~3) | q, k = 8 * q8 + 2 * q;
            const float v0 = __shfl_sync(0xffffffffu, out[q8][0], src), v1 = __shfl_sync(0xffffffffu, out[q8][1], src);
            const float v2 = __shfl_sync(0xffffffffu, out[q8][2], src), v3 = __shfl_sync(0xffffffffu, out[q8][3], src);
            rowv[0][k] = v0 + sBh[k]; rowv[0][k + 1] = v1 + sBh[k + 1];
            rowv[1][k] = v2 + sBh[k]; rowv[1][k + 1] = v3 + sBh[k + 1];
        }
    }
    if (t < 2) {
        const int64_t r = row0 + 16 * warp + g + 8 * t;
        if (r < p.m) {
            float z[NC];
#pragma unroll
            for (int k = 0; k < NC; ++k) z[k] = t ? rowv[1][k] : rowv[0][k];
            int a;
            float lp, ent, value;
            pb_sample_row<NC>(z, p.n_act, pb_policy_uniform(p.seed, offset, r), a, lp, ent, value);
            p.actions[r] = a;
            p.logprobs[r] = lp;
            p.values[r] = value;
            if (p.entropies) p.entropies[r] = ent;
        }
    }
    if (p.ticket) {
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            if (atomicAdd(p.ticket, 1u) == gridDim.x - 1) {
                *p.ticket = 0u;
                *p.counter = offset + 1ull;
                __threadfence();
            }
        }
    }
}

template <int NC>
int launch(const PolicyParams& p, int hid, cudaStream_t stream) {
    const unsigned grid = (unsigned)pb_ceil_div(p.m, PM_ROWS);
    if (hid == PM_H) {
        const size_t smem = (size_t)(PM_ROWS + PM_H) * PM_PITCH * sizeof(float);
        PB_CUDA(cudaFuncSetAttribute(k_policy_mlp_sample<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_policy_mlp_sample<NC><<<grid, PM_THREADS, smem, stream>>>(p);
    } else {
        const size_t smem = (size_t)(PM_ROWS + 2 * (NC > 16 ? 128 + NC : 128)) * PM_PITCH * sizeof(float);
        PB_CUDA(cudaFuncSetAttribute(k_policy_mlp_sample_wide<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_policy_mlp_sample_wide<NC><<<grid, PM_THREADS, smem, stream>>>(p, hid);
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

}  // namespace

extern "C" int pb_policy_mlp_sample(const float* obs, int64_t obs_stride, const float* w_enc, const float* b_enc,
                                    const float* w_heads, const float* b_heads, int64_t m, int32_t in_features,
                                    int32_t hidden_size, int32_t n_act, uint64_t seed, uint64_t* counter_dev,
                                    uint32_t* ticket_dev, int64_t* actions, float* logprobs, float* values, float* entropies, void* stream) {
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "pb_policy_mlp_sample: negative m");
    if (m == 0) return PB_OK;
    PB_REQUIRE(in_features == PM_K && hidden_size >= PM_H && hidden_size <= PW_HMAX && hidden_size % PM_H == 0,
               PB_ERR_UNSUPPORTED,
               "pb_policy_mlp_sample: built for 128 input features and 128, 256, 384 or 512 hidden units (got %d, %d)",
               in_features, hidden_size);
    PB_REQUIRE(n_act >= 1 && n_act <= 31, PB_ERR_UNSUPPORTED, "pb_policy_mlp_sample: n_act must be in [1, 31]");
    PB_REQUIRE(obs && w_enc && b_enc && w_heads && b_heads && actions && logprobs && values, PB_ERR_INVALID,
               "pb_policy_mlp_sample: null pointer");
    PB_REQUIRE(obs_stride >= PM_K && obs_stride % 4 == 0 && ((uintptr_t)obs & 15) == 0 && ((uintptr_t)w_enc & 15) == 0,
               PB_ERR_INVALID, "pb_policy_mlp_sample: obs / w_enc must be 16-byte aligned, stride a multiple of 4");
    PB_REQUIRE(!ticket_dev || counter_dev, PB_ERR_INVALID, "pb_policy_mlp_sample: ticket_dev needs counter_dev");
    PB_REQUIRE(n_act + 1 <= 16 || ((uintptr_t)w_heads & 15) == 0, PB_ERR_INVALID,
               "pb_policy_mlp_sample: w_heads must be 16-byte aligned for more than 15 actions");
    PolicyParams p{obs, obs_stride, w_enc, b_enc, w_heads, b_heads, m, n_act, seed, counter_dev, ticket_dev,
                   actions, logprobs, values, entropies};
    // w_heads / b_heads: the head matrix of models.Default.head_matrix, 8 rows for n_act <= 7, 16 for n_act <= 15, else 32
    cudaStream_t s = (cudaStream_t)stream;
    return n_act + 1 <= 8 ? launch<8>(p, hidden_size, s) : n_act + 1 <= 16 ? launch<16>(p, hidden_size, s) : launch<32>(p, hidden_size, s);
}
