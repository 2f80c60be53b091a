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
//   * the two heads (n_act logits + value, padded to 8 columns) are a second mma whose A operand is the accumulator
//     fragment itself (the k order of the second product is permuted to match the C-fragment layout);
//   * a quad shuffle gathers each row's 8 outputs, one lane per row does logsumexp / inverse-CDF sampling / logprob /
//     entropy and writes action, logprob, value straight into the rollout rows.
// Tensor-core path note: this is a 128x128x128 tile per CTA, far below the size where a wgmma pipeline pays; the large
// training GEMMs of the generic path stay on cuBLAS.
#include "pb_common.cuh"
#include "tma.cuh"

namespace {

constexpr int PM_K = 128;           // obs features
constexpr int PM_H = 128;           // hidden units
constexpr int PM_PITCH = PM_K + 8;  // shared row pitch in floats (544 B): conflict-free 64-bit fragment loads

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
struct PolicyParams {
    const float* obs; int64_t obs_stride;      // [M][128] fp32
    const float* w_enc; const float* b_enc;    // [128][128], [128]
    const float* w_heads; const float* b_heads;  // [8][128], [8]  (n_act logits | value | zero pad)
    int64_t m; int n_act;
    uint64_t seed; uint64_t* counter; unsigned int* ticket;
    int64_t* actions; float* logprobs; float* values; float* entropies;   // [M] each (entropies may be null)
};

// 64 rows per CTA, one warp per 16 rows: 128 threads, 104 KB shared -> 2 CTAs per SM, 256 CTAs at 16384 rows
constexpr int PM_ROWS = 64;
constexpr int PM_THREADS = 2 * PM_ROWS;

__global__ void __launch_bounds__(PM_THREADS) k_policy_mlp_sample(PolicyParams p) {
    extern __shared__ __align__(128) float smem[];
    float* sX = smem;                              // [64][136]
    float* sW = smem + PM_ROWS * PM_PITCH;         // [128][136]  (row = hidden unit, col = input feature)
    __shared__ float sWh[8][PM_H];
    __shared__ float sBe[PM_H];
    __shared__ float sBh[8];
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
    for (int i = tid; i < 8 * PM_H; i += PM_THREADS) sWh[i >> 7][i & 127] = p.w_heads[i];
    if (tid < PM_H) sBe[tid] = p.b_enc[tid];
    if (tid < 8) sBh[tid] = p.b_heads[tid];
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
    // ---- bias + ReLU on the accumulators; heads = hidden @ Wh^T as a second mma with A = the C fragments:
    //      C fragment of n-tile nt holds columns 8nt + {2t, 2t+1} of rows {g, g+8}; use them as k slots {t, t+4}
    float out[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
        const int c0 = 8 * nt + 2 * t;
        const float b0 = sBe[c0], b1 = sBe[c0 + 1];
        uint32_t a[4];
        a[0] = to_tf32(fmaxf(acc[nt][0] + b0, 0.f));      // (g,   col c0)   -> k slot t
        a[1] = to_tf32(fmaxf(acc[nt][2] + b0, 0.f));      // (g+8, col c0)   -> k slot t
        a[2] = to_tf32(fmaxf(acc[nt][1] + b1, 0.f));      // (g,   col c0+1) -> k slot t+4
        a[3] = to_tf32(fmaxf(acc[nt][3] + b1, 0.f));      // (g+8, col c0+1) -> k slot t+4
        mma_tf32(out, a, to_tf32(sWh[g][c0]), to_tf32(sWh[g][c0 + 1]));   // B[k slot][n = g]
    }
    // out: (row g, cols 2t, 2t+1), (row g+8, cols 2t, 2t+1).  Gather the 8 columns of a row across its quad.
    float rowv[2][8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int src = (lane & ~3) | q;
        const float v0 = __shfl_sync(0xffffffffu, out[0], src), v1 = __shfl_sync(0xffffffffu, out[1], src);
        const float v2 = __shfl_sync(0xffffffffu, out[2], src), v3 = __shfl_sync(0xffffffffu, out[3], src);
        rowv[0][2 * q] = v0 + sBh[2 * q]; rowv[0][2 * q + 1] = v1 + sBh[2 * q + 1];
        rowv[1][2 * q] = v2 + sBh[2 * q]; rowv[1][2 * q + 1] = v3 + sBh[2 * q + 1];
    }
    // lane t == 0 finishes row g, lane t == 1 finishes row g + 8
    if (t < 2) {
        const int64_t r = row0 + 16 * warp + g + 8 * t;
        if (r < p.m) {
            float z[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) z[k] = t ? rowv[1][k] : rowv[0][k];
            float mx = -INFINITY;
#pragma unroll
            for (int k = 0; k < 8; ++k) if (k < p.n_act) mx = fmaxf(mx, z[k]);
            float sum = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) if (k < p.n_act) sum += expf(z[k] - mx);
            const float lse = mx + logf(sum);
            const uint32_t rnd = pb_mix32(p.seed * 0x9E3779B97F4A7C15ull + offset * 0xD1B54A32D192ED03ull +
                                          (uint64_t)r * 0x2545F4914F6CDD1Dull);
            const float u = (float)(rnd >> 8) * (1.0f / 16777216.0f);
            float cdf = 0.f, ent = 0.f, lp = 0.f, value = 0.f;
            int a = -1;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (k < p.n_act) {
                    const float nl = z[k] - lse, pk = expf(nl);
                    ent -= pk * nl;
                    cdf += pk;
                    if (a < 0 && u < cdf) { a = k; lp = nl; }
                }
                if (k == p.n_act) value = z[k];
            }
            if (a < 0) {   // rounding left cdf a hair below u: last action with non-negligible probability
#pragma unroll
                for (int k = 7; k >= 0; --k)
                    if (a < 0 && k < p.n_act && z[k] - lse > -80.f) { a = k; lp = z[k] - lse; }
                if (a < 0) { a = p.n_act - 1; lp = z[a] - lse; }
            }
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

}  // namespace

extern "C" int pb_policy_mlp_sample(const float* obs, int64_t obs_stride, const float* w_enc, const float* b_enc,
                                    const float* w_heads, const float* b_heads, int64_t m, int32_t in_features,
                                    int32_t hidden_size, int32_t n_act, uint64_t seed, uint64_t* counter_dev,
                                    uint32_t* ticket_dev, int64_t* actions, float* logprobs, float* values, float* entropies, void* stream) {
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "pb_policy_mlp_sample: negative m");
    if (m == 0) return PB_OK;
    PB_REQUIRE(in_features == PM_K && hidden_size == PM_H, PB_ERR_UNSUPPORTED,
               "pb_policy_mlp_sample: built for 128 input features and 128 hidden units (got %d, %d)", in_features,
               hidden_size);
    PB_REQUIRE(n_act >= 1 && n_act <= 7, PB_ERR_UNSUPPORTED, "pb_policy_mlp_sample: n_act must be in [1, 7]");
    PB_REQUIRE(obs && w_enc && b_enc && w_heads && b_heads && actions && logprobs && values, PB_ERR_INVALID,
               "pb_policy_mlp_sample: null pointer");
    PB_REQUIRE(obs_stride >= PM_K && obs_stride % 4 == 0 && ((uintptr_t)obs & 15) == 0 && ((uintptr_t)w_enc & 15) == 0,
               PB_ERR_INVALID, "pb_policy_mlp_sample: obs / w_enc must be 16-byte aligned, stride a multiple of 4");
    PB_REQUIRE(!ticket_dev || counter_dev, PB_ERR_INVALID, "pb_policy_mlp_sample: ticket_dev needs counter_dev");
    PolicyParams p{obs, obs_stride, w_enc, b_enc, w_heads, b_heads, m, n_act, seed, counter_dev, ticket_dev,
                   actions, logprobs, values, entropies};
    const size_t smem = (size_t)(PM_ROWS + PM_H) * PM_PITCH * sizeof(float);
    PB_CUDA(cudaFuncSetAttribute(k_policy_mlp_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_policy_mlp_sample<<<(unsigned)pb_ceil_div(m, PM_ROWS), PM_THREADS, smem, (cudaStream_t)stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
