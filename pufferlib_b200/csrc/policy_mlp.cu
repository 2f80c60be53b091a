// policy_mlp.cu -- the rollout-time forward of models.Default fused with the sampling epilogue, ONE launch per env step.
//
// Replaces, inside the evaluate loop (reference clean_pufferl.py:107-117), the chain
//   encoder Linear + ReLU -> action head + value head (pufferlib/models.py:12-62) -> sample_logits
//   (pufferlib/frameworks/cleanrl.py:25-47) -> Experience.store of value / logprob / action (clean_pufferl.py:443-446)
// which the library path runs as 2 GEMM launches + sampler + counter update.  At rollout time M = num_envs rows (16384),
// so the GEMMs are tiny (0.5 GFLOP at H = 128) and launch/latency bound; here a CTA owns 64 rows:
//   * the 64x128 fp32 observation tile and the encoder weights land in shared memory as 512-byte bulk copies
//     (cp.async.bulk, one per row, on mbarriers);
//   * the hidden layer in chunks of 128 units: hidden = relu(X W^T + b) on the tensor cores (mma.sync m16n8k8 TF32, fp32
//     accumulate; a warp owns 16 rows x 128 columns, accumulators stay in registers -- `hidden` is never written to
//     memory);
//   * the two heads (n_act logits + value, padded to NC = 8 columns for n_act <= 7, 16 for n_act <= 15, 32 for
//     n_act <= 31) are a second mma whose A operand is the chunk's accumulator fragment itself (the k order of the second
//     product is permuted to match the C-fragment layout), accumulated over the chunks; NC = 16 and 32 are two and four
//     n8 blocks on the same A fragments;
//   * pb_sample_epilogue (policy_sample.cuh) adds the head bias, samples, and writes action, logprob, value straight into
//     the rollout rows.
// Tensor-core path note: this is a 128x128x128 tile per chunk, far below the size where a wgmma pipeline pays; the large
// training GEMMs of the generic path stay on cuBLAS.
//
// One kernel template, k_policy_mlp_sample<NC, HMAX>, for every hidden size H (a multiple of 128 up to HMAX):
//   * HMAX = 128: W_enc stays resident, [128][136] (68 KB), loaded in two halves on two mbarriers so the first 8 n-tiles
//     start while the second half is in flight: 104 KB of dynamic shared memory -> 2 CTAs per SM, 256 CTAs at 16384
//     rows.  NC = 32: a static [32][128] head copy (16 KB) would leave room for one CTA per SM only, so the head rows are
//     read into registers (8 float4 per thread) before the hidden product and written over W_enc once every warp is done
//     with it.
//   * HMAX = 512 (H = 256, 384, 512): chunk c is W_enc rows [128c, 128c + 128) (64 KB), streamed into a two-stage ring;
//     x tile 34 KB + ring 136 KB + heads / encoder bias up to 34 KB -> one CTA per SM.  NC = 32: the whole [32][512]
//     head matrix (64 KB) does not fit beside the ring, so each ring stage also carries the chunk's 128 columns of the 32
//     head rows (17 KB per stage, 204 KB of dynamic shared memory), and a stage is refilled after the chunk's head
//     product, not before it.
// Every instance sums in the same order: acc[nt] over k-steps 0..15, the head accumulators over chunks, then n-tiles.
#include "pb_common.cuh"
#include "policy_sample.cuh"
#include "tma.cuh"

namespace {

constexpr int PM_K = 128;           // obs features
constexpr int PM_H = 128;           // hidden units per chunk
constexpr int PM_HMAX = 512;        // largest hidden size
constexpr int PM_PITCH = PM_K + 8;  // shared row pitch in floats (544 B): conflict-free 64-bit fragment loads
constexpr int PM_ROWS = 64;         // rows per CTA, one warp per 16 rows
constexpr int PM_THREADS = 2 * PM_ROWS;

struct PolicyParams {
    const float* obs; int64_t obs_stride;      // [M][128] fp32
    const float* w_enc; const float* b_enc;    // [H][128], [H]
    const float* w_heads; const float* b_heads;  // [NC][H], [NC]  (n_act logits | value | zero pad)
    int hid;
    PbSampleOut sample;
};

// Rows of sW after the x tile: W_enc whole at HMAX = 128, else two ring stages of a chunk's W_enc rows (| its head
// columns at NC = 32).
__host__ __device__ constexpr int pm_stage_rows(int nc) { return nc > 16 ? PM_H + nc : PM_H; }
constexpr int pm_w_rows(int nc, int hmax) { return hmax == PM_H ? PM_H : 2 * pm_stage_rows(nc); }

// acc[nt] += x W^T over the 16 k-steps of a chunk, n-tiles [N0, N1): a warp's 16 rows x 8 hidden units per n-tile.
// The sum over k is order-free, so k slots (t, t+4) of a k-step are mapped to the ADJACENT columns (8ks + 2t,
// 8ks + 2t + 1) for both operands: every fragment is one 64-bit shared load (pitch 136: conflict-free).  A is rounded to
// TF32 here; W arrives pre-rounded (models.Default.encoder_weight_tf32).
template <int N0, int N1>
__device__ __forceinline__ void hidden_product(float (&acc)[16][4], const float* xa, const float* wbase) {
#pragma unroll 4
    for (int ks = 0; ks < 16; ++ks) {
        const float2 x0 = *reinterpret_cast<const float2*>(xa + 8 * ks);
        const float2 x1 = *reinterpret_cast<const float2*>(xa + 8 * PM_PITCH + 8 * ks);
        const uint32_t a[4] = {to_tf32(x0.x), to_tf32(x1.x), to_tf32(x0.y), to_tf32(x1.y)};
#pragma unroll
        for (int nt = N0; nt < N1; ++nt) {
            const float2 w = *reinterpret_cast<const float2*>(wbase + 8 * nt * PM_PITCH + 8 * ks);   // B[k][n] = W[n][k]
            mma_tf32(acc[nt], a, __float_as_uint(w.x), __float_as_uint(w.y));
        }
    }
}

// Bias + ReLU on a chunk's accumulators, then out += hidden @ Wh^T as a second mma with A = the C fragments: the C
// fragment of n-tile nt holds columns 8nt + {2t, 2t+1} of rows {g, g+8}; use them as k slots {t, t+4}.  Head block q8
// (columns 8q8..8q8+7) takes B from head row 8q8 + g: wh[(8q8 + g) * pitch + column of the chunk].  be: the chunk's
// encoder bias.
template <int NC>
__device__ __forceinline__ void head_product(float (&out)[NC / 8][4], const float (&acc)[16][4], const float* be,
                                             const float* wh, int pitch, int g, int t) {
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
        const int c0 = 8 * nt + 2 * t;
        const float b0 = be[c0], b1 = be[c0 + 1];
        uint32_t a[4];
        a[0] = to_tf32(fmaxf(acc[nt][0] + b0, 0.f));      // (g,   col c0)   -> k slot t
        a[1] = to_tf32(fmaxf(acc[nt][2] + b0, 0.f));      // (g+8, col c0)   -> k slot t
        a[2] = to_tf32(fmaxf(acc[nt][1] + b1, 0.f));      // (g,   col c0+1) -> k slot t+4
        a[3] = to_tf32(fmaxf(acc[nt][3] + b1, 0.f));      // (g+8, col c0+1) -> k slot t+4
#pragma unroll
        for (int q8 = 0; q8 < NC / 8; ++q8) {   // B[k slot][n = g]
            const float2 hw = *reinterpret_cast<const float2*>(wh + (8 * q8 + g) * pitch + c0);
            mma_tf32(out[q8], a, to_tf32(hw.x), to_tf32(hw.y));
        }
    }
}

// Shared memory sets the occupancy (2 CTAs per SM at HMAX = 128, 1 at 512); the bound of 1 CTA per SM leaves ptxas the
// whole register file to schedule with.
template <int NC, int HMAX>
__global__ void __launch_bounds__(PM_THREADS, 1) k_policy_mlp_sample(PolicyParams p) {
    constexpr bool RESIDENT = HMAX == PM_H;        // W_enc whole in sW; else a two-stage ring of chunks
    constexpr bool BIG_HEADS = NC > 16;            // head rows in sW (over W_enc, or with each ring stage), not in sWh
    constexpr int STAGE_ROWS = RESIDENT ? PM_H : pm_stage_rows(NC);
    constexpr uint32_t ROW_BYTES = PM_K * 4u;
    extern __shared__ __align__(128) float smem[];
    float* sX = smem;                              // [64][136]
    float* sW = smem + PM_ROWS * PM_PITCH;         // [pm_w_rows][136]  (row = hidden unit, col = input feature)
    __shared__ __align__(16) float sWh[BIG_HEADS ? 1 : NC][HMAX];
    __shared__ float sBe[HMAX];
    __shared__ float sBh[NC];
    // resident: [0] obs tile + W rows 0..63, [1] W rows 64..127; ring: [0] obs tile, [1 + s] ring stage s
    __shared__ __align__(8) uint64_t bars[RESIDENT ? 2 : 3];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int hid = RESIDENT ? PM_H : p.hid;
    const int n_chunks = hid >> 7;
    const int64_t row0 = (int64_t)blockIdx.x * PM_ROWS;
    const int valid = (int)((p.sample.m - row0) < PM_ROWS ? (p.sample.m - row0) : PM_ROWS);
    const uint64_t offset = p.sample.counter ? *p.sample.counter : 0ull;   // read by every CTA before its exit ticket

    // ring stage s <- chunk c: W_enc rows [128c, 128c + 128) (| the chunk's columns of the NC head rows)
    auto load_stage = [&](int s, int c) {
        tma_load_1d(sW + (s * STAGE_ROWS + tid) * PM_PITCH, p.w_enc + (int64_t)(PM_H * c + tid) * PM_K, ROW_BYTES,
                    &bars[1 + s]);
        if (BIG_HEADS && tid < NC)
            tma_load_1d(sW + (s * STAGE_ROWS + PM_H + tid) * PM_PITCH, p.w_heads + (int64_t)tid * hid + PM_H * c,
                        ROW_BYTES, &bars[1 + s]);
    };

    // ---- stage the observation tile and the weights: one 512-byte bulk copy (TMA engine) per row
    if (tid == 0) {
        for (int i = 0; i < (RESIDENT ? 2 : 3); ++i) mbar_init(&bars[i], 1);
        mbar_fence_init();
        if constexpr (RESIDENT) {
            mbar_expect_tx(&bars[0], (uint32_t)(valid + 64) * ROW_BYTES);
            mbar_expect_tx(&bars[1], 64u * ROW_BYTES);
        } else {
            mbar_expect_tx(&bars[0], (uint32_t)valid * ROW_BYTES);
            mbar_expect_tx(&bars[1], STAGE_ROWS * ROW_BYTES);
            mbar_expect_tx(&bars[2], STAGE_ROWS * ROW_BYTES);   // n_chunks >= 2
        }
    }
    if (tid >= valid && tid < PM_ROWS) {           // rows past M: zeros
#pragma unroll 8
        for (int q = 0; q < PM_K / 4; ++q) *reinterpret_cast<float4*>(sX + tid * PM_PITCH + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    constexpr int WH_REGS = RESIDENT && BIG_HEADS ? NC * PM_H / 4 / PM_THREADS : 1;
    float4 wh[WH_REGS];                            // resident NC = 32: float4 i = tid + 128 j of w_heads
    if constexpr (RESIDENT && BIG_HEADS) {
#pragma unroll
        for (int j = 0; j < WH_REGS; ++j) wh[j] = *reinterpret_cast<const float4*>(p.w_heads + 4 * (tid + PM_THREADS * j));
    }
    // encoder bias and, at NC <= 16, the head rows: column 128c + tid of each chunk c.  Every load is issued before the
    // first store, so one round trip to memory covers them all.
    constexpr int SWH_ROWS = BIG_HEADS ? 0 : NC;
    float be[HMAX / PM_H], whc[HMAX / PM_H][SWH_ROWS + 1];
#pragma unroll
    for (int c = 0; c < HMAX / PM_H; ++c) {
        if (c < n_chunks) {
            be[c] = p.b_enc[PM_H * c + tid];
#pragma unroll
            for (int r = 0; r < SWH_ROWS; ++r) whc[c][r] = p.w_heads[r * hid + PM_H * c + tid];
        }
    }
#pragma unroll
    for (int c = 0; c < HMAX / PM_H; ++c) {
        if (c < n_chunks) {
            sBe[PM_H * c + tid] = be[c];
#pragma unroll
            for (int r = 0; r < SWH_ROWS; ++r) sWh[r][PM_H * c + tid] = whc[c][r];
        }
    }
    if (tid < NC) sBh[tid] = p.b_heads[tid];
    __syncthreads();
    if (tid < valid) tma_load_1d(sX + tid * PM_PITCH, p.obs + (row0 + tid) * p.obs_stride, ROW_BYTES, &bars[0]);
    if constexpr (RESIDENT) {
        tma_load_1d(sW + tid * PM_PITCH, p.w_enc + (int64_t)tid * PM_K, ROW_BYTES, &bars[tid >> 6]);
    } else {
        load_stage(0, 0);
        load_stage(1, 1);
        mbar_wait(&bars[0], 0);
    }

    // ---- per chunk: warp w's rows 16w..16w+15 x 128 hidden units (16 n-tiles), K = 128 (16 k-steps), then its share of
    //      the NC head columns
    float out[NC / 8][4];
#pragma unroll
    for (int q8 = 0; q8 < NC / 8; ++q8) { out[q8][0] = out[q8][1] = out[q8][2] = out[q8][3] = 0.f; }
    const float* xa = sX + (16 * warp + g) * PM_PITCH + 2 * t;
#pragma unroll 1
    for (int c = 0; c < n_chunks; ++c) {
        const int s = c & 1;
        const float* stage = sW + s * STAGE_ROWS * PM_PITCH;
        // stage s is free once every warp has read it: refill it with chunk c + 2 (tid 0 arrives with the byte count
        // before the barrier, so the copies can only complete the phase after it)
        auto refill = [&] {
            if (c + 2 < n_chunks && tid == 0) mbar_expect_tx(&bars[1 + s], STAGE_ROWS * ROW_BYTES);
            __syncthreads();
            if (c + 2 < n_chunks) load_stage(s, c + 2);
        };
        float acc[16][4];
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
        if constexpr (RESIDENT) {
            mbar_wait(&bars[0], 0);
            hidden_product<0, 8>(acc, xa, sW + g * PM_PITCH + 2 * t);
            mbar_wait(&bars[1], 0);
            hidden_product<8, 16>(acc, xa, sW + g * PM_PITCH + 2 * t);
        } else {
            mbar_wait(&bars[1 + s], (uint32_t)(c >> 1) & 1u);
            hidden_product<0, 16>(acc, xa, stage + g * PM_PITCH + 2 * t);
        }
        if constexpr (RESIDENT && BIG_HEADS) {   // every warp is done with W_enc: head row r -> sW row r
            __syncthreads();
#pragma unroll
            for (int j = 0; j < WH_REGS; ++j) {
                const int i = tid + PM_THREADS * j;
                *reinterpret_cast<float4*>(sW + (i >> 5) * PM_PITCH + 4 * (i & 31)) = wh[j];
            }
            __syncthreads();
            head_product<NC>(out, acc, sBe, sW, PM_PITCH, g, t);
        } else if constexpr (BIG_HEADS) {         // the chunk's head columns ride in the stage: refill after them
            head_product<NC>(out, acc, sBe + PM_H * c, stage + PM_H * PM_PITCH, PM_PITCH, g, t);
            refill();
        } else {
            if constexpr (!RESIDENT) refill();
            head_product<NC>(out, acc, sBe + PM_H * c, &sWh[0][PM_H * c], HMAX, g, t);
        }
    }
    pb_sample_epilogue<NC>(out, sBh, p.sample, row0 + 16 * warp + g, offset);
}

template <int NC>
int launch(const PolicyParams& p, cudaStream_t stream) {
    const bool resident = p.hid == PM_H;
    void (*kernel)(PolicyParams) = resident ? k_policy_mlp_sample<NC, PM_H> : k_policy_mlp_sample<NC, PM_HMAX>;
    const size_t smem = (size_t)(PM_ROWS + pm_w_rows(NC, resident ? PM_H : PM_HMAX)) * PM_PITCH * sizeof(float);
    PB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)pb_ceil_div(p.sample.m, PM_ROWS), PM_THREADS, smem, stream>>>(p);
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
    PB_REQUIRE(in_features == PM_K && hidden_size >= PM_H && hidden_size <= PM_HMAX && hidden_size % PM_H == 0,
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
    PolicyParams p{obs, obs_stride, w_enc, b_enc, w_heads, b_heads, hidden_size,
                   {m, n_act, seed, counter_dev, ticket_dev, actions, logprobs, values, entropies}};
    // w_heads / b_heads: the head matrix of models.Default.head_matrix, 8 rows for n_act <= 7, 16 for n_act <= 15, else 32
    cudaStream_t s = (cudaStream_t)stream;
    return n_act + 1 <= 8 ? launch<8>(p, s) : n_act + 1 <= 16 ? launch<16>(p, s) : launch<32>(p, s);
}
