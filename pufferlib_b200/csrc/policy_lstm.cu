// policy_lstm.cu -- the rollout-time step of LSTMWrapper(models.Default) fused with the sampling epilogue and the in-place
// LSTM state update, ONE launch per env step.
//
// Replaces, inside the evaluate loop (reference clean_pufferl.py:100-117), the chain
//   encoder Linear + ReLU (pufferlib/models.py:12-62) -> nn.LSTM on a length-1 sequence (models.py:64-111) -> both heads
//   -> sample_logits (frameworks/cleanrl.py:25-47) -> lstm_h / lstm_c[:, env_id] = h, c (clean_pufferl.py:100-105) ->
//   Experience.store of value / logprob / action (clean_pufferl.py:443-446)
// which the library path runs as a GEMM, cuDNN's LSTM (the [N][512] gates through HBM), a head GEMM, about ten sampling
// kernels and three copies.  Per row r < m:
//   e   = relu(x W_enc^T + b_enc)                       x: [m][F] fp32, F <= 128
//   z   = e W_ih^T + h W_hh^T + (b_ih + b_hh)           [512], PyTorch gate order i, f, g, o
//   c'  = sigmoid(f) c + sigmoid(i) tanh(g),  h' = sigmoid(o) tanh(c')     (h, c overwritten in place)
//   out = h' W_cat^T + b_cat                            n_act logits | value | zero pad (8 or 16 columns)
//   then the sampling epilogue and row stores that pb_policy_mlp_sample uses too (pb_sample_epilogue, policy_sample.cuh).
// The state is not reset on done, like the reference and the unfused path.
//
// Layout.  A CTA owns 128 rows, 8 warps x 16 rows, 1 CTA per SM (128 CTAs at N = 16384: one wave on 132 SMs).
//   * x is staged by coalesced loads into a zero-padded [128][136] tile (squared rows are 196 B: not 16-byte aligned, so
//     no bulk copy); W_enc arrives pre-packed [128][136] (TF32, zero-padded K) in one bulk copy (TMA engine).
//   * encoder: mma.sync m16n8k8 TF32, a warp's 16 x 128 accumulator tile stays in registers.  relu(acc + b) becomes the A
//     fragments of the gate product directly (the k-slot trick of policy_mlp.cu: k slots (t, t+4) of k-step ks are the
//     ADJACENT columns 8ks + 2t, 8ks + 2t + 1 for both operands); h_prev is loaded from HBM straight into A fragments of
//     the same shape.  The whole [16 rows][256] A operand (e | h) lives in 128 registers per thread for the gate loop.
//   * gates: 16 chunks of 8 hidden units; a chunk is 32 gate columns [i(8) | f(8) | g(8) | o(8)], so n-tile j of the
//     chunk is gate j and a thread's accumulator columns 2t, 2t+1 are units 8ch + 2t, 8ch + 2t + 1: all four gates of a
//     (row, unit) land in one thread and the cell update needs no exchange.  c is read and written in that fragment
//     layout (float2 per row), h' is written to HBM and becomes the A fragment of the head mma, accumulated over chunks.
//   * the packed gate weights [16][32][264] (528 KB, rows padded to a conflict-free 264-float pitch on the host) stream
//     from L2 through a 2-stage ring of 33 KB bulk copies; the refill of a stage overlaps the cell update of the chunk.
//   Shared memory: x 68 KB + W_enc 68 KB + ring 66 KB + heads / biases 11 KB = 213 KB.
// Why mma.sync and not a wgmma design (m64n32k8 SS, e and h_prev in a swizzled shared A tile): with the A operand in
// registers neither the encoder output nor h_prev goes through shared memory (no swizzled tile, no descriptors), and the
// four gates of a unit still land in one thread.  Measured (H100 80GB HBM3, 400 W power limit, CUDA graph of 256 steps):
// 64.6 us per step at N = 16384 (0.195 of the 12.6 us HBM bound) and 53.5 us at N = 64, i.e. one CTA's 16-chunk chain
// (encoder, then per chunk: ring wait, 128 mma per warp, CTA barrier, cell update) takes ~50 us on its own SM and sets
// the time at every size.  Shortening that chain (wgmma, a deeper ring in the dead x-tile region, 2-CTA multicast of
// the weight stream) is where further speed is; none of it is measured yet.
//
// k_policy_lstm_sample_256 (below) is the same step at LSTM size 256, with e in registers and h_prev in a shared tile.
//
// Operand rounding: every tensor-core operand is rounded to nearest TF32 (cvt.rna: ties away from zero): x, relu(e + b),
// h_prev and h' in the kernel, W_enc and the gate weights on the host (models.LSTMWrapper.fused_operands), W_cat in the
// kernel.  Accumulation, biases, the cell update and the sampler are fp32.
#include "pb_common.cuh"
#include "lstm_cell.cuh"
#include "policy_sample.cuh"
#include "tma.cuh"

namespace {

constexpr int PL_ROWS = 128;                       // rows per CTA
constexpr int PL_THREADS = 256;                    // 8 warps x 16 rows
// PL_F, PL_H, PL_XP, PL_GP, PL_CHUNKS, PL_CHUNK(_BYTES), PL_WENC_BYTES: lstm_cell.cuh

// shared-memory carve-up, in floats
constexpr int SM_X = 0;                            // [128][136] observation tile
constexpr int SM_WE = SM_X + PL_ROWS * PL_XP;      // [128][136] W_enc (row = hidden unit)
constexpr int SM_WG = SM_WE + PL_H * PL_XP;        // [2][32][264] gate-weight ring
constexpr int SM_WH = SM_WG + 2 * PL_CHUNK;        // [16][136] head matrix
constexpr int SM_BE = SM_WH + 16 * PL_XP;          // [128] b_enc
constexpr int SM_BG = SM_BE + PL_H;                // [16][32] b_ih + b_hh, chunk order
constexpr int SM_BH = SM_BG + 4 * PL_H;            // [16] head bias
constexpr int SM_FLOATS = SM_BH + 16;
constexpr size_t PL_SMEM = (size_t)SM_FLOATS * sizeof(float);
static_assert(PL_SMEM <= 227 * 1024, "shared memory over the sm_90 per-CTA limit");
static_assert((SM_WE * 4) % 16 == 0 && (SM_WG * 4) % 16 == 0 && PL_CHUNK_BYTES % 16 == 0, "bulk copy alignment");

struct LstmParams {
    const float* obs; int64_t obs_stride; int in_features;
    const float* w_enc; const float* b_enc;        // [128][136] TF32, [128]
    const float* w_gates; const float* b_gates;    // [16][32][264] TF32, [16][32]
    const float* w_heads; const float* b_heads;    // [NC][128], [NC]
    float* h; int64_t h_stride; float* c; int64_t c_stride;   // [m][128] each, read then overwritten
    PbSampleOut sample;
};

template <int NC>
__global__ void __launch_bounds__(PL_THREADS, 1) k_policy_lstm_sample(LstmParams p) {
    extern __shared__ __align__(128) float smem[];
    float* sX = smem + SM_X;
    float* sWe = smem + SM_WE;
    float* sWg = smem + SM_WG;
    float* sWh = smem + SM_WH;
    float* sBe = smem + SM_BE;
    float* sBg = smem + SM_BG;
    float* sBh = smem + SM_BH;
    __shared__ __align__(8) uint64_t bars[3];      // [0]: W_enc, [1 + s]: gate-weight ring stage s
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int64_t row0 = (int64_t)blockIdx.x * PL_ROWS;
    const int valid = (int)((p.sample.m - row0) < PL_ROWS ? (p.sample.m - row0) : PL_ROWS);
    const uint64_t offset = p.sample.counter ? *p.sample.counter : 0ull;   // read by every CTA before its exit ticket

    // ---- weights by bulk copy: W_enc and the first two gate chunks are in flight while x, h and the small operands load
    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1);
        mbar_fence_init();
        mbar_expect_tx(&bars[0], PL_WENC_BYTES);
        tma_load_1d(sWe, p.w_enc, PL_WENC_BYTES, &bars[0]);
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            mbar_expect_tx(&bars[1 + s], PL_CHUNK_BYTES);
            tma_load_1d(sWg + s * PL_CHUNK, p.w_gates + (int64_t)s * PL_CHUNK, PL_CHUNK_BYTES, &bars[1 + s]);
        }
    }
    // ---- x tile: coalesced loads (any F, any alignment), zero padding past F and past m
    const int F = p.in_features;
    for (int i = tid; i < PL_ROWS * PL_F; i += PL_THREADS) {
        const int r = i >> 7, k = i & (PL_F - 1);
        sX[r * PL_XP + k] = (r < valid && k < F) ? p.obs[(row0 + r) * p.obs_stride + k] : 0.f;
    }
    if (tid < PL_H) sBe[tid] = p.b_enc[tid];
    for (int i = tid; i < 4 * PL_H; i += PL_THREADS) sBg[i] = p.b_gates[i];
    for (int i = tid; i < NC * PL_H; i += PL_THREADS) sWh[(i >> 7) * PL_XP + (i & (PL_H - 1))] = p.w_heads[i];
    if (tid < NC) sBh[tid] = p.b_heads[tid];

    // ---- h_prev straight into A fragments: k-step ks holds columns 8ks + 2t (slot t) and 8ks + 2t + 1 (slot t + 4)
    const int lr = 16 * warp + g;                  // local rows lr (fragment rows g) and lr + 8 (g + 8)
    const bool va = lr < valid, vb = lr + 8 < valid;
    float* h_a = p.h + (row0 + lr) * p.h_stride;
    float* h_b = h_a + 8 * p.h_stride;
    float* c_a = p.c + (row0 + lr) * p.c_stride;
    float* c_b = c_a + 8 * p.c_stride;
    uint32_t hA[16][4];
#pragma unroll
    for (int ks = 0; ks < 16; ++ks) {
        const float2 x0 = va ? *reinterpret_cast<const float2*>(h_a + 8 * ks + 2 * t) : make_float2(0.f, 0.f);
        const float2 x1 = vb ? *reinterpret_cast<const float2*>(h_b + 8 * ks + 2 * t) : make_float2(0.f, 0.f);
        lstm_a_frag(hA[ks], x0.x, x0.y, x1.x, x1.y);
    }
    __syncthreads();                               // x tile, small operands and the barrier inits are visible

    // ---- encoder: warp w owns rows 16w..16w+15 and all 128 hidden columns; K = F rounded up to 8 (the rest is zero)
    float acc[16][4];
    mbar_wait(&bars[0], 0);
    lstm_encoder(acc, sX + lr * PL_XP + 2 * t, sWe + g * PL_XP + 2 * t, F);
    // relu(acc + b) as A fragments: C fragment of n-tile nt = columns 8nt + {2t, 2t+1} of rows {g, g+8} -> k slots {t, t+4}
    lstm_encoder_relu(acc, sBe, t);
    uint32_t eA[16][4];
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) lstm_a_frag(eA[nt], acc[nt][0], acc[nt][1], acc[nt][2], acc[nt][3]);

    // ---- gates chunk by chunk, cell update in registers, head product accumulated over the chunks
    float out[NC / 8][4];
#pragma unroll
    for (int q = 0; q < NC / 8; ++q) { out[q][0] = out[q][1] = out[q][2] = out[q][3] = 0.f; }
    const float* wlane = sWg + g * PL_GP + 2 * t;
#pragma unroll 1
    for (int ch = 0; ch < PL_CHUNKS; ++ch) {
        const int s = ch & 1;
        const int u0 = 8 * ch + 2 * t;             // this thread's units u0, u0 + 1
        const float2 ca = va ? *reinterpret_cast<const float2*>(c_a + u0) : make_float2(0.f, 0.f);
        const float2 cb = vb ? *reinterpret_cast<const float2*>(c_b + u0) : make_float2(0.f, 0.f);
        float gacc[4][4];
        mbar_wait(&bars[1 + s], (uint32_t)(ch >> 1) & 1u);
        lstm_gate_chunk(gacc, eA, hA, wlane + s * PL_CHUNK);
        __syncthreads();                           // every warp is done with stage s: refill it with chunk ch + 2
        if (tid == 0 && ch + 2 < PL_CHUNKS) {
            mbar_expect_tx(&bars[1 + s], PL_CHUNK_BYTES);
            tma_load_1d(sWg + s * PL_CHUNK, p.w_gates + (int64_t)(ch + 2) * PL_CHUNK, PL_CHUNK_BYTES, &bars[1 + s]);
        }
        // gacc[j][e]: gate j of (row g, u0), (row g, u0 + 1), (row g + 8, u0), (row g + 8, u0 + 1) for e = 0..3
        const float cp[4] = {ca.x, ca.y, cb.x, cb.y};
        float act[4][4], cn[4], hn[4];
        lstm_cell(gacc, sBg + 32 * ch + 2 * t, cp, act, cn, hn);
        if (va) {
            *reinterpret_cast<float2*>(c_a + u0) = make_float2(cn[0], cn[1]);
            *reinterpret_cast<float2*>(h_a + u0) = make_float2(hn[0], hn[1]);
        }
        if (vb) {
            *reinterpret_cast<float2*>(c_b + u0) = make_float2(cn[2], cn[3]);
            *reinterpret_cast<float2*>(h_b + u0) = make_float2(hn[2], hn[3]);
        }
        // heads: this chunk is k-step ch of h' W_cat^T
        lstm_head_chunk<NC>(out, hn, sWh, g, u0);
    }

    pb_sample_epilogue<NC>(out, sBh, p.sample, row0 + lr, offset);
}

// The H = 256 step (LSTMWrapper(Default(hidden_size=256), 256, 256)): the same function with the geometry of
// lstm_cell.cuh's PW_* block.  A CTA owns 64 rows, 4 warps x 16 rows (256 CTAs at N = 16384: 1.94 waves on 132 SMs).
//   * encoder: W_enc [256][136] (one 136 KB bulk copy) and the x tile [64][136] sit where the gate-weight ring and the h
//     tile go later; a warp's 16 x 256 accumulator becomes eA, the A fragments of k-steps 0..31 (128 registers).
//   * then the ring's first two stages are requested and each warp loads its 16 rows of h_prev into the h tile
//     [64][264] (TF32); k-steps 32..63 of every chunk read their A fragments from there (64-bit loads).
//   * gates: 32 chunks of 8 units from the packed [32][32][520] weights (2.1 MB per CTA per step from L2, 33 KB per
//     row) through a 2-stage ring of 65 KB bulk copies; cell update, state stores and heads as at H = 128.
template <int NC>
__global__ void __launch_bounds__(128, 1) k_policy_lstm_sample_256(LstmParams p) {
    extern __shared__ __align__(128) float smem[];
    float* sX = smem + SW_X;
    float* sWe = smem + SW_WE;
    float* sWg = smem + SW_WG;
    float* sHt = smem + SW_HT;
    float* sWh = smem + SW_WH;
    float* sBe = smem + SW_BE;
    float* sBg = smem + SW_BG;
    float* sBh = smem + SW_BH;
    __shared__ __align__(8) uint64_t bars[3];      // [0]: W_enc, [1 + s]: gate-weight ring stage s
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int64_t row0 = (int64_t)blockIdx.x * PW_ROWS;
    const int valid = (int)((p.sample.m - row0) < PW_ROWS ? (p.sample.m - row0) : PW_ROWS);
    const uint64_t offset = p.sample.counter ? *p.sample.counter : 0ull;

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1);
        mbar_fence_init();
        mbar_expect_tx(&bars[0], PW_WENC_BYTES);
        tma_load_1d(sWe, p.w_enc, PW_WENC_BYTES, &bars[0]);
    }
    const int F = p.in_features;
    for (int i = tid; i < PW_ROWS * PL_F; i += 128) {
        const int r = i >> 7, k = i & (PL_F - 1);
        sX[r * PL_XP + k] = (r < valid && k < F) ? p.obs[(row0 + r) * p.obs_stride + k] : 0.f;
    }
    for (int i = tid; i < PW_H; i += 128) sBe[i] = p.b_enc[i];
    for (int i = tid; i < 4 * PW_H; i += 128) sBg[i] = p.b_gates[i];
    for (int i = tid; i < NC * PW_H; i += 128) sWh[(i >> 8) * PW_HP + (i & (PW_H - 1))] = p.w_heads[i];
    if (tid < NC) sBh[tid] = p.b_heads[tid];
    __syncthreads();

    const int lr = 16 * warp + g;
    const bool va = lr < valid, vb = lr + 8 < valid;
    uint32_t eA[32][4];
    {
        float acc[32][4];
        mbar_wait(&bars[0], 0);
        lstm_encoder(acc, sX + lr * PL_XP + 2 * t, sWe + g * PL_XP + 2 * t, F);
        lstm_encoder_relu(acc, sBe, t);
#pragma unroll
        for (int nt = 0; nt < 32; ++nt) lstm_a_frag(eA[nt], acc[nt][0], acc[nt][1], acc[nt][2], acc[nt][3]);
    }
    fence_proxy_async_smem();                      // the x tile's generic writes before the ring's bulk copies
    __syncthreads();                               // W_enc and the x tile are consumed: ring and h tile from here
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            mbar_expect_tx(&bars[1 + s], PW_CHUNK_BYTES);
            tma_load_1d(sWg + s * PW_CHUNK, p.w_gates + (int64_t)s * PW_CHUNK, PW_CHUNK_BYTES, &bars[1 + s]);
        }
    }
    float* h_a = p.h + (row0 + lr) * p.h_stride;
    float* h_b = h_a + 8 * p.h_stride;
    float* c_a = p.c + (row0 + lr) * p.c_stride;
    float* c_b = c_a + 8 * p.c_stride;
    // h_prev of this warp's rows into the h tile before any of them is overwritten (only this warp reads them)
    lstm_load_h_tile(sHt, 16 * warp, lane, [&](int r) -> const float* {
        return 16 * warp + r < valid ? p.h + (row0 + 16 * warp + r) * p.h_stride : nullptr;
    });
    __syncwarp();

    float out[NC / 8][4];
#pragma unroll
    for (int q = 0; q < NC / 8; ++q) { out[q][0] = out[q][1] = out[q][2] = out[q][3] = 0.f; }
    const float* wlane = sWg + g * PW_GP + 2 * t;
    const float* hs = sHt + lr * PW_HP + 2 * t;
#pragma unroll 1
    for (int ch = 0; ch < PW_CHUNKS; ++ch) {
        const int s = ch & 1;
        const int u0 = 8 * ch + 2 * t;
        const float2 ca = va ? *reinterpret_cast<const float2*>(c_a + u0) : make_float2(0.f, 0.f);
        const float2 cb = vb ? *reinterpret_cast<const float2*>(c_b + u0) : make_float2(0.f, 0.f);
        float gacc[4][4];
        mbar_wait(&bars[1 + s], (uint32_t)(ch >> 1) & 1u);
        lstm_gate_chunk_256(gacc, eA, hs, wlane + s * PW_CHUNK);
        __syncthreads();                           // every warp is done with stage s: refill it with chunk ch + 2
        if (tid == 0 && ch + 2 < PW_CHUNKS) {
            mbar_expect_tx(&bars[1 + s], PW_CHUNK_BYTES);
            tma_load_1d(sWg + s * PW_CHUNK, p.w_gates + (int64_t)(ch + 2) * PW_CHUNK, PW_CHUNK_BYTES, &bars[1 + s]);
        }
        const float cp[4] = {ca.x, ca.y, cb.x, cb.y};
        float act[4][4], cn[4], hn[4];
        lstm_cell(gacc, sBg + 32 * ch + 2 * t, cp, act, cn, hn);
        if (va) {
            *reinterpret_cast<float2*>(c_a + u0) = make_float2(cn[0], cn[1]);
            *reinterpret_cast<float2*>(h_a + u0) = make_float2(hn[0], hn[1]);
        }
        if (vb) {
            *reinterpret_cast<float2*>(c_b + u0) = make_float2(cn[2], cn[3]);
            *reinterpret_cast<float2*>(h_b + u0) = make_float2(hn[2], hn[3]);
        }
        lstm_head_chunk<NC, PW_HP>(out, hn, sWh, g, u0);
    }
    pb_sample_epilogue<NC>(out, sBh, p.sample, row0 + lr, offset);
}

template <int NC>
int launch(const LstmParams& p, cudaStream_t stream) {
    PB_CUDA(cudaFuncSetAttribute(k_policy_lstm_sample<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PL_SMEM));
    k_policy_lstm_sample<NC><<<(unsigned)pb_ceil_div(p.sample.m, PL_ROWS), PL_THREADS, PL_SMEM, stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

template <int NC>
int launch_256(const LstmParams& p, cudaStream_t stream) {
    PB_CUDA(cudaFuncSetAttribute(k_policy_lstm_sample_256<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)PW_SMEM));
    k_policy_lstm_sample_256<NC><<<(unsigned)pb_ceil_div(p.sample.m, PW_ROWS), 128, PW_SMEM, stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

}  // namespace

extern "C" int pb_policy_lstm_sample(const float* obs, int64_t obs_stride, int32_t in_features, const float* w_enc,
                                     const float* b_enc, const float* w_gates, const float* b_gates, const float* w_heads,
                                     const float* b_heads, float* h, int64_t h_stride, float* c, int64_t c_stride,
                                     int64_t m, int32_t input_size, int32_t hidden_size, int32_t n_act, uint64_t seed,
                                     uint64_t* counter_dev, uint32_t* ticket_dev, int64_t* actions, float* logprobs,
                                     float* values, float* entropies, void* stream) {
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "pb_policy_lstm_sample: negative m");
    if (m == 0) return PB_OK;
    PB_REQUIRE(in_features >= 1 && in_features <= PL_F, PB_ERR_UNSUPPORTED,
               "pb_policy_lstm_sample: observation features must be in [1, %d] (got %d)", PL_F, in_features);
    PB_REQUIRE(input_size == hidden_size && (hidden_size == PL_H || hidden_size == PW_H), PB_ERR_UNSUPPORTED,
               "pb_policy_lstm_sample: built for LSTM input size = hidden size = %d or %d (got %d, %d)", PL_H, PW_H,
               input_size, hidden_size);
    PB_REQUIRE(n_act >= 1 && n_act <= 15, PB_ERR_UNSUPPORTED, "pb_policy_lstm_sample: n_act must be in [1, 15]");
    PB_REQUIRE(obs && w_enc && b_enc && w_gates && b_gates && w_heads && b_heads && h && c && actions && logprobs && values,
               PB_ERR_INVALID, "pb_policy_lstm_sample: null pointer");
    PB_REQUIRE(obs_stride >= in_features, PB_ERR_INVALID, "pb_policy_lstm_sample: obs_stride < in_features");
    PB_REQUIRE(((uintptr_t)w_enc & 15) == 0 && ((uintptr_t)w_gates & 15) == 0, PB_ERR_INVALID,
               "pb_policy_lstm_sample: w_enc / w_gates must be 16-byte aligned");
    PB_REQUIRE(((uintptr_t)h & 7) == 0 && ((uintptr_t)c & 7) == 0 && h_stride >= hidden_size &&
                   c_stride >= hidden_size && h_stride % 2 == 0 && c_stride % 2 == 0,
               PB_ERR_INVALID, "pb_policy_lstm_sample: h / c must be 8-byte aligned with even row strides >= %d",
               hidden_size);
    PB_REQUIRE(!ticket_dev || counter_dev, PB_ERR_INVALID, "pb_policy_lstm_sample: ticket_dev needs counter_dev");
    LstmParams p{obs, obs_stride, in_features, w_enc, b_enc, w_gates, b_gates, w_heads, b_heads, h, h_stride, c, c_stride,
                 {m, n_act, seed, counter_dev, ticket_dev, actions, logprobs, values, entropies}};
    if (hidden_size == PW_H)
        return n_act + 1 <= 8 ? launch_256<8>(p, (cudaStream_t)stream) : launch_256<16>(p, (cudaStream_t)stream);
    return n_act + 1 <= 8 ? launch<8>(p, (cudaStream_t)stream) : launch<16>(p, (cudaStream_t)stream);
}
