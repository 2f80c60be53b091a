// lstm_cell.cuh -- the LSTMWrapper(models.Default) cell pieces shared by the rollout step (policy_lstm.cu,
// pb_policy_lstm_sample) and the training forward (lstm_bptt.cu, pb_lstm_bptt_forward), so that both compute the same
// function bit for bit:
//   * the packed-operand geometry (models.LSTMWrapper.fused_operands builds the packs);
//   * the encoder product of one warp's 16 rows from a staged x tile and the resident W_enc (mma.sync TF32);
//   * relu(acc + b_enc) as the A fragments of the gate product (k-slot trick: k slots (t, t+4) of k-step ks are the
//     adjacent columns 8ks + 2t, 8ks + 2t + 1 for both operands);
//   * one chunk of 8 hidden units of the gate product ([e | h_prev] x 32 gate columns i(8) | f(8) | g(8) | o(8));
//   * the cell update of a thread's 2 rows x 2 units, and the head product accumulated chunk by chunk.
// Fragment element order of a chunk, e = 0..3: (row g, unit u0), (row g, u0 + 1), (row g + 8, u0), (row g + 8, u0 + 1)
// with u0 = 8 ch + 2t -- the C fragment of n-tile j of the chunk is gate j of those four (row, unit) pairs.
// Two sizes H = input size = hidden size: 128 (PL_*) and 256 (PW_*, the geometry of the H = 256 kernels below).
#pragma once
#include "policy_sample.cuh"

constexpr int PL_F = 128;                          // x tile columns (obs features, zero padded)
constexpr int PL_H = 128;                          // LSTM input size = hidden size
constexpr int PL_XP = PL_F + 8;                    // 136: x / W_enc / W_heads pitch (conflict-free 64-bit loads)
constexpr int PL_GP = 2 * PL_H + 8;                // 264: gate-weight row pitch, K = [e (128) | h (128)] + pad
constexpr int PL_CHUNKS = PL_H / 8;                // 16 chunks of 8 units = 32 gate columns
constexpr int PL_CHUNK = 32 * PL_GP;               // floats per chunk (33792 B)
constexpr uint32_t PL_CHUNK_BYTES = PL_CHUNK * 4u;
constexpr uint32_t PL_WENC_BYTES = PL_H * PL_XP * 4u;

__device__ __forceinline__ float pb_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// H = 256: one CTA owns 64 rows (4 warps x 16).  e stays in registers as the A fragments of k-steps 0..31 (128
// registers, as [e | h] at H = 128); h_prev is read as A fragments from the h tile [64][264] (TF32, 64-bit loads of the
// k-slot trick, conflict-free at pitch 264).  Shared memory, in floats: the ring and the h tile, which first hold W_enc
// and the x tile for the encoder, then the heads and the biases (PW_SMEM = 222 784 B).
constexpr int PW_H = 256;
constexpr int PW_ROWS = 64;                        // rows (segments) per CTA
constexpr int PW_HP = PW_H + 8;                    // 264: h tile / W_heads pitch
constexpr int PW_GP = 2 * PW_H + 8;                // 520: gate-weight row pitch, K = [e (256) | h (256)] + pad
constexpr int PW_CHUNKS = PW_H / 8;                // 32 chunks of 8 units
constexpr int PW_CHUNK = 32 * PW_GP;               // floats per chunk (66560 B)
constexpr uint32_t PW_CHUNK_BYTES = PW_CHUNK * 4u;
constexpr uint32_t PW_WENC_BYTES = PW_H * PL_XP * 4u;
constexpr int SW_WG = 0;                           // [2][32][520] gate-weight ring
constexpr int SW_HT = SW_WG + 2 * PW_CHUNK;        // [64][264] h_prev tile, TF32
constexpr int SW_WE = 0;                           // [256][136] W_enc (encoder phase, over the ring)
constexpr int SW_X = SW_WE + PW_H * PL_XP;         // [64][136] x tile (encoder phase, over the h tile)
constexpr int SW_WH = SW_HT + PW_ROWS * PW_HP;     // [16][264] head matrix
constexpr int SW_BE = SW_WH + 16 * PW_HP;          // [256] b_enc
constexpr int SW_BG = SW_BE + PW_H;                // [32][32] b_ih + b_hh, chunk order
constexpr int SW_BH = SW_BG + 4 * PW_H;            // [16] head bias
constexpr size_t PW_SMEM = (size_t)(SW_BH + 16) * sizeof(float);
static_assert(SW_X + PW_ROWS * PL_XP <= SW_WH, "W_enc and the x tile must fit in the ring and h tile");
static_assert(PW_SMEM <= 227 * 1024, "shared memory over the sm_90 per-CTA limit");
static_assert((SW_HT * 4) % 16 == 0 && (SW_X * 4) % 16 == 0 && PW_CHUNK_BYTES % 16 == 0, "bulk copy alignment");

// acc[nt] += x[16 rows][F] W_enc^T for n-tile nt (hidden units 8nt..8nt+7), NT = H / 8.  xa = sX + lr * PL_XP + 2t,
// wb = sWe + g * PL_XP + 2t; K = F rounded up to 8 (the tile is zero past F).
template <int NT>
__device__ __forceinline__ void lstm_encoder(float (&acc)[NT][4], const float* xa, const float* wb, int F) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
    const int ksteps = (F + 7) >> 3;
#pragma unroll 2
    for (int ks = 0; ks < ksteps; ++ks) {
        const float2 x0 = *reinterpret_cast<const float2*>(xa + 8 * ks);
        const float2 x1 = *reinterpret_cast<const float2*>(xa + 8 * PL_XP + 8 * ks);
        const uint32_t a[4] = {to_tf32(x0.x), to_tf32(x1.x), to_tf32(x0.y), to_tf32(x1.y)};
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const float2 w = *reinterpret_cast<const float2*>(wb + 8 * nt * PL_XP + 8 * ks);   // B[k][n] = W[n][k]
            mma_tf32(acc[nt], a, __float_as_uint(w.x), __float_as_uint(w.y));
        }
    }
}

// relu(acc + b) in place: C fragment of n-tile nt = columns 8nt + {2t, 2t+1} of rows {g, g+8}
template <int NT>
__device__ __forceinline__ void lstm_encoder_relu(float (&acc)[NT][4], const float* sBe, int t) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const int c0 = 8 * nt + 2 * t;
        const float b0 = sBe[c0], b1 = sBe[c0 + 1];
        acc[nt][0] = fmaxf(acc[nt][0] + b0, 0.f);
        acc[nt][1] = fmaxf(acc[nt][1] + b1, 0.f);
        acc[nt][2] = fmaxf(acc[nt][2] + b0, 0.f);
        acc[nt][3] = fmaxf(acc[nt][3] + b1, 0.f);
    }
}

// A fragment of k-step ks from the four values (row g, col 8ks+2t), (g, +1), (g+8, 8ks+2t), (g+8, +1) in element order
__device__ __forceinline__ void lstm_a_frag(uint32_t (&a)[4], float v0, float v1, float v2, float v3) {
    a[0] = to_tf32(v0); a[1] = to_tf32(v2); a[2] = to_tf32(v1); a[3] = to_tf32(v3);
}

// gacc[j] = [e | h_prev] (this warp's 16 rows) x gate j of the chunk; wc = this lane's view of the chunk
// (stage base + g * PL_GP + 2t)
__device__ __forceinline__ void lstm_gate_chunk(float (&gacc)[4][4], const uint32_t (&eA)[16][4],
                                                const uint32_t (&hA)[16][4], const float* wc) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { gacc[j][0] = gacc[j][1] = gacc[j][2] = gacc[j][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 32; ++ks) {
        const uint32_t(&a)[4] = ks < 16 ? eA[ks] : hA[ks - 16];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 w = *reinterpret_cast<const float2*>(wc + 8 * j * PL_GP + 8 * ks);
            mma_tf32(gacc[j], a, __float_as_uint(w.x), __float_as_uint(w.y));
        }
    }
}

// the H = 256 chunk: gacc[j] = [e | h_prev] x gate j, e (k-steps 0..31) from registers, h_prev (k-steps 32..63) from
// this warp's rows of the TF32 h tile.  hs = tile + lr * PW_HP + 2t, wc = stage base + g * PW_GP + 2t
__device__ __forceinline__ void lstm_gate_chunk_256(float (&gacc)[4][4], const uint32_t (&eA)[32][4], const float* hs,
                                                    const float* wc) {
#pragma unroll
    for (int j = 0; j < 4; ++j) { gacc[j][0] = gacc[j][1] = gacc[j][2] = gacc[j][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 32; ++ks) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 w = *reinterpret_cast<const float2*>(wc + 8 * j * PW_GP + 8 * ks);
            mma_tf32(gacc[j], eA[ks], __float_as_uint(w.x), __float_as_uint(w.y));
        }
    }
#pragma unroll
    for (int ks = 0; ks < 32; ++ks) {
        const float2 x0 = *reinterpret_cast<const float2*>(hs + 8 * ks);
        const float2 x1 = *reinterpret_cast<const float2*>(hs + 8 * PW_HP + 8 * ks);
        const uint32_t a[4] = {__float_as_uint(x0.x), __float_as_uint(x1.x), __float_as_uint(x0.y), __float_as_uint(x1.y)};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 w = *reinterpret_cast<const float2*>(wc + 8 * j * PW_GP + 8 * (32 + ks));
            mma_tf32(gacc[j], a, __float_as_uint(w.x), __float_as_uint(w.y));
        }
    }
}

// this warp's 16 rows of the H = 256 h tile from rows src(r) (fp32, 256 floats each; null = zeros), rounded to TF32
// (cvt.rna) on the way in.  rows: this warp's first tile row; src(r) for r = 0..15.
template <typename Src>
__device__ __forceinline__ void lstm_load_h_tile(float* sHt, int rows, int lane, Src src) {
#pragma unroll 4
    for (int i = lane; i < 16 * (PW_H / 2); i += 32) {
        const int r = i / (PW_H / 2), k = 2 * (i % (PW_H / 2));
        const float* p = src(r);
        const float2 v = p ? *reinterpret_cast<const float2*>(p + k) : make_float2(0.f, 0.f);
        *reinterpret_cast<float2*>(sHt + (rows + r) * PW_HP + k) =
            make_float2(__uint_as_float(to_tf32(v.x)), __uint_as_float(to_tf32(v.y)));
    }
}

// the cell update of the four (row, unit) elements: bg = sBg + 32 ch + 2t (b_ih + b_hh in chunk order), cp = c_prev;
// act[j][e] = sigmoid(i), sigmoid(f), tanh(g), sigmoid(o)
__device__ __forceinline__ void lstm_cell(const float (&gacc)[4][4], const float* bg, const float (&cp)[4],
                                          float (&act)[4][4], float (&cn)[4], float (&hn)[4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int q = e & 1;
        const float zi = gacc[0][e] + bg[q], zf = gacc[1][e] + bg[8 + q];
        const float zg = gacc[2][e] + bg[16 + q], zo = gacc[3][e] + bg[24 + q];
        act[0][e] = pb_sigmoid(zi);
        act[1][e] = pb_sigmoid(zf);
        act[2][e] = tanhf(zg);
        act[3][e] = pb_sigmoid(zo);
        cn[e] = act[1][e] * cp[e] + act[0][e] * act[2][e];
        hn[e] = act[3][e] * tanhf(cn[e]);
    }
}

// heads: chunk ch is k-step ch of h' W_cat^T (slots t <-> unit u0, t + 4 <-> unit u0 + 1); sWh pitch P
template <int NC, int P = PL_XP>
__device__ __forceinline__ void lstm_head_chunk(float (&out)[NC / 8][4], const float (&hn)[4], const float* sWh, int g,
                                                int u0) {
    uint32_t a[4];
    lstm_a_frag(a, hn[0], hn[1], hn[2], hn[3]);
#pragma unroll
    for (int q = 0; q < NC / 8; ++q) {
        const float* wh = sWh + (8 * q + g) * P + u0;
        mma_tf32(out[q], a, to_tf32(wh[0]), to_tf32(wh[1]));
    }
}
