// lstm_bptt.cu -- the training-time forward and backward of LSTMWrapper(models.Default) over a minibatch of bptt segments
// (B segments x T steps), for the fused recurrent update (models._LSTMBPTTFunction).
//
// Replaces, inside train() (reference clean_pufferl.py:186-238 with the [rows, bptt, *obs] segments of :188-191), the
// encoder GEMM, cuDNN's LSTM forward and backward over the segment and the head GEMM.  Rows are in (b, t) order
// (row b*T + t), as experience.b_obs[mb] is laid out.
//
// pb_lstm_bptt_forward, per segment b and step t (the formula of pb_policy_lstm_sample, with the same shared pieces:
// lstm_cell.cuh):
//   e = relu(x W_enc^T + b_enc);  z = e W_ih^T + h W_hh^T + (b_ih + b_hh);  c' = sigmoid(f) c + sigmoid(i) tanh(g);
//   h' = sigmoid(o) tanh(c');  out = h' W_cat^T + b_cat  (packed [B*T][R] rows, R = 8 or 16: logits | value | zero pad)
// A CTA owns 128 segments (8 warps x 16 rows).  Phase 1 runs the encoder for all T steps (x tile staged by coalesced
// loads, W_enc resident, as in policy_lstm.cu) and writes e to the saved-activation rows.  Phase 2 walks the T steps:
// the region of the x tile and W_enc now holds c and h of the 128 segments in the threads' own fragment layout
// ([chunk][warp][lane] float4, 64 KB each), so the state never leaves the SM between steps; e comes back from the saved
// row the same thread wrote; the gate weights stream from L2 through the 2-stage ring of policy_lstm.cu, continuing
// across steps.  Each chunk's cell update writes h_prev, the four gate activations, c and h to the saved row.
//
// pb_lstm_bptt_backward walks the same tiles in reverse time, dh and dc carried on chip (shared memory, own fragments):
//   dh_t += W_cat^T dOut_t                                           (fp32 FFMA, R <= 16 terms)
//   dc_t += dh_t sigmoid(o) (1 - tanh^2 c_t)
//   dz    = [dc tanh g s'(i), dc c_{t-1} s'(f), dc sigmoid(i) (1 - tanh^2 g), dh tanh c_t s'(o)]   -> HBM [B*T][512]
//   [de | dh_{t-1}] = dz [W_ih | W_hh]                               (mma.sync TF32, fp32 accumulators in registers)
//   dc_{t-1} = dc_t sigmoid(f);  dPre_enc = de * (e > 0)             -> HBM [B*T][128]
// The product reads a transposed packing of the gate weights (models.LSTMWrapper.gate_weights_transposed): per chunk of
// 8 units, [256 output columns][40] with column 8j + u = gate j of unit 8ch + u, so that the four dz values of a thread's
// (row, unit) pairs are directly the A fragments of four k-steps (the k-slot trick) and the B fragments are conflict-free
// 64-bit loads (pitch 40).  The weight gradients are library GEMMs on dz, dPre and the saved rows (models.py).
//
// Row addresses.  Segment b = (e, g) = (b / G, b % G) reads x(b, t) = obs + e s_e + g s_g + t s_t and writes dPre row
// (b, t) at dpre + e d_e + g d_g + t d_t; every other buffer stays dense in row b*T + t.  pb_lstm_bptt_forward / _backward
// are the gathered case (G = 1: a contiguous [B, T, F] copy, dPre row b*T + t); the _rows entry points also take the
// segment view of Experience.segment_obs, which reads minibatch mb of the reference in place from the arrival-order
// rollout buffer and writes dPre in the order of its G observation slabs (layouts in include/pufferlib_b200.h).  The
// forward computes its CTA's 128 x-row bases once (pad columns of the x tile); the backward its two dPre row bases once
// per thread.  Nothing else changes: the same values reach the same fragment slots, so both layouts give bitwise the
// same out, state, saved rows, dz and (permuted) dPre.
//
// Saved-activation row (1024 floats = 4096 B per (b, t) row): [e (128) | h_prev (128) | sigmoid(i) | sigmoid(f) |
// tanh(g) | sigmoid(o) (4 x 128, unit-major) | c_t (128) | h_t (128)]; [e | h_prev] is the operand of dW_ih | dW_hh,
// h_t that of dW_cat.  At B*T = 524 288 rows (breakout's minibatch) that is 2.1 GB.
//
// LSTM size 256: k_lstm_bptt_fwd_256 / k_lstm_bptt_bwd_256 below (64 segments per CTA; their own layout notes).
//
// Tile choice.  128 segments per CTA, one CTA per SM (shared memory): every CTA streams the 528 KB of gate weights per
// step from L2, so fewer, fuller CTAs stream less.  At the headline shape B = 32 768 that is 256 CTAs = 1.94 waves on
// 132 SMs, both waves nearly full (124 CTAs in the second); 64-segment CTAs would give 512 CTAs = 3.88 waves and twice
// the weight traffic per row.
//
// Operand rounding is that of pb_policy_lstm_sample (every tensor-core operand rounded to nearest TF32, cvt.rna;
// accumulation, biases and the cell fp32), so the forward at T = 1 computes what the rollout step computes.  In the
// backward, dz (and the packed weights, on the host) are rounded to TF32 for the product; everything else is fp32.
//
// Resources (nvcc 12.9 -Xptxas -v, sm_90a): forward 218 176 B shared memory, 211 / 216 registers (8 / 16 head
// columns); backward 221 184 B shared memory, 232 registers; no spills.  Time (bench_lstm.py, H100 80GB HBM3,
// 700 W power limit): forward + loss + backward of a 524 288-row minibatch 7.53 ms, vs 35.65 ms on cuDNN autograd.
#include "lstm_cell.cuh"
#include "pb_common.cuh"
#include "policy_sample.cuh"
#include "tma.cuh"

namespace {

constexpr int BT_ROWS = 128;                       // segments per CTA
constexpr int BT_THREADS = 256;                    // 8 warps x 16 segments
constexpr int SV = 1024;                           // floats per saved row
constexpr int SV_E = 0, SV_HP = 128, SV_ACT = 256, SV_C = 768, SV_H = 896;
constexpr int FRAG = PL_CHUNKS * 8 * 32 * 4;       // floats of one per-thread fragment array [chunk][warp][lane][4]

// forward shared memory, in floats: phase 1 [x tile | W_enc] and phase 2 [c | h] share the first region
constexpr int SF_X = 0;                            // [128][136] x tile (phase 1)
constexpr int SF_WE = SF_X + BT_ROWS * PL_XP;      // [128][136] W_enc (phase 1)
constexpr int SF_C = 0;                            // c fragments (phase 2)
constexpr int SF_H = SF_C + FRAG;                  // h fragments (phase 2)
constexpr int SF_WG = SF_WE + PL_H * PL_XP;        // [2][32][264] gate-weight ring
constexpr int SF_WH = SF_WG + 2 * PL_CHUNK;        // [16][136] head matrix
constexpr int SF_BE = SF_WH + 16 * PL_XP;          // [128] b_enc
constexpr int SF_BG = SF_BE + PL_H;                // [16][32] b_ih + b_hh, chunk order
constexpr int SF_BH = SF_BG + 4 * PL_H;            // [16] head bias
constexpr size_t FWD_SMEM = (size_t)(SF_BH + 16) * sizeof(float);
static_assert(SF_H + FRAG <= SF_WG, "c | h must fit in the phase-1 region");
static_assert(FWD_SMEM <= 227 * 1024, "shared memory over the sm_90 per-CTA limit");
static_assert((SF_WE * 4) % 16 == 0 && (SF_WG * 4) % 16 == 0, "bulk copy alignment");

// backward: transposed gate weights, [2 stages][256][40] ring, dh and dc fragments, head matrix [16][128]
constexpr int BW_P = 40;
constexpr int BW_CHUNK = 2 * PL_H * BW_P;          // floats per chunk (40960 B)
constexpr uint32_t BW_CHUNK_BYTES = BW_CHUNK * 4u;
constexpr int SB_WT = 0;
constexpr int SB_DH = SB_WT + 2 * BW_CHUNK;
constexpr int SB_DC = SB_DH + FRAG;
constexpr int SB_WH = SB_DC + FRAG;
constexpr size_t BWD_SMEM = (size_t)(SB_WH + 16 * PL_H) * sizeof(float);
static_assert(BWD_SMEM <= 227 * 1024, "shared memory over the sm_90 per-CTA limit");
static_assert(BW_CHUNK_BYTES % 16 == 0, "bulk copy alignment");

struct FwdParams {
    const float* obs; int64_t s_e, s_g, s_t; int groups; int in_features;   // x(b, t) = obs + (b/G) s_e + (b%G) s_g + t s_t
    int64_t batch; int steps;
    const float* h0; const float* c0;              // [B][128] or null (zeros)
    const float* w_enc; const float* b_enc;        // [128][136] TF32, [128]
    const float* w_gates; const float* b_gates;    // [16][32][264] TF32, [16][32]
    const float* w_heads; const float* b_heads;    // [NC][128], [NC]
    float* out; float* h_out; float* c_out; float* saved;
};

struct BwdParams {
    const float* dout; const float* saved; const float* c0;
    const float* w_gates_t; const float* w_heads;  // [16][256][40] TF32, [NC][128]
    int64_t batch; int steps; int n_act;
    float* dz; float* dpre;
    int groups; int64_t d_e, d_g, d_t;             // dPre row (b, t) at dpre + (b/G) d_e + (b%G) d_g + t d_t
};

// this thread's slot of a [chunk][warp][lane] float4 fragment array
__device__ __forceinline__ float4* frag(float* base, int ch, int warp, int lane) {
    return reinterpret_cast<float4*>(base) + (ch * 8 + warp) * 32 + lane;
}
__device__ __forceinline__ float2 ld2(const float* p, bool ok) {
    return ok ? *reinterpret_cast<const float2*>(p) : make_float2(0.f, 0.f);
}
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
// x-row base of local segment r (floats from obs), kept in the pad columns 128..129 of the x tile's row r: the tile load
// writes and lstm_encoder reads columns < 128 only, so the 128 bases are computed once and cost no shared memory
__device__ __forceinline__ int64_t* xrow(float* sX, int r) { return reinterpret_cast<int64_t*>(sX + r * PL_XP + PL_F); }

template <int NC>
__global__ void __launch_bounds__(BT_THREADS, 1) k_lstm_bptt_fwd(FwdParams p) {
    extern __shared__ __align__(128) float smem[];
    float* sX = smem + SF_X;
    float* sWe = smem + SF_WE;
    float* sC = smem + SF_C;
    float* sH = smem + SF_H;
    float* sWg = smem + SF_WG;
    float* sWh = smem + SF_WH;
    float* sBe = smem + SF_BE;
    float* sBg = smem + SF_BG;
    float* sBh = smem + SF_BH;
    __shared__ __align__(8) uint64_t bars[3];      // [0]: W_enc, [1 + s]: gate-weight ring stage s
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int T = p.steps, F = p.in_features;
    const int64_t b0 = (int64_t)blockIdx.x * BT_ROWS;
    const int valid = (int)((p.batch - b0) < BT_ROWS ? (p.batch - b0) : BT_ROWS);
    const int items = T * PL_CHUNKS;               // gate chunks streamed by this CTA, in (t, chunk) order

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1);
        mbar_fence_init();
        mbar_expect_tx(&bars[0], PL_WENC_BYTES);
        tma_load_1d(sWe, p.w_enc, PL_WENC_BYTES, &bars[0]);
#pragma unroll
        for (int s = 0; s < 2; ++s) {              // items >= 16 > 2: the first two chunks are always needed
            mbar_expect_tx(&bars[1 + s], PL_CHUNK_BYTES);
            tma_load_1d(sWg + s * PL_CHUNK, p.w_gates + (int64_t)s * PL_CHUNK, PL_CHUNK_BYTES, &bars[1 + s]);
        }
    }
    if (tid < PL_H) sBe[tid] = p.b_enc[tid];
    for (int i = tid; i < 4 * PL_H; i += BT_THREADS) sBg[i] = p.b_gates[i];
    for (int i = tid; i < NC * PL_H; i += BT_THREADS) sWh[(i >> 7) * PL_XP + (i & (PL_H - 1))] = p.w_heads[i];
    if (tid < NC) sBh[tid] = p.b_heads[tid];
    if (tid < BT_ROWS) {                           // visible after the first barrier of phase 1
        const int64_t b = b0 + tid;
        *xrow(sX, tid) = (b / p.groups) * p.s_e + (b % p.groups) * p.s_g;
    }

    const int lr = 16 * warp + g;                  // local segments lr (fragment rows g) and lr + 8 (g + 8)
    const bool va = lr < valid, vb = lr + 8 < valid;
    const int64_t ra0 = (b0 + lr) * T, rb0 = ra0 + 8 * (int64_t)T;   // rows (b, 0) of the two segments

    // ---- phase 1: e = relu(x W_enc^T + b_enc) for every step, to the saved rows
#pragma unroll 1
    for (int st = 0; st < T; ++st) {
        __syncthreads();                           // the previous step's tile is consumed
        for (int i = tid; i < BT_ROWS * PL_F; i += BT_THREADS) {
            const int r = i >> 7, k = i & (PL_F - 1);
            sX[r * PL_XP + k] = (r < valid && k < F) ? p.obs[*xrow(sX, r) + st * p.s_t + k] : 0.f;
        }
        __syncthreads();
        if (st == 0) mbar_wait(&bars[0], 0);
        float acc[16][4];
        lstm_encoder(acc, sX + lr * PL_XP + 2 * t, sWe + g * PL_XP + 2 * t, F);
        lstm_encoder_relu(acc, sBe, t);
        float* sa = p.saved + (ra0 + st) * SV + SV_E + 2 * t;
        float* sb = p.saved + (rb0 + st) * SV + SV_E + 2 * t;
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) {
            if (va) st2(sa + 8 * nt, acc[nt][0], acc[nt][1]);
            if (vb) st2(sb + 8 * nt, acc[nt][2], acc[nt][3]);
        }
    }
    __syncthreads();                               // x tile and W_enc are dead: the region becomes c | h

    // ---- phase 2: the recurrence.  c, h of this thread's (row, unit) pairs in its own fragment slots
#pragma unroll
    for (int ch = 0; ch < PL_CHUNKS; ++ch) {
        const int u0 = 8 * ch + 2 * t;
        const float2 ha = ld2(p.h0 + (b0 + lr) * PL_H + u0, va && p.h0), hb = ld2(p.h0 + (b0 + lr + 8) * PL_H + u0, vb && p.h0);
        const float2 ca = ld2(p.c0 + (b0 + lr) * PL_H + u0, va && p.c0), cb = ld2(p.c0 + (b0 + lr + 8) * PL_H + u0, vb && p.c0);
        *frag(sH, ch, warp, lane) = make_float4(ha.x, ha.y, hb.x, hb.y);
        *frag(sC, ch, warp, lane) = make_float4(ca.x, ca.y, cb.x, cb.y);
    }
    const float* wlane = sWg + g * PL_GP + 2 * t;
    int it = 0;
#pragma unroll 1
    for (int st = 0; st < T; ++st) {
        const int64_t ra = ra0 + st, rb = rb0 + st;
        float* sa = p.saved + ra * SV;
        float* sb = p.saved + rb * SV;
        uint32_t eA[16][4], hA[16][4];
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const float2 e0 = ld2(sa + SV_E + 8 * k + 2 * t, va), e1 = ld2(sb + SV_E + 8 * k + 2 * t, vb);
            lstm_a_frag(eA[k], e0.x, e0.y, e1.x, e1.y);
            const float4 hv = *frag(sH, k, warp, lane);
            lstm_a_frag(hA[k], hv.x, hv.y, hv.z, hv.w);
        }
        float out[NC / 8][4];
#pragma unroll
        for (int q = 0; q < NC / 8; ++q) { out[q][0] = out[q][1] = out[q][2] = out[q][3] = 0.f; }
#pragma unroll 1
        for (int ch = 0; ch < PL_CHUNKS; ++ch, ++it) {
            const int s = it & 1;
            const int u0 = 8 * ch + 2 * t;
            float gacc[4][4];
            mbar_wait(&bars[1 + s], (uint32_t)(it >> 1) & 1u);
            lstm_gate_chunk(gacc, eA, hA, wlane + s * PL_CHUNK);
            __syncthreads();                       // every warp is done with stage s: refill it with item it + 2
            if (tid == 0 && it + 2 < items) {
                mbar_expect_tx(&bars[1 + s], PL_CHUNK_BYTES);
                tma_load_1d(sWg + s * PL_CHUNK, p.w_gates + (int64_t)((it + 2) % PL_CHUNKS) * PL_CHUNK, PL_CHUNK_BYTES,
                            &bars[1 + s]);
            }
            const float4 cv = *frag(sC, ch, warp, lane), hv = *frag(sH, ch, warp, lane);
            const float cp[4] = {cv.x, cv.y, cv.z, cv.w};
            float act[4][4], cn[4], hn[4];
            lstm_cell(gacc, sBg + 32 * ch + 2 * t, cp, act, cn, hn);
            *frag(sC, ch, warp, lane) = make_float4(cn[0], cn[1], cn[2], cn[3]);
            *frag(sH, ch, warp, lane) = make_float4(hn[0], hn[1], hn[2], hn[3]);
            if (va) {
                st2(sa + SV_HP + u0, hv.x, hv.y);
#pragma unroll
                for (int j = 0; j < 4; ++j) st2(sa + SV_ACT + 128 * j + u0, act[j][0], act[j][1]);
                st2(sa + SV_C + u0, cn[0], cn[1]);
                st2(sa + SV_H + u0, hn[0], hn[1]);
            }
            if (vb) {
                st2(sb + SV_HP + u0, hv.z, hv.w);
#pragma unroll
                for (int j = 0; j < 4; ++j) st2(sb + SV_ACT + 128 * j + u0, act[j][2], act[j][3]);
                st2(sb + SV_C + u0, cn[2], cn[3]);
                st2(sb + SV_H + u0, hn[2], hn[3]);
            }
            if (st == T - 1) {
                if (va) {
                    st2(p.h_out + (b0 + lr) * PL_H + u0, hn[0], hn[1]);
                    st2(p.c_out + (b0 + lr) * PL_H + u0, cn[0], cn[1]);
                }
                if (vb) {
                    st2(p.h_out + (b0 + lr + 8) * PL_H + u0, hn[2], hn[3]);
                    st2(p.c_out + (b0 + lr + 8) * PL_H + u0, cn[2], cn[3]);
                }
            }
            lstm_head_chunk<NC>(out, hn, sWh, g, u0);
        }
        // out[q]: (row g, cols 8q + 2t, +1), (row g + 8, same)
#pragma unroll
        for (int q = 0; q < NC / 8; ++q) {
            const int k = 8 * q + 2 * t;
            if (va) st2(p.out + ra * NC + k, out[q][0] + sBh[k], out[q][1] + sBh[k + 1]);
            if (vb) st2(p.out + rb * NC + k, out[q][2] + sBh[k], out[q][3] + sBh[k + 1]);
        }
    }
}

template <int NC>
__global__ void __launch_bounds__(BT_THREADS, 1) k_lstm_bptt_bwd(BwdParams p) {
    extern __shared__ __align__(128) float smem[];
    float* sWt = smem + SB_WT;
    float* sDH = smem + SB_DH;
    float* sDC = smem + SB_DC;
    float* sWh = smem + SB_WH;
    __shared__ __align__(8) uint64_t bars[2];      // ring stage s
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int T = p.steps;
    const int64_t b0 = (int64_t)blockIdx.x * BT_ROWS;
    const int valid = (int)((p.batch - b0) < BT_ROWS ? (p.batch - b0) : BT_ROWS);
    const int items = T * PL_CHUNKS;

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_fence_init();
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            mbar_expect_tx(&bars[s], BW_CHUNK_BYTES);
            tma_load_1d(sWt + s * BW_CHUNK, p.w_gates_t + (int64_t)s * BW_CHUNK, BW_CHUNK_BYTES, &bars[s]);
        }
    }
    for (int i = tid; i < NC * PL_H; i += BT_THREADS) sWh[i] = p.w_heads[i];
#pragma unroll
    for (int ch = 0; ch < PL_CHUNKS; ++ch) *frag(sDC, ch, warp, lane) = make_float4(0.f, 0.f, 0.f, 0.f);   // dc_T = 0
    __syncthreads();                               // head matrix and barrier inits are visible

    const int lr = 16 * warp + g;
    const bool va = lr < valid, vb = lr + 8 < valid;
    const int64_t ra0 = (b0 + lr) * T, rb0 = ra0 + 8 * (int64_t)T;
    const int64_t ba = b0 + lr, bb = ba + 8;       // dPre rows (b, 0) of the two segments
    float* const dpa = p.dpre + (ba / p.groups) * p.d_e + (ba % p.groups) * p.d_g;
    float* const dpb = p.dpre + (bb / p.groups) * p.d_e + (bb % p.groups) * p.d_g;
    const float* wlane = sWt + g * BW_P + 2 * t;
    // acc[0..15]: de (n-tile nt = encoder units 8nt..), acc[16 + ch]: dh_{t-1} of chunk ch, both in chunk element order
    float acc[32][4];
#pragma unroll
    for (int nt = 0; nt < 32; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }   // dh_T = 0
    int it = 0;
#pragma unroll 1
    for (int st = T - 1; st >= 0; --st) {
        const int64_t ra = ra0 + st, rb = rb0 + st;
        const float* sa = p.saved + ra * SV;
        const float* sb = p.saved + rb * SV;
        // ---- dh_t = (recurrent part) + W_cat^T dOut_t, to this thread's dh slots
        {
            float da[NC], db[NC];
#pragma unroll
            for (int k = 0; k < NC; k += 2) {
                const float2 x0 = ld2(p.dout + ra * NC + k, va), x1 = ld2(p.dout + rb * NC + k, vb);
                da[k] = x0.x; da[k + 1] = x0.y; db[k] = x1.x; db[k + 1] = x1.y;
            }
#pragma unroll
            for (int ch = 0; ch < PL_CHUNKS; ++ch) {
                float d[4] = {acc[16 + ch][0], acc[16 + ch][1], acc[16 + ch][2], acc[16 + ch][3]};
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    if (k <= p.n_act) {
                        const float2 w = *reinterpret_cast<const float2*>(sWh + k * PL_H + 8 * ch + 2 * t);
                        d[0] += da[k] * w.x; d[1] += da[k] * w.y; d[2] += db[k] * w.x; d[3] += db[k] * w.y;
                    }
                }
                *frag(sDH, ch, warp, lane) = make_float4(d[0], d[1], d[2], d[3]);
            }
        }
#pragma unroll
        for (int nt = 0; nt < 32; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
        // c_{t-1}: the previous row of the segment, or c0 (zeros when null) at t = 0
        const float* cpa = st > 0 ? sa - SV + SV_C : (p.c0 ? p.c0 + (b0 + lr) * PL_H : nullptr);
        const float* cpb = st > 0 ? sb - SV + SV_C : (p.c0 ? p.c0 + (b0 + lr + 8) * PL_H : nullptr);
#pragma unroll 1
        for (int ch = 0; ch < PL_CHUNKS; ++ch, ++it) {
            const int s = it & 1;
            const int u0 = 8 * ch + 2 * t;
            const float4 dhv = *frag(sDH, ch, warp, lane), dcv = *frag(sDC, ch, warp, lane);
            const float dh[4] = {dhv.x, dhv.y, dhv.z, dhv.w}, dc0[4] = {dcv.x, dcv.y, dcv.z, dcv.w};
            float act[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 x0 = ld2(sa + SV_ACT + 128 * j + u0, va), x1 = ld2(sb + SV_ACT + 128 * j + u0, vb);
                act[j][0] = x0.x; act[j][1] = x0.y; act[j][2] = x1.x; act[j][3] = x1.y;
            }
            const float2 c0a = ld2(sa + SV_C + u0, va), c0b = ld2(sb + SV_C + u0, vb);
            const float2 c1a = ld2(cpa + u0, va && cpa), c1b = ld2(cpb + u0, vb && cpb);
            const float ct[4] = {c0a.x, c0a.y, c0b.x, c0b.y}, cprev[4] = {c1a.x, c1a.y, c1b.x, c1b.y};
            float dz[4][4], dcn[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float si = act[0][e], sf = act[1][e], tg = act[2][e], so = act[3][e];
                const float tc = tanhf(ct[e]);
                const float dc = dc0[e] + dh[e] * so * (1.f - tc * tc);
                dz[0][e] = dc * tg * si * (1.f - si);
                dz[1][e] = dc * cprev[e] * sf * (1.f - sf);
                dz[2][e] = dc * si * (1.f - tg * tg);
                dz[3][e] = dh[e] * tc * so * (1.f - so);
                dcn[e] = dc * sf;
            }
            *frag(sDC, ch, warp, lane) = make_float4(dcn[0], dcn[1], dcn[2], dcn[3]);
            uint32_t zA[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (va) st2(p.dz + ra * 512 + 128 * j + u0, dz[j][0], dz[j][1]);
                if (vb) st2(p.dz + rb * 512 + 128 * j + u0, dz[j][2], dz[j][3]);
                lstm_a_frag(zA[j], dz[j][0], dz[j][1], dz[j][2], dz[j][3]);
            }
            // [de | dh_{t-1}] += dz_chunk [W_ih | W_hh]_chunk: k-step j of the chunk = gate j of its 8 units
            mbar_wait(&bars[s], (uint32_t)(it >> 1) & 1u);
            const float* wc = wlane + s * BW_CHUNK;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int nt = 0; nt < 32; ++nt) {
                    const float2 w = *reinterpret_cast<const float2*>(wc + 8 * nt * BW_P + 8 * j);
                    mma_tf32(acc[nt], zA[j], __float_as_uint(w.x), __float_as_uint(w.y));
                }
            }
            __syncthreads();                       // every warp is done with stage s: refill it with item it + 2
            if (tid == 0 && it + 2 < items) {
                mbar_expect_tx(&bars[s], BW_CHUNK_BYTES);
                tma_load_1d(sWt + s * BW_CHUNK, p.w_gates_t + (int64_t)((it + 2) % PL_CHUNKS) * BW_CHUNK, BW_CHUNK_BYTES,
                            &bars[s]);
            }
        }
        // ---- dPre_enc = de * (e > 0)
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) {
            const int k = 8 * nt + 2 * t;
            const float2 ea = ld2(sa + SV_E + k, va), eb = ld2(sb + SV_E + k, vb);
            if (va) st2(dpa + st * p.d_t + k, ea.x > 0.f ? acc[nt][0] : 0.f, ea.y > 0.f ? acc[nt][1] : 0.f);
            if (vb) st2(dpb + st * p.d_t + k, eb.x > 0.f ? acc[nt][2] : 0.f, eb.y > 0.f ? acc[nt][3] : 0.f);
        }
    }
}

// ---- H = 256 (LSTMWrapper(Default(hidden_size=256), 256, 256)).  Saved row 2048 floats: [e (256) | h_prev (256) |
// sigmoid(i) | sigmoid(f) | tanh(g) | sigmoid(o) (4 x 256) | c_t (256) | h_t (256)]; dz rows [1024], dPre rows [256].
constexpr int SV2 = 2048;
constexpr int SV2_E = 0, SV2_HP = 256, SV2_ACT = 512, SV2_C = 1536, SV2_H = 1792;
// backward: [2 stages][512][40] transposed ring (80 KB per chunk) and the dh fragments [chunk][row group][lane]
constexpr int BW2_CHUNK = 2 * PW_H * BW_P;
constexpr uint32_t BW2_CHUNK_BYTES = BW2_CHUNK * 4u;
constexpr int FRAG2 = PW_CHUNKS * 4 * 32 * 4;
constexpr int SB2_DH = 2 * BW2_CHUNK;
constexpr size_t BWD2_SMEM = (size_t)(SB2_DH + FRAG2) * sizeof(float);
static_assert(BWD2_SMEM <= 227 * 1024, "shared memory over the sm_90 per-CTA limit");

// The forward at H = 256: 64 segments per CTA, 4 warps, the shared-memory plan of pb_policy_lstm_sample's H = 256 step
// (lstm_cell.cuh, PW_*).  Phase 1 runs the encoder for all T steps with W_enc and the x tile over the ring and h tile.
// Phase 2 walks the steps: at each step every warp reloads its 16 rows of the h tile from h_{t-1} (the saved rows it
// wrote, or h0); the state it needs per (row, unit) -- h_prev for the saved row and c_prev -- comes back from the saved
// row of step t-1 that the same thread wrote (or h0 / c0), so c and h round-trip through L2 / HBM once per step
// (2 KB per segment, against the 8 KB saved row written) instead of occupying 128 KB of shared memory.
template <int NC>
__global__ void __launch_bounds__(128, 1) k_lstm_bptt_fwd_256(FwdParams p) {
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
    const int T = p.steps, F = p.in_features;
    const int64_t b0 = (int64_t)blockIdx.x * PW_ROWS;
    const int valid = (int)((p.batch - b0) < PW_ROWS ? (p.batch - b0) : PW_ROWS);
    const int items = T * PW_CHUNKS;

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1);
        mbar_fence_init();
        mbar_expect_tx(&bars[0], PW_WENC_BYTES);
        tma_load_1d(sWe, p.w_enc, PW_WENC_BYTES, &bars[0]);
    }
    for (int i = tid; i < PW_H; i += 128) sBe[i] = p.b_enc[i];
    for (int i = tid; i < 4 * PW_H; i += 128) sBg[i] = p.b_gates[i];
    for (int i = tid; i < NC * PW_H; i += 128) sWh[(i >> 8) * PW_HP + (i & (PW_H - 1))] = p.w_heads[i];
    if (tid < NC) sBh[tid] = p.b_heads[tid];
    if (tid < PW_ROWS) {
        const int64_t b = b0 + tid;
        *xrow(sX, tid) = (b / p.groups) * p.s_e + (b % p.groups) * p.s_g;
    }

    const int lr = 16 * warp + g;
    const bool va = lr < valid, vb = lr + 8 < valid;
    const int64_t ra0 = (b0 + lr) * T, rb0 = ra0 + 8 * (int64_t)T;

    // ---- phase 1: e = relu(x W_enc^T + b_enc) for every step, to the saved rows
#pragma unroll 1
    for (int st = 0; st < T; ++st) {
        __syncthreads();
        for (int i = tid; i < PW_ROWS * PL_F; i += 128) {
            const int r = i >> 7, k = i & (PL_F - 1);
            sX[r * PL_XP + k] = (r < valid && k < F) ? p.obs[*xrow(sX, r) + st * p.s_t + k] : 0.f;
        }
        __syncthreads();
        if (st == 0) mbar_wait(&bars[0], 0);
        float acc[32][4];
        lstm_encoder(acc, sX + lr * PL_XP + 2 * t, sWe + g * PL_XP + 2 * t, F);
        lstm_encoder_relu(acc, sBe, t);
        float* sa = p.saved + (ra0 + st) * SV2 + SV2_E + 2 * t;
        float* sb = p.saved + (rb0 + st) * SV2 + SV2_E + 2 * t;
#pragma unroll
        for (int nt = 0; nt < 32; ++nt) {
            if (va) st2(sa + 8 * nt, acc[nt][0], acc[nt][1]);
            if (vb) st2(sb + 8 * nt, acc[nt][2], acc[nt][3]);
        }
    }
    fence_proxy_async_smem();                      // the x tile's generic writes before the ring's bulk copies
    __syncthreads();                               // x tile and W_enc are dead: the region becomes ring | h tile
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {              // items >= 32 > 2
            mbar_expect_tx(&bars[1 + s], PW_CHUNK_BYTES);
            tma_load_1d(sWg + s * PW_CHUNK, p.w_gates + (int64_t)s * PW_CHUNK, PW_CHUNK_BYTES, &bars[1 + s]);
        }
    }

    // ---- phase 2: the recurrence
    const float* wlane = sWg + g * PW_GP + 2 * t;
    const float* hs = sHt + lr * PW_HP + 2 * t;
    int it = 0;
#pragma unroll 1
    for (int st = 0; st < T; ++st) {
        const int64_t ra = ra0 + st, rb = rb0 + st;
        float* sa = p.saved + ra * SV2;
        float* sb = p.saved + rb * SV2;
        // h_{t-1} (or h0): the previous step's last stores of this warp's lanes are ordered before the reload
        __syncwarp();
        lstm_load_h_tile(sHt, 16 * warp, lane, [&](int r) -> const float* {
            const int lrow = 16 * warp + r;
            if (lrow >= valid) return nullptr;
            if (st > 0) return p.saved + ((b0 + lrow) * T + st - 1) * SV2 + SV2_H;
            return p.h0 ? p.h0 + (b0 + lrow) * PW_H : nullptr;
        });
        __syncwarp();
        // h_prev and c_prev of this thread's (row, unit) pairs: the saved row of step t-1 it wrote, or h0 / c0
        const float* hpa = st > 0 ? sa - SV2 + SV2_H : (p.h0 ? p.h0 + (b0 + lr) * PW_H : nullptr);
        const float* hpb = st > 0 ? sb - SV2 + SV2_H : (p.h0 ? p.h0 + (b0 + lr + 8) * PW_H : nullptr);
        const float* cpa = st > 0 ? sa - SV2 + SV2_C : (p.c0 ? p.c0 + (b0 + lr) * PW_H : nullptr);
        const float* cpb = st > 0 ? sb - SV2 + SV2_C : (p.c0 ? p.c0 + (b0 + lr + 8) * PW_H : nullptr);
        uint32_t eA[32][4];
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            const float2 e0 = ld2(sa + SV2_E + 8 * k + 2 * t, va), e1 = ld2(sb + SV2_E + 8 * k + 2 * t, vb);
            lstm_a_frag(eA[k], e0.x, e0.y, e1.x, e1.y);
        }
        float out[NC / 8][4];
#pragma unroll
        for (int q = 0; q < NC / 8; ++q) { out[q][0] = out[q][1] = out[q][2] = out[q][3] = 0.f; }
#pragma unroll 1
        for (int ch = 0; ch < PW_CHUNKS; ++ch, ++it) {
            const int s = it & 1;
            const int u0 = 8 * ch + 2 * t;
            const float2 ha = ld2(hpa + u0, va && hpa), hb = ld2(hpb + u0, vb && hpb);
            const float2 ca = ld2(cpa + u0, va && cpa), cb = ld2(cpb + u0, vb && cpb);
            float gacc[4][4];
            mbar_wait(&bars[1 + s], (uint32_t)(it >> 1) & 1u);
            lstm_gate_chunk_256(gacc, eA, hs, wlane + s * PW_CHUNK);
            __syncthreads();                       // every warp is done with stage s: refill it with item it + 2
            if (tid == 0 && it + 2 < items) {
                mbar_expect_tx(&bars[1 + s], PW_CHUNK_BYTES);
                tma_load_1d(sWg + s * PW_CHUNK, p.w_gates + (int64_t)((it + 2) % PW_CHUNKS) * PW_CHUNK, PW_CHUNK_BYTES,
                            &bars[1 + s]);
            }
            const float cp[4] = {ca.x, ca.y, cb.x, cb.y};
            float act[4][4], cn[4], hn[4];
            lstm_cell(gacc, sBg + 32 * ch + 2 * t, cp, act, cn, hn);
            if (va) {
                st2(sa + SV2_HP + u0, ha.x, ha.y);
#pragma unroll
                for (int j = 0; j < 4; ++j) st2(sa + SV2_ACT + PW_H * j + u0, act[j][0], act[j][1]);
                st2(sa + SV2_C + u0, cn[0], cn[1]);
                st2(sa + SV2_H + u0, hn[0], hn[1]);
            }
            if (vb) {
                st2(sb + SV2_HP + u0, hb.x, hb.y);
#pragma unroll
                for (int j = 0; j < 4; ++j) st2(sb + SV2_ACT + PW_H * j + u0, act[j][2], act[j][3]);
                st2(sb + SV2_C + u0, cn[2], cn[3]);
                st2(sb + SV2_H + u0, hn[2], hn[3]);
            }
            if (st == T - 1) {
                if (va) {
                    st2(p.h_out + (b0 + lr) * PW_H + u0, hn[0], hn[1]);
                    st2(p.c_out + (b0 + lr) * PW_H + u0, cn[0], cn[1]);
                }
                if (vb) {
                    st2(p.h_out + (b0 + lr + 8) * PW_H + u0, hn[2], hn[3]);
                    st2(p.c_out + (b0 + lr + 8) * PW_H + u0, cn[2], cn[3]);
                }
            }
            lstm_head_chunk<NC, PW_HP>(out, hn, sWh, g, u0);
        }
#pragma unroll
        for (int q = 0; q < NC / 8; ++q) {
            const int k = 8 * q + 2 * t;
            if (va) st2(p.out + ra * NC + k, out[q][0] + sBh[k], out[q][1] + sBh[k + 1]);
            if (vb) st2(p.out + rb * NC + k, out[q][2] + sBh[k], out[q][3] + sBh[k + 1]);
        }
    }
}

// The backward at H = 256: 64 segments per CTA, 8 warps.  Warp w takes row group w & 3 (16 segments) and output half
// w >> 2 of the product [de | dh_{t-1}] = dz [W_ih | W_hh]: half 0 accumulates de (256 columns, 128 registers), half 1
// dh_{t-1}, whose C fragment of n-tile ch is exactly the chunk-ch fragment the next (earlier) step needs.  Both halves
// compute the cell backward of every chunk (the same values: the A fragments of their product); half 0 writes dz.
// dh_t goes through shared memory (half 1 adds W_cat^T dOut_t and publishes it); dc_{t-1} is kept in the dPre row of step
// t-1, which only receives its dPre value after its own step has read dc back (half 0 writes both, each read is
// separated from the next write by a CTA barrier).  Shared memory: ring 2 x 80 KB + dh 64 KB = 224 KB; W_cat is read
// through L1.  The transposed gate weights stream from L2 at 2.6 MB per CTA per step (41 KB per segment).
template <int NC>
__global__ void __launch_bounds__(256, 1) k_lstm_bptt_bwd_256(BwdParams p) {
    extern __shared__ __align__(128) float smem[];
    float* sWt = smem;
    float* sDH = smem + SB2_DH;
    __shared__ __align__(8) uint64_t bars[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3, rg = warp & 3, half = warp >> 2;
    const int T = p.steps;
    const int64_t b0 = (int64_t)blockIdx.x * PW_ROWS;
    const int valid = (int)((p.batch - b0) < PW_ROWS ? (p.batch - b0) : PW_ROWS);
    const int items = T * PW_CHUNKS;

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_fence_init();
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            mbar_expect_tx(&bars[s], BW2_CHUNK_BYTES);
            tma_load_1d(sWt + s * BW2_CHUNK, p.w_gates_t + (int64_t)s * BW2_CHUNK, BW2_CHUNK_BYTES, &bars[s]);
        }
    }
    __syncthreads();                               // barrier inits are visible

    const int lr = 16 * rg + g;
    const bool va = lr < valid, vb = lr + 8 < valid;
    const int64_t ra0 = (b0 + lr) * T, rb0 = ra0 + 8 * (int64_t)T;
    const int64_t ba = b0 + lr, bb = ba + 8;
    float* const dpa = p.dpre + (ba / p.groups) * p.d_e + (ba % p.groups) * p.d_g;
    float* const dpb = p.dpre + (bb / p.groups) * p.d_e + (bb % p.groups) * p.d_g;
    const float* wlane = sWt + (PW_H * half + g) * BW_P + 2 * t;
    float acc[32][4];
#pragma unroll
    for (int nt = 0; nt < 32; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }   // dh_T = 0
    int it = 0;
#pragma unroll 1
    for (int st = T - 1; st >= 0; --st) {
        const int64_t ra = ra0 + st, rb = rb0 + st;
        const float* sa = p.saved + ra * SV2;
        const float* sb = p.saved + rb * SV2;
        // ---- dh_t = (recurrent part, half 1's accumulators) + W_cat^T dOut_t, to the dh fragments
        if (half == 1) {
            float da[NC], db[NC];
#pragma unroll
            for (int k = 0; k < NC; k += 2) {
                const float2 x0 = ld2(p.dout + ra * NC + k, va), x1 = ld2(p.dout + rb * NC + k, vb);
                da[k] = x0.x; da[k + 1] = x0.y; db[k] = x1.x; db[k + 1] = x1.y;
            }
#pragma unroll
            for (int ch = 0; ch < PW_CHUNKS; ++ch) {
                float d[4] = {acc[ch][0], acc[ch][1], acc[ch][2], acc[ch][3]};
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    if (k <= p.n_act) {
                        const float2 w = __ldg(reinterpret_cast<const float2*>(p.w_heads + k * PW_H + 8 * ch + 2 * t));
                        d[0] += da[k] * w.x; d[1] += da[k] * w.y; d[2] += db[k] * w.x; d[3] += db[k] * w.y;
                    }
                }
                reinterpret_cast<float4*>(sDH)[(ch * 4 + rg) * 32 + lane] = make_float4(d[0], d[1], d[2], d[3]);
            }
        }
#pragma unroll
        for (int nt = 0; nt < 32; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }
        __syncthreads();                           // dh_t is visible to both halves
        const float* cpa = st > 0 ? sa - SV2 + SV2_C : (p.c0 ? p.c0 + (b0 + lr) * PW_H : nullptr);
        const float* cpb = st > 0 ? sb - SV2 + SV2_C : (p.c0 ? p.c0 + (b0 + lr + 8) * PW_H : nullptr);
        const bool carry = st < T - 1;             // dc_t in the dPre row of step t (zero at t = T - 1)
#pragma unroll 1
        for (int ch = 0; ch < PW_CHUNKS; ++ch, ++it) {
            const int s = it & 1;
            const int u0 = 8 * ch + 2 * t;
            const float4 dhv = reinterpret_cast<const float4*>(sDH)[(ch * 4 + rg) * 32 + lane];
            const float2 dca = ld2(dpa + st * p.d_t + u0, va && carry), dcb = ld2(dpb + st * p.d_t + u0, vb && carry);
            const float dh[4] = {dhv.x, dhv.y, dhv.z, dhv.w}, dc0[4] = {dca.x, dca.y, dcb.x, dcb.y};
            float act[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 x0 = ld2(sa + SV2_ACT + PW_H * j + u0, va), x1 = ld2(sb + SV2_ACT + PW_H * j + u0, vb);
                act[j][0] = x0.x; act[j][1] = x0.y; act[j][2] = x1.x; act[j][3] = x1.y;
            }
            const float2 c0a = ld2(sa + SV2_C + u0, va), c0b = ld2(sb + SV2_C + u0, vb);
            const float2 c1a = ld2(cpa + u0, va && cpa), c1b = ld2(cpb + u0, vb && cpb);
            const float ct[4] = {c0a.x, c0a.y, c0b.x, c0b.y}, cprev[4] = {c1a.x, c1a.y, c1b.x, c1b.y};
            float dz[4][4], dcn[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float si = act[0][e], sf = act[1][e], tg = act[2][e], so = act[3][e];
                const float tc = tanhf(ct[e]);
                const float dc = dc0[e] + dh[e] * so * (1.f - tc * tc);
                dz[0][e] = dc * tg * si * (1.f - si);
                dz[1][e] = dc * cprev[e] * sf * (1.f - sf);
                dz[2][e] = dc * si * (1.f - tg * tg);
                dz[3][e] = dh[e] * tc * so * (1.f - so);
                dcn[e] = dc * sf;
            }
            uint32_t zA[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j) lstm_a_frag(zA[j], dz[j][0], dz[j][1], dz[j][2], dz[j][3]);
            if (half == 0) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (va) st2(p.dz + ra * (4 * PW_H) + PW_H * j + u0, dz[j][0], dz[j][1]);
                    if (vb) st2(p.dz + rb * (4 * PW_H) + PW_H * j + u0, dz[j][2], dz[j][3]);
                }
                if (st > 0) {                      // dc_{t-1} to the dPre row of step t - 1
                    if (va) st2(dpa + (st - 1) * p.d_t + u0, dcn[0], dcn[1]);
                    if (vb) st2(dpb + (st - 1) * p.d_t + u0, dcn[2], dcn[3]);
                }
            }
            mbar_wait(&bars[s], (uint32_t)(it >> 1) & 1u);
            const float* wc = wlane + s * BW2_CHUNK;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int nt = 0; nt < 32; ++nt) {
                    const float2 w = *reinterpret_cast<const float2*>(wc + 8 * nt * BW_P + 8 * j);
                    mma_tf32(acc[nt], zA[j], __float_as_uint(w.x), __float_as_uint(w.y));
                }
            }
            __syncthreads();                       // every warp is done with stage s (and with dc_t of chunk ch)
            if (tid == 0 && it + 2 < items) {
                mbar_expect_tx(&bars[s], BW2_CHUNK_BYTES);
                tma_load_1d(sWt + s * BW2_CHUNK, p.w_gates_t + (int64_t)((it + 2) % PW_CHUNKS) * BW2_CHUNK,
                            BW2_CHUNK_BYTES, &bars[s]);
            }
        }
        // ---- dPre_enc = de * (e > 0), over the carried dc_t (every read of it was before the last barrier)
        if (half == 0) {
#pragma unroll
            for (int nt = 0; nt < 32; ++nt) {
                const int k = 8 * nt + 2 * t;
                const float2 ea = ld2(sa + SV2_E + k, va), eb = ld2(sb + SV2_E + k, vb);
                if (va) st2(dpa + st * p.d_t + k, ea.x > 0.f ? acc[nt][0] : 0.f, ea.y > 0.f ? acc[nt][1] : 0.f);
                if (vb) st2(dpb + st * p.d_t + k, eb.x > 0.f ? acc[nt][2] : 0.f, eb.y > 0.f ? acc[nt][3] : 0.f);
            }
        }
    }
}

template <typename K, typename P>
int launch(K kernel, const P& p, size_t smem, cudaStream_t stream, int rows = BT_ROWS, int threads = BT_THREADS) {
    PB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)pb_ceil_div(p.batch, rows), threads, smem, stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

bool aligned(const void* ptr, uintptr_t a) { return ((uintptr_t)ptr & (a - 1)) == 0; }

// The checks and launch behind both forward entry points: x(b, t) = obs + (b / G) s_e + (b % G) s_g + t s_t (floats)
int forward_rows(const char* fn, const float* obs, int32_t in_features, int64_t batch, int32_t steps, int32_t groups,
                 int64_t s_e, int64_t s_g, int64_t s_t, const float* h0, const float* c0, const float* w_enc,
                 const float* b_enc, const float* w_gates, const float* b_gates, const float* w_heads,
                 const float* b_heads, int32_t input_size, int32_t hidden_size, int32_t n_act, float* out, float* h_out,
                 float* c_out, float* saved, void* stream) {
    PB_REQUIRE(batch >= 0 && steps >= 1, PB_ERR_INVALID, "%s: need batch >= 0 and steps >= 1", fn);
    PB_REQUIRE(groups >= 1 && batch % groups == 0, PB_ERR_INVALID, "%s: need groups >= 1 dividing batch (got %d, %lld)",
               fn, groups, (long long)batch);
    PB_REQUIRE(in_features >= 1 && in_features <= PL_F, PB_ERR_UNSUPPORTED,
               "%s: observation features must be in [1, %d] (got %d)", fn, PL_F, in_features);
    PB_REQUIRE(input_size == hidden_size && (hidden_size == PL_H || hidden_size == PW_H), PB_ERR_UNSUPPORTED,
               "%s: built for LSTM input size = hidden size = %d or %d (got %d, %d)", fn, PL_H, PW_H, input_size,
               hidden_size);
    PB_REQUIRE(n_act >= 1 && n_act <= 15, PB_ERR_UNSUPPORTED, "%s: n_act must be in [1, 15]", fn);
    if (batch == 0) return PB_OK;
    PB_REQUIRE(obs && w_enc && b_enc && w_gates && b_gates && w_heads && b_heads && out && h_out && c_out && saved,
               PB_ERR_INVALID, "%s: null pointer", fn);
    PB_REQUIRE(s_e >= in_features && s_t >= in_features && (groups == 1 || s_g >= in_features), PB_ERR_INVALID,
               "%s: observation strides must be at least in_features", fn);
    PB_REQUIRE(aligned(w_enc, 16) && aligned(w_gates, 16), PB_ERR_INVALID, "%s: w_enc / w_gates must be 16-byte aligned",
               fn);
    PB_REQUIRE(aligned(out, 8) && aligned(h_out, 8) && aligned(c_out, 8) && aligned(saved, 8) && aligned(h0, 8) &&
                   aligned(c0, 8),
               PB_ERR_INVALID, "%s: out / h / c / saved must be 8-byte aligned", fn);
    FwdParams p{obs, s_e, s_g, s_t, groups, in_features, batch, steps, h0, c0, w_enc, b_enc, w_gates, b_gates, w_heads,
                b_heads, out, h_out, c_out, saved};
    cudaStream_t s = (cudaStream_t)stream;
    if (hidden_size == PW_H)
        return n_act + 1 <= 8 ? launch(k_lstm_bptt_fwd_256<8>, p, PW_SMEM, s, PW_ROWS, 128)
                              : launch(k_lstm_bptt_fwd_256<16>, p, PW_SMEM, s, PW_ROWS, 128);
    return n_act + 1 <= 8 ? launch(k_lstm_bptt_fwd<8>, p, FWD_SMEM, s) : launch(k_lstm_bptt_fwd<16>, p, FWD_SMEM, s);
}

// The checks and launch behind both backward entry points: dPre row (b, t) at dpre + (b / G) d_e + (b % G) d_g + t d_t
int backward_rows(const char* fn, const float* dout, const float* saved, const float* c0, const float* w_gates_t,
                  const float* w_heads, int64_t batch, int32_t steps, int32_t input_size, int32_t hidden_size,
                  int32_t n_act, int32_t groups, int64_t d_e, int64_t d_g, int64_t d_t, float* dz, float* dpre,
                  void* stream) {
    PB_REQUIRE(batch >= 0 && steps >= 1, PB_ERR_INVALID, "%s: need batch >= 0 and steps >= 1", fn);
    PB_REQUIRE(groups >= 1 && batch % groups == 0, PB_ERR_INVALID, "%s: need groups >= 1 dividing batch (got %d, %lld)",
               fn, groups, (long long)batch);
    PB_REQUIRE(input_size == hidden_size && (hidden_size == PL_H || hidden_size == PW_H), PB_ERR_UNSUPPORTED,
               "%s: built for LSTM input size = hidden size = %d or %d (got %d, %d)", fn, PL_H, PW_H, input_size,
               hidden_size);
    PB_REQUIRE(n_act >= 1 && n_act <= 15, PB_ERR_UNSUPPORTED, "%s: n_act must be in [1, 15]", fn);
    if (batch == 0) return PB_OK;
    PB_REQUIRE(dout && saved && w_gates_t && w_heads && dz && dpre, PB_ERR_INVALID, "%s: null pointer", fn);
    PB_REQUIRE(d_e >= hidden_size && d_t >= hidden_size && (groups == 1 || d_g >= hidden_size) && d_e % 2 == 0 &&
                   d_g % 2 == 0 && d_t % 2 == 0,
               PB_ERR_INVALID, "%s: dPre strides must be even and at least %d floats", fn, hidden_size);
    PB_REQUIRE(aligned(w_gates_t, 16), PB_ERR_INVALID, "%s: w_gates_t must be 16-byte aligned", fn);
    PB_REQUIRE(aligned(dout, 8) && aligned(saved, 8) && aligned(c0, 8) && aligned(w_heads, 8) && aligned(dz, 8) &&
                   aligned(dpre, 8),
               PB_ERR_INVALID, "%s: dout / saved / c0 / w_heads / dz / dpre must be 8-byte aligned", fn);
    BwdParams p{dout, saved, c0, w_gates_t, w_heads, batch, steps, n_act, dz, dpre, groups, d_e, d_g, d_t};
    cudaStream_t s = (cudaStream_t)stream;
    if (hidden_size == PW_H)
        return n_act + 1 <= 8 ? launch(k_lstm_bptt_bwd_256<8>, p, BWD2_SMEM, s, PW_ROWS, 256)
                              : launch(k_lstm_bptt_bwd_256<16>, p, BWD2_SMEM, s, PW_ROWS, 256);
    return n_act + 1 <= 8 ? launch(k_lstm_bptt_bwd<8>, p, BWD_SMEM, s) : launch(k_lstm_bptt_bwd<16>, p, BWD_SMEM, s);
}

}  // namespace

extern "C" int pb_lstm_bptt_forward(const float* obs, int64_t obs_stride, int32_t in_features, int64_t batch,
                                    int32_t steps, const float* h0, const float* c0, const float* w_enc,
                                    const float* b_enc, const float* w_gates, const float* b_gates,
                                    const float* w_heads, const float* b_heads, int32_t input_size,
                                    int32_t hidden_size, int32_t n_act, float* out, float* h_out, float* c_out,
                                    float* saved, void* stream) {
    // the gathered layout: one group, row b*T + t at obs + (b*T + t) * obs_stride
    return forward_rows("pb_lstm_bptt_forward", obs, in_features, batch, steps, 1, (int64_t)steps * obs_stride, 0,
                        obs_stride, h0, c0, w_enc, b_enc, w_gates, b_gates, w_heads, b_heads, input_size, hidden_size,
                        n_act, out, h_out, c_out, saved, stream);
}

extern "C" int pb_lstm_bptt_forward_rows(const float* obs, int32_t in_features, int64_t batch, int32_t steps,
                                         int32_t groups, int64_t stride_e, int64_t stride_g, int64_t stride_t,
                                         const float* h0, const float* c0, const float* w_enc, const float* b_enc,
                                         const float* w_gates, const float* b_gates, const float* w_heads,
                                         const float* b_heads, int32_t input_size, int32_t hidden_size, int32_t n_act,
                                         float* out, float* h_out, float* c_out, float* saved, void* stream) {
    return forward_rows("pb_lstm_bptt_forward_rows", obs, in_features, batch, steps, groups, stride_e, stride_g,
                        stride_t, h0, c0, w_enc, b_enc, w_gates, b_gates, w_heads, b_heads, input_size, hidden_size,
                        n_act, out, h_out, c_out, saved, stream);
}

extern "C" int pb_lstm_bptt_backward(const float* dout, const float* saved, const float* c0, const float* w_gates_t,
                                     const float* w_heads, int64_t batch, int32_t steps, int32_t input_size,
                                     int32_t hidden_size, int32_t n_act, float* dz, float* dpre, void* stream) {
    // dPre dense [B*T][H] in row order b*T + t
    return backward_rows("pb_lstm_bptt_backward", dout, saved, c0, w_gates_t, w_heads, batch, steps, input_size,
                         hidden_size, n_act, 1, (int64_t)steps * hidden_size, 0, hidden_size, dz, dpre, stream);
}

extern "C" int pb_lstm_bptt_backward_rows(const float* dout, const float* saved, const float* c0,
                                          const float* w_gates_t, const float* w_heads, int64_t batch, int32_t steps,
                                          int32_t input_size, int32_t hidden_size, int32_t n_act, int32_t groups,
                                          int64_t dpre_stride_e, int64_t dpre_stride_g, int64_t dpre_stride_t,
                                          float* dz, float* dpre, void* stream) {
    return backward_rows("pb_lstm_bptt_backward_rows", dout, saved, c0, w_gates_t, w_heads, batch, steps, input_size,
                         hidden_size, n_act, groups, dpre_stride_e, dpre_stride_g, dpre_stride_t, dz, dpre, stream);
}
