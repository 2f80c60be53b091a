// mlp_update.cu -- the whole minibatch forward + PPO loss + backward of models.Default in ONE persistent Hopper kernel
// (wgmma + TMA + mbarrier): the observations are read from HBM once, `hidden` / `dPre` never leave the SM.
//
// Replaces, per minibatch of clean_pufferl.train (policy = models.Default with 128 input features, 128 hidden units,
// <= 7 actions), the chain
//     hidden = relu(x W_enc^T + b_enc)            (library GEMM, writes 268 MB at M = 524288)
//     out    = hidden W_heads^T + b_heads         (library GEMM, reads hidden)
//     pb_ppo_loss(out) -> dOut, statistics        (csrc/ppo_loss.cu)
//     pb_mlp_tail_backward(dOut, hidden) -> dPre, dW_heads, db_enc, db_heads      (csrc/mlp_tail.cu, reads hidden, writes dPre)
//     dW_enc = dPre^T x                           (split-K library GEMM, reads dPre and x)
// which streams `hidden` / `dPre` through HBM five times.  Here the algorithmic traffic is x once + 28 B of per-row scalars.
//
// One kernel, k_mlp_update, two warpgroups (256 threads), one CTA per SM looping over 64-row tiles of the minibatch:
//   * thread 0 keeps NSTAGE x tiles in flight (TMA, K-major SWIZZLE_128B), W_enc is resident in shared memory;
//   * hidden^T [128 hidden units][64 rows] = W_enc . x^T on the tensor core (wgmma SS, warpgroup wg: hidden units
//     64wg..64wg+63), so every thread holds two hidden units x 32 rows in registers;
//   * relu(hidden)^T goes to shared memory once (K-major [hidden unit][row]); the head products, the loss row math (four
//     lanes per row), g^T = W_heads^T dOut^T, dPre^T = g^T masked by the ReLU, db_enc and dW_heads^T = relu(h)^T dOut all
//     work on the registers of that accumulator layout;
//   * dW_enc^T [feature][hidden unit] += x^T . dPre on the tensor core (wgmma RS: x^T fragments read from the x tile, dPre^T
//     from shared memory as the K-major B operand); the accumulator stays in registers across all tiles of the CTA.
// Per-CTA partials go to a workspace and k_update_reduce sums them deterministically into the flat gradient buffer
// [dW_enc (hid x feat) | dW_heads (8 x hid) | db_enc | db_heads] of clean_pufferl._DefaultMLPUpdate, leaving per-block
// sums of squares for pb_clip_adam_parts.
//
// Epilogue precision (pb_mlp_update_set_variant): variant 2 (default) takes the head, g^T and dW_heads products on mma.sync
// with TF32 operands and fp32 accumulation -- the precision class of torch.set_float32_matmul_precision('high'), which
// clean_pufferl sets; variant 1 forms the head and g^T products with fp32 FFMAs.  The dPre-to-HBM mode (dW_enc by the
// caller) runs the variant-1 epilogue.  Every mbarrier wait is bounded (tma.cuh: __trap instead of a hang).
#include <cuda.h>
#include <stdlib.h>

#include "pb_common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace {

constexpr int TILE_M = 64, HID = 128, FEAT = 128, NO = 8;
constexpr int KBLK = 32;                               // floats per 128-byte swizzle row
constexpr int W_KBLK_BYTES = HID * KBLK * 4;           // 16 KiB: [128 hidden units][32 features]
constexpr int X_KBLK_BYTES = TILE_M * KBLK * 4;        // 8 KiB: [64 rows][32 features]
constexpr int X_TILE_BYTES = 4 * X_KBLK_BYTES;         // 32 KiB
constexpr int G_KBLK_BYTES = HID * 32 * 4;             // 16 KiB: [128 hidden units][32 rows]
constexpr int NSTAGE = 3;                              // x tiles in flight per SM
constexpr int THREADS = 256;                           // two warpgroups
constexpr int SM_W = 0;                                // W_enc, K-major SWIZZLE_128B, resident
constexpr int SM_X = 4 * W_KBLK_BYTES;                 // NSTAGE x tiles, K-major SWIZZLE_128B
constexpr int SM_G = SM_X + NSTAGE * X_TILE_BYTES;     // relu(h)^T, then dPre^T: two [128 hidden][32 rows] K-major blocks
constexpr int SM_WH = SM_G + 2 * G_KBLK_BYTES;         // W_heads [8][128]
constexpr int SM_BE = SM_WH + NO * HID * 4;            // b_enc [128]
constexpr int SM_OUT = SM_BE + HID * 4;                // head outputs [2 hidden halves][64 rows][8]
constexpr int SM_DO = SM_OUT + 2 * TILE_M * NO * 4;    // dOut [64 rows][8]
constexpr int SM_RED = SM_DO + TILE_M * NO * 4;        // db_heads partials [8 warps][8]
constexpr int SM_BAR = SM_RED + 8 * NO * 4;
constexpr int SMEM_TOTAL = SM_BAR + 64;
constexpr int TAIL = NO * HID + HID + NO;              // dW_heads | db_enc | db_heads
static_assert(SMEM_TOTAL <= 227 * 1024, "shared memory budget (227 KiB per block on sm_90)");

struct FusedParams {
    const int64_t* actions;
    const float* old_logprobs;
    const float* adv;
    const float* returns;      // nullable: returns = advantages (raw) + old_values (clean_pufferl.py:476-481)
    const float* old_values;
    const float* adv_norm;     // nullable: (mean, 1 / (std + 1e-8)) of this minibatch's raw advantages (:211-213)
    int64_t row_slab_stride;   // per-row arrays: slab s starts at element s * row_slab_stride (slab_rows: slab-major)
    int64_t m;                 // rows of the minibatch (all slabs): the 1/M of the loss means
    int64_t slab_rows;         // R
    int64_t slab_stride_rows;  // distance between slab starts, in rows of the x tensor map
    int tiles_per_slab, n_tiles;
    int n_act;
    float clip, vclip, vf_coef, ent_coef;
    int clip_vloss;
    float* part_dw;            // [grid][FEAT][HID]
    float* part_tail;          // [grid][TAIL]
    double* stats;             // [8]
    float* dpre_out;           // DW_KERNEL = false: dPre [m][128] (slab-major rows) for the caller's dW GEMM
    float* dbg_hidden;         // nullable [m][128]
    float* dbg_dpre;           // nullable [m][128]
    float* dbg_dout;           // nullable [m][8]
    const float* w_heads;      // [8][128], b_enc [128], b_heads [8]
    const float* b_enc;
    const float* b_heads;
};

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// mma.sync m16n8k8 TF32: a0 (g, t)  a1 (g + 8, t)  a2 (g, t + 4)  a3 (g + 8, t + 4);  b0 (k = t, n = g)  b1 (k = t + 4, n = g);
// c0 c1 (g, 2t + {0,1})  c2 c3 (g + 8, 2t + {0,1})      [g = lane >> 2, t = lane & 3]
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// byte offset of element (hidden unit n, tile row l) in the relu(h)^T / dPre^T buffer: two K-major SWIZZLE_128B blocks of
// [128 hidden units][32 rows] (rows 0..31, 32..63) -- the layout of a wgmma B operand with N = hidden units, K = rows
__device__ __forceinline__ uint32_t g_off(int n, int l) {
    return (uint32_t)((l >> 5) * G_KBLK_BYTES + n * 128 + ((((l & 31) >> 2) ^ (n & 7)) << 4) + (l & 3) * 4);
}
// byte offset of element (tile row r, feature f) in an x tile (four K-major SWIZZLE_128B blocks of [64 rows][32 features])
__device__ __forceinline__ uint32_t x_off(int r, int f) {
    return (uint32_t)((f >> 5) * X_KBLK_BYTES + r * 128 + ((((f & 31) >> 2) ^ (r & 7)) << 4) + (f & 3) * 4);
}

struct RowStats { float pg, v, ent, okl, kl, clipped; };

// The row math of k_ppo_loss<PACKED> (csrc/ppo_loss.cu; clean_pufferl.py:202-238 + frameworks/cleanrl.py:25-47) with FOUR
// lanes per row: lane `sub` (0..3) of the row owns outputs sub and sub + 4 (logits below n_act, the value at index n_act);
// row-wide maxima / sums go through width-4 shuffles.  Every lane of the warp must call it (shuffles).  Returns dOut of the
// two owned outputs (already scaled by 1/M) and the six per-row statistics.
__device__ __forceinline__ RowStats ppo_row_sub(float z_lo, float z_hi, int sub, int lane, const FusedParams& p, int act,
                                                float old_lp, float adv, float ret, float old_v, float& g_lo, float& g_hi) {
    const unsigned full = 0xffffffffu;
    const int n = p.n_act;
    const bool lo_ok = sub < n, hi_ok = sub + 4 < n;
    float mx = fmaxf(lo_ok ? z_lo : -INFINITY, hi_ok ? z_hi : -INFINITY);
    mx = fmaxf(mx, __shfl_xor_sync(full, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(full, mx, 2));
    float sum = (lo_ok ? expf(z_lo - mx) : 0.f) + (hi_ok ? expf(z_hi - mx) : 0.f);
    sum += __shfl_xor_sync(full, sum, 1);
    sum += __shfl_xor_sync(full, sum, 2);
    const float lse = mx + logf(sum);
    const float nl_lo = z_lo - lse, nl_hi = z_hi - lse;
    const float pk_lo = lo_ok ? expf(nl_lo) : 0.f, pk_hi = hi_ok ? expf(nl_hi) : 0.f;
    float ent = -(lo_ok ? pk_lo * nl_lo : 0.f) - (hi_ok ? pk_hi * nl_hi : 0.f);
    ent += __shfl_xor_sync(full, ent, 1);
    ent += __shfl_xor_sync(full, ent, 2);
    const int a = act < 0 ? 0 : (act >= n ? n - 1 : act);
    const int base = lane & ~3;
    const float nl_a = __shfl_sync(full, (a >> 2) ? nl_hi : nl_lo, base | (a & 3));
    const float v_new = __shfl_sync(full, (n >> 2) ? z_hi : z_lo, base | (n & 3));
    const float logratio = nl_a - old_lp;
    const float ratio = expf(logratio);
    const float pg1 = -adv * ratio;
    const float rc = fminf(fmaxf(ratio, 1.f - p.clip), 1.f + p.clip);
    const float pg2 = -adv * rc;
    const float pg = fmaxf(pg1, pg2);
    const float in_range = (ratio >= 1.f - p.clip && ratio <= 1.f + p.clip) ? 1.f : 0.f;
    float g_ratio;
    if (pg1 > pg2) g_ratio = -adv;
    else if (pg1 < pg2) g_ratio = -adv * in_range;
    else g_ratio = 0.5f * (-adv) + 0.5f * (-adv * in_range);
    const float inv_m = 1.0f / (float)p.m;
    const float g_nlp = g_ratio * ratio * inv_m;
    const float dv = v_new - ret;
    float vl, g_v;
    if (p.clip_vloss) {
        const float d = v_new - old_v;
        const float dc = fminf(fmaxf(d, -p.vclip), p.vclip);
        const float vc = old_v + dc;
        const float vu = dv * dv, vcl = (vc - ret) * (vc - ret);
        vl = fmaxf(vu, vcl);
        const float v_in = (d >= -p.vclip && d <= p.vclip) ? 1.f : 0.f;
        const float gu = 2.f * dv, gc = 2.f * (vc - ret) * v_in;
        g_v = vu > vcl ? gu : (vu < vcl ? gc : 0.5f * (gu + gc));
    } else {
        vl = dv * dv;
        g_v = 2.f * dv;
    }
    const float gv_out = 0.5f * p.vf_coef * g_v * inv_m;
    const float g_ent = p.ent_coef * inv_m;
    g_lo = lo_ok ? g_nlp * ((sub == a ? 1.f : 0.f) - pk_lo) + g_ent * pk_lo * (nl_lo + ent) : 0.f;
    g_hi = hi_ok ? g_nlp * ((sub + 4 == a ? 1.f : 0.f) - pk_hi) + g_ent * pk_hi * (nl_hi + ent) : 0.f;
    if (sub == n) g_lo = gv_out;
    if (sub + 4 == n) g_hi = gv_out;
    RowStats s;
    s.pg = pg; s.v = vl; s.ent = ent; s.okl = -logratio; s.kl = (ratio - 1.f) - logratio;
    s.clipped = fabsf(ratio - 1.f) > p.clip ? 1.f : 0.f;
    return s;
}

// TF32_EPI  : head / g^T / dW_heads products on mma.sync with TF32 operands (variant 2); else fp32 FFMAs for the head and
//             g^T products and TF32 (round-to-nearest operands) for dW_heads (variant 1)
// DW_KERNEL : dW_enc^T accumulated on the tensor core; else dPre goes to HBM (p.dpre_out) and the caller forms dW_enc
template <bool TF32_EPI, bool DW_KERNEL>
__global__ void __launch_bounds__(THREADS, 1)
k_mlp_update(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const FusedParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* w_full = reinterpret_cast<uint64_t*>(smem + SM_BAR);
    uint64_t* x_full = w_full + 1;                                 // [NSTAGE]
    float* wh = reinterpret_cast<float*>(smem + SM_WH);
    const float* be = reinterpret_cast<const float*>(smem + SM_BE);
    float* outp = reinterpret_cast<float*>(smem + SM_OUT);
    float* dos = reinterpret_cast<float*>(smem + SM_DO);
    float* red = reinterpret_cast<float*>(smem + SM_RED);
    uint8_t* gbuf = smem + SM_G;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int wg = warp >> 2, wq = warp & 3;
    const int n_my = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // tiles of this CTA (>= 1)

    auto issue = [&](int it) {           // thread 0: x tile `it` of this CTA into stage it % NSTAGE
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        const int64_t row0 = (int64_t)(tile / p.tiles_per_slab) * p.slab_stride_rows + (int64_t)(tile % p.tiles_per_slab) * TILE_M;
        const int s = it % NSTAGE;
        mbar_expect_tx(&x_full[s], X_TILE_BYTES);
        for (int kb = 0; kb < 4; ++kb)
            tma_load_2d(smem + SM_X + s * X_TILE_BYTES + kb * X_KBLK_BYTES, &map_x, kb * KBLK, (int)row0, &x_full[s]);
    };
    if (tid == 0) {
        mbar_init(w_full, 1);
        for (int s = 0; s < NSTAGE; ++s) mbar_init(&x_full[s], 1);
        mbar_fence_init();
    }
    for (int i = tid; i < NO * HID; i += THREADS) wh[i] = p.w_heads[i];
    if (tid < HID) reinterpret_cast<float*>(smem + SM_BE)[tid] = p.b_enc[tid];
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(w_full, 4 * W_KBLK_BYTES);
        for (int kb = 0; kb < 4; ++kb) tma_load_2d(smem + SM_W + kb * W_KBLK_BYTES, &map_w, kb * KBLK, 0, w_full);
        for (int it = 0; it < NSTAGE && it < n_my; ++it) issue(it);
    }

    // this thread's two hidden units in the hidden^T accumulator (rows of the wgmma D fragment)
    const int hr0 = 64 * wg + 16 * wq + g, hr1 = hr0 + 8;
    // the loss: four lanes per tile row (ppo_row_sub)
    const int lr = tid >> 2, sub = tid & 3;
    const float bh_lo = p.b_heads[sub], bh_hi = p.b_heads[sub + 4];
    // W_heads operands, resident in registers
    uint32_t hb[8][2], ga[4];            // TF32_EPI: heads B fragments (hidden half warp >> 2), g^T A fragment
    float whr[2][NO];                    // fp32 epilogue: W_heads[a][hr0], W_heads[a][hr1]
    if (TF32_EPI) {
        const int hh = warp >> 2;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            hb[ks][0] = to_tf32(wh[g * HID + 64 * hh + 8 * ks + t]);
            hb[ks][1] = to_tf32(wh[g * HID + 64 * hh + 8 * ks + t + 4]);
        }
        ga[0] = to_tf32(wh[t * HID + hr0]);
        ga[1] = to_tf32(wh[t * HID + hr1]);
        ga[2] = to_tf32(wh[(t + 4) * HID + hr0]);
        ga[3] = to_tf32(wh[(t + 4) * HID + hr1]);
    } else {
#pragma unroll
        for (int a = 0; a < NO; ++a) {
            whr[0][a] = wh[a * HID + hr0];
            whr[1][a] = wh[a * HID + hr1];
        }
    }

    float dwacc[64];                     // dW_enc^T [feature 64wg + 16wq + g (+8)][hidden unit 8j + 2t (+1)]
#pragma unroll
    for (int i = 0; i < 64; ++i) dwacc[i] = 0.f;
    float dwh[4] = {0.f, 0.f, 0.f, 0.f};  // dW_heads^T [hr0 | hr1][head 2t | 2t + 1]
    float be_acc[2] = {0.f, 0.f};        // db_enc[hr0], db_enc[hr1] over this thread's rows
    float bh_acc[2] = {0.f, 0.f};        // db_heads[sub], [sub + 4] over this thread's loss rows
    double st[6] = {0, 0, 0, 0, 0, 0};
    const float adv_mean = p.adv_norm ? p.adv_norm[0] : 0.f, adv_rstd = p.adv_norm ? p.adv_norm[1] : 1.f;
    const bool need_old_v = p.clip_vloss || !p.returns;
    const uint32_t w_addr = smem_u32(smem + SM_W), g_addr = smem_u32(gbuf);

    for (int it = 0; it < n_my; ++it) {
        const int s = it % NSTAGE;
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        const int slab = tile / p.tiles_per_slab, tis = tile - slab * p.tiles_per_slab;
        const int64_t lrow0 = (int64_t)tis * TILE_M;                          // slab-local row of tile row 0
        const int rows_left = (int)(p.slab_rows - lrow0 < TILE_M ? p.slab_rows - lrow0 : TILE_M);
        const int64_t i0 = (int64_t)slab * p.slab_rows + lrow0;               // slab-major position (dPre / debug rows)
        // per-row inputs of the loss row (issued before the waits: their latency hides behind the forward product)
        const bool valid = lr < rows_left;
        int act = 0;
        float old_lp = 0.f, adv = 0.f, ret = 0.f, old_v = 0.f;
        if (valid) {
            const int64_t ri = (int64_t)slab * p.row_slab_stride + lrow0 + lr;
            act = (int)p.actions[ri];
            old_lp = p.old_logprobs[ri];
            adv = p.adv[ri];
            if (need_old_v) old_v = p.old_values[ri];
            if (p.returns) ret = p.returns[ri];
        }
        if (it == 0) mbar_wait(w_full, 0);
        mbar_wait(&x_full[s], (uint32_t)((it / NSTAGE) & 1));
        const uint8_t* xs = smem + SM_X + s * X_TILE_BYTES;
        const uint32_t x_addr = smem_u32(xs);

        // ---- 1. hidden^T = W_enc[64wg .. 64wg + 63] . x^T  (M = hidden units, N = 64 rows, K = 128 features)
        float h[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) h[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < 4; ++kb)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_m64n64k8_ss(h, wgmma_desc_sw128(w_addr + kb * W_KBLK_BYTES + wg * 8192 + k * 32),
                                  wgmma_desc_sw128(x_addr + kb * X_KBLK_BYTES + k * 32), (kb | k) ? 1 : 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(h);

        // ---- 2. relu(h + b_enc)^T -> shared memory (the operand of the head products)
        {
            const float b0 = be[hr0], b1 = be[hr1];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                h[4 * j] = fmaxf(h[4 * j] + b0, 0.f);
                h[4 * j + 1] = fmaxf(h[4 * j + 1] + b0, 0.f);
                h[4 * j + 2] = fmaxf(h[4 * j + 2] + b1, 0.f);
                h[4 * j + 3] = fmaxf(h[4 * j + 3] + b1, 0.f);
                const int l = 8 * j + 2 * t;
                *reinterpret_cast<float2*>(gbuf + g_off(hr0, l)) = make_float2(h[4 * j], h[4 * j + 1]);
                *reinterpret_cast<float2*>(gbuf + g_off(hr1, l)) = make_float2(h[4 * j + 2], h[4 * j + 3]);
                if (p.dbg_hidden) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int le = l + (e & 1), he = (e & 2) ? hr1 : hr0;
                        if (le < rows_left) p.dbg_hidden[(i0 + le) * HID + he] = h[4 * j + e];
                    }
                }
            }
        }
        __syncthreads();

        // ---- 3. head products: out[row][a] = relu(h)[row] . W_heads[a]
        if (TF32_EPI) {      // warp: rows 16(warp & 3) .. +15, hidden half warp >> 2; partial sums of the two halves to outp
            const int l0 = 16 * (warp & 3) + g, hh = warp >> 2;
            float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const int n0 = 64 * hh + 8 * ks + t;
                const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(gbuf + g_off(n0, l0)),
                                       *reinterpret_cast<const uint32_t*>(gbuf + g_off(n0, l0 + 8)),
                                       *reinterpret_cast<const uint32_t*>(gbuf + g_off(n0 + 4, l0)),
                                       *reinterpret_cast<const uint32_t*>(gbuf + g_off(n0 + 4, l0 + 8))};
                mma_tf32(c, a, hb[ks][0], hb[ks][1]);
            }
            *reinterpret_cast<float2*>(outp + (hh * TILE_M + l0) * NO + 2 * t) = make_float2(c[0], c[1]);
            *reinterpret_cast<float2*>(outp + (hh * TILE_M + l0 + 8) * NO + 2 * t) = make_float2(c[2], c[3]);
        } else {             // thread = (row, pair of heads), fp32 FFMAs over all 128 hidden units
            const int l = tid & (TILE_M - 1), a0 = 2 * (tid >> 6);
            float o0 = 0.f, o1 = 0.f;
            if (a0 <= p.n_act) {
#pragma unroll 8
                for (int n = 0; n < HID; ++n) {
                    const float rh = *reinterpret_cast<const float*>(gbuf + g_off(n, l));
                    o0 = fmaf(rh, wh[a0 * HID + n], o0);
                    o1 = fmaf(rh, wh[(a0 + 1) * HID + n], o1);
                }
            }
            *reinterpret_cast<float2*>(outp + l * NO + a0) = make_float2(o0, o1);
        }
        __syncthreads();

        // ---- 4. the loss row math -> dOut of the tile
        {
            float z_lo = bh_lo + outp[lr * NO + sub], z_hi = bh_hi + outp[lr * NO + sub + 4];
            if (TF32_EPI) {
                z_lo += outp[(TILE_M + lr) * NO + sub];
                z_hi += outp[(TILE_M + lr) * NO + sub + 4];
            }
            const float r_ = p.returns ? ret : adv + old_v;       // returns = raw advantages + old values (:476-481)
            const float a_ = (adv - adv_mean) * adv_rstd;
            float g_lo, g_hi;
            const RowStats rs = ppo_row_sub(z_lo, z_hi, sub, lane, p, act, old_lp, a_, r_, old_v, g_lo, g_hi);
            if (!valid) g_lo = g_hi = 0.f;
            if (valid && sub == 0) {
                st[0] += rs.pg; st[1] += rs.v; st[2] += rs.ent; st[3] += rs.okl; st[4] += rs.kl; st[5] += rs.clipped;
            }
            bh_acc[0] += g_lo;
            bh_acc[1] += g_hi;
            dos[lr * NO + sub] = g_lo;
            dos[lr * NO + sub + 4] = g_hi;
            if (p.dbg_dout && valid) {
                p.dbg_dout[(i0 + lr) * 8 + sub] = g_lo;
                p.dbg_dout[(i0 + lr) * 8 + sub + 4] = g_hi;
            }
        }
        __syncthreads();

        // ---- 5. g^T = W_heads^T dOut^T (same fragment layout as hidden^T), dPre^T = g^T where relu(h) > 0, db_enc, and
        //         dW_heads^T += relu(h)^T dOut with the hidden^T registers as the A fragments (k = t <-> row 8j + 2t,
        //         k = t + 4 <-> row 8j + 2t + 1)
        float dp[32];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (TF32_EPI) {
                float c[4] = {0.f, 0.f, 0.f, 0.f};
                mma_tf32(c, ga, __float_as_uint(dos[(8 * j + g) * NO + t]), __float_as_uint(dos[(8 * j + g) * NO + t + 4]));
                dp[4 * j] = c[0]; dp[4 * j + 1] = c[1]; dp[4 * j + 2] = c[2]; dp[4 * j + 3] = c[3];
            } else {
                const int l = 8 * j + 2 * t;
                const float4 d0a = *reinterpret_cast<const float4*>(dos + l * NO), d0b = *reinterpret_cast<const float4*>(dos + l * NO + 4);
                const float4 d1a = *reinterpret_cast<const float4*>(dos + (l + 1) * NO), d1b = *reinterpret_cast<const float4*>(dos + (l + 1) * NO + 4);
                const float d0[8] = {d0a.x, d0a.y, d0a.z, d0a.w, d0b.x, d0b.y, d0b.z, d0b.w};
                const float d1[8] = {d1a.x, d1a.y, d1a.z, d1a.w, d1b.x, d1b.y, d1b.z, d1b.w};
                float s00 = 0.f, s01 = 0.f, s10 = 0.f, s11 = 0.f;
#pragma unroll
                for (int a = 0; a < NO; ++a) {
                    s00 = fmaf(d0[a], whr[0][a], s00);
                    s01 = fmaf(d1[a], whr[0][a], s01);
                    s10 = fmaf(d0[a], whr[1][a], s10);
                    s11 = fmaf(d1[a], whr[1][a], s11);
                }
                dp[4 * j] = s00; dp[4 * j + 1] = s01; dp[4 * j + 2] = s10; dp[4 * j + 3] = s11;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) dp[4 * j + e] = h[4 * j + e] > 0.f ? dp[4 * j + e] : 0.f;
            be_acc[0] += dp[4 * j] + dp[4 * j + 1];
            be_acc[1] += dp[4 * j + 2] + dp[4 * j + 3];
            const float b0 = dos[(8 * j + 2 * t) * NO + g], b1 = dos[(8 * j + 2 * t + 1) * NO + g];
            if (TF32_EPI) {
                const uint32_t a[4] = {__float_as_uint(h[4 * j]), __float_as_uint(h[4 * j + 2]), __float_as_uint(h[4 * j + 1]),
                                       __float_as_uint(h[4 * j + 3])};
                mma_tf32(dwh, a, __float_as_uint(b0), __float_as_uint(b1));
            } else {
                const uint32_t a[4] = {to_tf32(h[4 * j]), to_tf32(h[4 * j + 2]), to_tf32(h[4 * j + 1]), to_tf32(h[4 * j + 3])};
                mma_tf32(dwh, a, to_tf32(b0), to_tf32(b1));
            }
            const int l = 8 * j + 2 * t;
            if (p.dbg_dpre) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int le = l + (e & 1), he = (e & 2) ? hr1 : hr0;
                    if (le < rows_left) p.dbg_dpre[(i0 + le) * HID + he] = dp[4 * j + e];
                }
            }
            // dPre^T over relu(h)^T (every read of relu(h)^T, step 3, is behind the last barrier): TF32 rounded to nearest as
            // the operand of the dW product, or exact for the row writes of the dPre-to-HBM mode
            if (DW_KERNEL) {
                *reinterpret_cast<uint2*>(gbuf + g_off(hr0, l)) = make_uint2(to_tf32(dp[4 * j]), to_tf32(dp[4 * j + 1]));
                *reinterpret_cast<uint2*>(gbuf + g_off(hr1, l)) = make_uint2(to_tf32(dp[4 * j + 2]), to_tf32(dp[4 * j + 3]));
            } else {
                *reinterpret_cast<float2*>(gbuf + g_off(hr0, l)) = make_float2(dp[4 * j], dp[4 * j + 1]);
                *reinterpret_cast<float2*>(gbuf + g_off(hr1, l)) = make_float2(dp[4 * j + 2], dp[4 * j + 3]);
            }
        }

        // ---- 6. dW_enc^T [64wg .. 64wg + 63][128] += x^T . dPre  (M = features, N = hidden units, K = 64 rows).  Both
        //         operands are rounded to nearest TF32 (truncation would bias a sum over the whole minibatch)
        if (DW_KERNEL) {
            fence_proxy_async_smem();            // dPre^T written by the generic proxy, read by the tensor core
            __syncthreads();
            const int f0 = 64 * wg + 16 * wq + g;
            uint32_t xa[8][4];                   // all A fragments of the tile: registers stay owned until the wait
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const int r0 = 8 * ks + t;
                xa[ks][0] = to_tf32(*reinterpret_cast<const float*>(xs + x_off(r0, f0)));
                xa[ks][1] = to_tf32(*reinterpret_cast<const float*>(xs + x_off(r0, f0 + 8)));
                xa[ks][2] = to_tf32(*reinterpret_cast<const float*>(xs + x_off(r0 + 4, f0)));
                xa[ks][3] = to_tf32(*reinterpret_cast<const float*>(xs + x_off(r0 + 4, f0 + 8)));
            }
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks)
                wgmma_m64n128k8_rs(dwacc, xa[ks], wgmma_desc_sw128(g_addr + (ks >> 2) * G_KBLK_BYTES + (ks & 3) * 32), 1);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(dwacc);
#pragma unroll
            for (int ks = 0; ks < 8; ++ks)
#pragma unroll
                for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(xa[ks][i])::"memory");
        } else {
            // ---- 6'. dPre rows to HBM: warp w writes rows 8w .. 8w + 7, one whole 512-byte row per store instruction
            __syncthreads();
#pragma unroll
            for (int k = 0; k < TILE_M / 8; ++k) {
                const int l = 8 * warp + k;
                if (l < rows_left) {
                    const int n = 4 * lane;
                    const float4 v = make_float4(*reinterpret_cast<const float*>(gbuf + g_off(n, l)),
                                                 *reinterpret_cast<const float*>(gbuf + g_off(n + 1, l)),
                                                 *reinterpret_cast<const float*>(gbuf + g_off(n + 2, l)),
                                                 *reinterpret_cast<const float*>(gbuf + g_off(n + 3, l)));
                    __stcs(reinterpret_cast<float4*>(p.dpre_out + (i0 + l) * HID + n), v);
                }
            }
        }
        __syncthreads();                         // every read of x stage s and of the shared tile buffers is done
        if (tid == 0 && it + NSTAGE < n_my) {
            fence_proxy_async_smem();
            issue(it + NSTAGE);
        }
    }

    // ================= per-CTA partials =================
    if (DW_KERNEL) {
        float* pd = p.part_dw + (int64_t)blockIdx.x * FEAT * HID;
        const int f0 = 64 * wg + 16 * wq + g;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            *reinterpret_cast<float2*>(pd + f0 * HID + 8 * j + 2 * t) = make_float2(dwacc[4 * j], dwacc[4 * j + 1]);
            *reinterpret_cast<float2*>(pd + (f0 + 8) * HID + 8 * j + 2 * t) = make_float2(dwacc[4 * j + 2], dwacc[4 * j + 3]);
        }
    }
    float* pt = p.part_tail + (int64_t)blockIdx.x * TAIL;
    pt[(2 * t) * HID + hr0] = dwh[0];
    pt[(2 * t + 1) * HID + hr0] = dwh[1];
    pt[(2 * t) * HID + hr1] = dwh[2];
    pt[(2 * t + 1) * HID + hr1] = dwh[3];
#pragma unroll
    for (int k = 0; k < 2; ++k) {        // db_enc: the four lanes of a hidden unit hold disjoint rows
        be_acc[k] += __shfl_xor_sync(0xffffffffu, be_acc[k], 1);
        be_acc[k] += __shfl_xor_sync(0xffffffffu, be_acc[k], 2);
    }
    if (t == 0) {
        pt[NO * HID + hr0] = be_acc[0];
        pt[NO * HID + hr1] = be_acc[1];
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)          // db_heads: the eight lanes with the same sub
#pragma unroll
        for (int off = 4; off < 32; off <<= 1) bh_acc[k] += __shfl_xor_sync(0xffffffffu, bh_acc[k], off);
    if (lane < 4) {
        red[warp * NO + lane] = bh_acc[0];
        red[warp * NO + lane + 4] = bh_acc[1];
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {        // loss statistics: the sub == 0 lanes hold this warp's rows
        double x = st[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
        if (lane == 0) atomicAdd(p.stats + k, x);
    }
    __syncthreads();
    if (tid < NO) {
        float v = 0.f;
        for (int w = 0; w < THREADS / 32; ++w) v += red[w * NO + tid];
        pt[NO * HID + HID + tid] = v;
    }
}

// Deterministic sum of the per-CTA partials into the flat gradient buffer:
//   gflat = [ dW_enc[hid][feat] (transposed from the partials' [feat][hid]) | dW_heads 8 x hid | db_enc | db_heads ]
// Block = 64 outputs x 4 partial groups; consecutive threads read consecutive partial elements (coalesced).
__global__ void __launch_bounds__(256) k_update_reduce(const float* __restrict__ part_dw, const float* __restrict__ part_tail,
                                                       int n_parts, float* __restrict__ gflat, double* __restrict__ sumsq_part) {
    __shared__ float sh[4][64];
    __shared__ double sq[2];
    const int e = blockIdx.x * 64 + (threadIdx.x & 63), grp = threadIdx.x >> 6;
    constexpr int NDW = FEAT * HID;
    float s = 0.f;
    if (e < NDW && !part_dw) {                // dW_enc is formed by the caller (dPre went to HBM); whole blocks: NDW % 64 == 0
        if (threadIdx.x == 0) sumsq_part[blockIdx.x] = 0.0;
        return;
    }
    if (e < NDW + TAIL) {
        const float* src = e < NDW ? part_dw + e : part_tail + (e - NDW);
        const int64_t stride = e < NDW ? NDW : TAIL;
#pragma unroll 4
        for (int pidx = grp; pidx < n_parts; pidx += 4) s += src[(int64_t)pidx * stride];
    }
    sh[grp][threadIdx.x & 63] = s;
    __syncthreads();
    if (grp == 0) {                           // warps 0 and 1
        float tot = 0.f;
        if (e < NDW + TAIL) {
            tot = sh[0][threadIdx.x] + sh[1][threadIdx.x] + sh[2][threadIdx.x] + sh[3][threadIdx.x];
            if (e < NDW) gflat[(e % HID) * FEAT + e / HID] = tot;      // partial element (f, j) -> dW_enc[j][f]
            else gflat[e] = tot;
        }
        // sum of squares of this block's 64 gradient elements: the global-norm pass of the optimizer step becomes a sum of
        // gridDim.x doubles (pb_clip_adam_parts), in a fixed order
        double d = (double)tot * (double)tot;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
        if ((threadIdx.x & 31) == 0) sq[threadIdx.x >> 5] = d;
    }
    __syncthreads();
    if (threadIdx.x == 0) sumsq_part[blockIdx.x] = sq[0] + sq[1];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D map of a [rows][128] fp32 matrix (row stride in floats), boxes of [box_rows][32 floats] with the 128-byte swizzle
int make_map2(EncodeTiledFn fn, CUtensorMap* map, const float* base, int64_t rows, int64_t row_stride_floats, int box_rows) {
    const cuuint64_t dims[2] = {(cuuint64_t)FEAT, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)row_stride_floats * 4};
    const cuuint32_t box[2] = {(cuuint32_t)KBLK, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_REQUIRE(r == CUDA_SUCCESS, PB_ERR_CUDA, "cuTensorMapEncodeTiled failed: %d", (int)r);
    return PB_OK;
}

int num_sms() { return pb_num_sms(); }

int g_update_variant = 2;     // 1 = fp32 head / g^T products, 2 = TF32 mma.sync epilogue

}  // namespace

extern "C" int pb_mlp_update_set_variant(int32_t variant) {
    PB_REQUIRE(variant == 1 || variant == 2, PB_ERR_INVALID, "pb_mlp_update_set_variant: 1 or 2");
    g_update_variant = variant;
    return PB_OK;
}

constexpr int REDUCE_BLOCKS = (FEAT * HID + TAIL + 63) / 64;

// workspace: per-CTA partials [SMs][FEAT * HID + TAIL] floats | REDUCE_BLOCKS doubles (sums of squares of the gradient)
extern "C" size_t pb_mlp_update_sumsq_offset(void) {
    return (((size_t)num_sms() * (FEAT * HID + TAIL) * sizeof(float)) + 15) & ~(size_t)15;
}
extern "C" int32_t pb_mlp_update_sumsq_parts(void) { return REDUCE_BLOCKS; }
extern "C" size_t pb_mlp_update_workspace_bytes(void) {
    return pb_mlp_update_sumsq_offset() + REDUCE_BLOCKS * sizeof(double);
}

extern "C" int pb_mlp_update_fused(const float* x, int64_t ldx, int64_t slab_rows, int64_t slab_stride_rows, int32_t n_slabs,
                                   const float* w_enc, const float* b_enc, const float* w_heads, const float* b_heads,
                                   const int64_t* actions, const float* old_logprobs, const float* advantages,
                                   const float* returns, const float* old_values, const float* adv_norm,
                                   int64_t row_slab_stride, int32_t n_act, float clip_coef,
                                   int32_t clip_vloss, float vf_clip_coef, float vf_coef, float ent_coef, float* grad_flat,
                                   double* stats8, void* workspace, size_t workspace_bytes, float* dpre_out,
                                   float* dbg_hidden, float* dbg_dpre, float* dbg_dout, void* stream) {
    PB_REQUIRE(x && w_enc && b_enc && w_heads && b_heads && actions && old_logprobs && advantages && grad_flat && stats8 &&
                   workspace && (returns || old_values),
               PB_ERR_INVALID, "pb_mlp_update_fused: null pointer");
    PB_REQUIRE(n_slabs == 1 || row_slab_stride >= slab_rows, PB_ERR_INVALID, "pb_mlp_update_fused: row slabs overlap");
    PB_REQUIRE(slab_rows >= 1 && n_slabs >= 1 && n_act >= 1 && n_act <= 7 && (!clip_vloss || old_values), PB_ERR_INVALID,
               "pb_mlp_update_fused: bad sizes (slab_rows %lld, n_slabs %d, n_act %d)", (long long)slab_rows, n_slabs, n_act);
    PB_REQUIRE(ldx >= FEAT && ldx % 4 == 0 && ((uintptr_t)x & 15) == 0 && ((uintptr_t)w_enc & 15) == 0, PB_ERR_INVALID,
               "pb_mlp_update_fused: x / w_enc must be 16-byte aligned, ldx a multiple of 4 floats");
    PB_REQUIRE(n_slabs == 1 || slab_stride_rows >= slab_rows, PB_ERR_INVALID, "pb_mlp_update_fused: slabs overlap");
    PB_REQUIRE(workspace_bytes >= pb_mlp_update_workspace_bytes(), PB_ERR_INVALID, "pb_mlp_update_fused: workspace too small");
    PB_REQUIRE(!dbg_hidden || dbg_dpre, PB_ERR_INVALID, "pb_mlp_update_fused: dbg_hidden needs dbg_dpre");
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    PB_REQUIRE(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) == cudaSuccess && fn &&
                   qr == cudaDriverEntryPointSuccess,
               PB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    const int64_t tiles_per_slab = (slab_rows + TILE_M - 1) / TILE_M;
    const int64_t n_tiles = tiles_per_slab * n_slabs;
    const int64_t map_rows = (int64_t)(n_slabs - 1) * slab_stride_rows + slab_rows;
    PB_REQUIRE(n_tiles <= 0x7FFFFFFF && map_rows <= 0x7FFFFFFF, PB_ERR_UNSUPPORTED, "pb_mlp_update_fused: too many rows");
    alignas(64) CUtensorMap map_x, map_w;
    int rc = make_map2((EncodeTiledFn)fn, &map_x, x, map_rows, ldx, TILE_M);
    if (rc == PB_OK) rc = make_map2((EncodeTiledFn)fn, &map_w, w_enc, HID, FEAT, HID);
    if (rc != PB_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int grid = n_tiles < num_sms() ? (int)n_tiles : num_sms();
    FusedParams p;
    p.actions = actions; p.old_logprobs = old_logprobs; p.adv = advantages; p.returns = returns; p.old_values = old_values;
    p.adv_norm = adv_norm; p.row_slab_stride = n_slabs > 1 ? row_slab_stride : slab_rows;
    p.m = slab_rows * n_slabs; p.slab_rows = slab_rows; p.slab_stride_rows = n_slabs > 1 ? slab_stride_rows : slab_rows;
    p.tiles_per_slab = (int)tiles_per_slab; p.n_tiles = (int)n_tiles; p.n_act = n_act;
    p.clip = clip_coef; p.vclip = vf_clip_coef; p.vf_coef = vf_coef; p.ent_coef = ent_coef; p.clip_vloss = clip_vloss;
    p.part_dw = (float*)workspace; p.part_tail = (float*)workspace + (size_t)num_sms() * FEAT * HID;
    p.w_heads = w_heads; p.b_enc = b_enc; p.b_heads = b_heads;
    p.stats = stats8; p.dpre_out = dpre_out; p.dbg_hidden = dbg_hidden; p.dbg_dpre = dbg_dpre; p.dbg_dout = dbg_dout;
    PB_CUDA(cudaMemsetAsync(stats8, 0, 8 * sizeof(double), s));
    static bool attr_set = false;
    if (!attr_set) {
        PB_CUDA(cudaFuncSetAttribute(k_mlp_update<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
        PB_CUDA(cudaFuncSetAttribute(k_mlp_update<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
        PB_CUDA(cudaFuncSetAttribute(k_mlp_update<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
        attr_set = true;
    }
    if (dpre_out) k_mlp_update<false, false><<<grid, THREADS, SMEM_TOTAL, s>>>(map_x, map_w, p);
    else if (g_update_variant == 2) k_mlp_update<true, true><<<grid, THREADS, SMEM_TOTAL, s>>>(map_x, map_w, p);
    else k_mlp_update<false, true><<<grid, THREADS, SMEM_TOTAL, s>>>(map_x, map_w, p);
    PB_LAUNCH_CHECK();
    k_update_reduce<<<REDUCE_BLOCKS, 256, 0, s>>>(dpre_out ? nullptr : p.part_dw, p.part_tail, grid, grad_flat,
                                                  reinterpret_cast<double*>((char*)workspace + pb_mlp_update_sumsq_offset()));
    PB_LAUNCH_CHECK();
    return PB_OK;
}
