// policy_sample.cuh -- pieces shared by every kernel that samples actions (policy_mlp.cu, policy_lstm.cu, sample.cu and
// the persistent rollout kernel of env_breakout.cu), with the tensor-core helpers of wgmma.cuh (to_tf32, mma_tf32):
//   * pb_policy_uniform: the counter-based uniform of a row, u = mix(seed, step counter, row) in [0, 1), 24 bits;
//   * pb_sample_row<NC>: one row's sampling epilogue over NC padded head outputs z[0..NC) = n_act logits | value | pad
//     (reference frameworks/cleanrl.py:25-47): lse = max z + log sum exp(z - max z), the probabilities
//     p_k = exp(z_k - lse) (softmax(normalized) of the reference), their running sums c_k and their total T = c_{n-1}.
//     The draw is the first k with u' < c_k.  For logits of ordinary size T is 1 up to the rounding of the p_k (a few
//     ulps) and u' = u.  When the logits share a large offset C, lse is rounded on the grid of ulp(C) and T misses 1 by
//     up to ulp(C)/2; that whole shortfall (or excess) would land on one action, so past |T - 1| > 2^-20 the draw
//     renormalises, u' = u*T, as torch.multinomial does with its weights.  The bias left below that bound is under 2^-20
//     of probability per row.  u <= 1 - 2^-24 gives fl(u*T) < T = the last running sum bit for bit, so the renormalised
//     draw always finds a k; otherwise (u >= T < 1, at most 2^-20 of the rows) it takes the last action with p_k > 0.
//     A zero-probability action is never drawn.  logprob = z_a - lse (the reference's normalized[a]);
//     entropy = -sum (p_k/T) * max(z_k - lse, -FLT_MAX) (cleanrl.entropy of softmax(normalized), -inf logits kept
//     finite as there).
//   * PbSampleOut and pb_sample_epilogue<NC>: the row outputs of the fused policy steps (policy_mlp.cu, policy_lstm.cu)
//     and the epilogue that fills them from a warp's head-product fragments and advances the stream counter.
#pragma once
#include "pb_common.cuh"
#include "wgmma.cuh"

__device__ __forceinline__ float pb_policy_uniform(uint64_t seed, uint64_t offset, int64_t row) {
    const uint32_t rnd = pb_mix32(seed * 0x9E3779B97F4A7C15ull + offset * 0xD1B54A32D192ED03ull +
                                  (uint64_t)row * 0x2545F4914F6CDD1Dull);
    return (float)(rnd >> 8) * (1.0f / 16777216.0f);
}

template <int NC>
__device__ __forceinline__ void pb_sample_row(const float (&z)[NC], int n_act, float u, int& action, float& logprob,
                                              float& entropy, float& value) {
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < NC; ++k) if (k < n_act) mx = fmaxf(mx, z[k]);
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < NC; ++k) if (k < n_act) sum += expf(z[k] - mx);
    const float lse = mx + logf(sum);
    float pk[NC];
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        pk[k] = k < n_act ? expf(z[k] - lse) : 0.f;
        tot += pk[k];                                  // the pad terms add exact zeros
    }
    const float uu = fabsf(tot - 1.f) > 0x1p-20f ? u * tot : u, inv = 1.f / tot;
    float cdf = 0.f, ent = 0.f, lp = 0.f, v = 0.f;
    int a = -1, last = 0;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        if (k < n_act) {
            const float nl = z[k] - lse;
            ent -= pk[k] * inv * fmaxf(nl, -3.4028234663852886e38f);
            cdf += pk[k];
            if (a < 0 && uu < cdf) { a = k; lp = nl; }
            if (pk[k] > 0.f) last = k;
        }
        if (k == n_act) v = z[k];
    }
    if (a < 0) {   // u >= T < 1 within the rounding of T: the last action with a non-zero probability
        a = last;
#pragma unroll
        for (int k = 0; k < NC; ++k) if (k == a) lp = z[k] - lse;    // static indices: z stays in registers
    }
    action = a;
    logprob = lp;
    entropy = ent;
    value = v;
}

// What a fused policy step writes: rows [0, m) of actions / logprobs / values (/ entropies), drawn with
// pb_policy_uniform(seed, *counter, row); with a ticket, the last CTA to leave advances *counter by one.
struct PbSampleOut {
    int64_t m; int n_act;
    uint64_t seed; uint64_t* counter; unsigned int* ticket;               // counter may be null (offset 0), ticket too
    int64_t* actions; float* logprobs; float* values; float* entropies;   // [m] each (entropies may be null)
};

// The sampling epilogue of a warp's 16 rows, called by every thread of the CTA.  out[q8] = (row g, cols 8q8 + 2t, +1),
// (row g + 8, same) of the head product, without its bias sBh[NC]; row = the global row of fragment row g; offset = the
// *counter every CTA read before it got here.  The NC columns of a row are gathered across its quad, lane t == 0
// finishes row g and lane t == 1 row g + 8.  Then the last CTA to leave advances the stream counter, so the host needs
// no separate "counter += 1" launch per env step.
template <int NC>
__device__ __forceinline__ void pb_sample_epilogue(const float (&out)[NC / 8][4], const float* sBh, const PbSampleOut& o,
                                                   int64_t row, uint64_t offset) {
    const int lane = threadIdx.x & 31, t = lane & 3;
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
        const int64_t r = row + 8 * t;
        if (r < o.m) {
            float z[NC];
#pragma unroll
            for (int k = 0; k < NC; ++k) z[k] = t ? rowv[1][k] : rowv[0][k];
            int a;
            float lp, ent, value;
            pb_sample_row<NC>(z, o.n_act, pb_policy_uniform(o.seed, offset, r), a, lp, ent, value);
            o.actions[r] = a;
            o.logprobs[r] = lp;
            o.values[r] = value;
            if (o.entropies) o.entropies[r] = ent;
        }
    }
    if (o.ticket) {
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            if (atomicAdd(o.ticket, 1u) == gridDim.x - 1) {
                *o.ticket = 0u;
                *o.counter = offset + 1ull;
                __threadfence();
            }
        }
    }
}
