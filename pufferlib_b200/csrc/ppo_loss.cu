// ppo_loss.cu -- the PPO minibatch loss of clean_pufferl.train, forward AND backward, in one pass (sm_90a).
//
// Replaces reference clean_pufferl.py:202-238 plus the action-given branch of sample_logits
// (reference pufferlib/frameworks/cleanrl.py:25-47) for one Discrete head:
//     normalized = logits - logsumexp(logits);  newlogprob = normalized[action];  entropy = -sum(p * normalized)
//     logratio = newlogprob - old_logprob;  ratio = exp(logratio)
//     old_approx_kl = mean(-logratio);  approx_kl = mean((ratio - 1) - logratio);  clipfrac = mean(|ratio - 1| > clip)
//     pg_loss = mean(max(-adv * ratio, -adv * clamp(ratio, 1 - clip, 1 + clip)))
//     v_loss  = 0.5 * mean(max((v - ret)^2, (old_v + clamp(v - old_v, -vclip, vclip) - ret)^2))   (or unclipped)
//     loss    = pg_loss - ent_coef * mean(entropy) + vf_coef * v_loss
// In the reference these are ~40 ATen elementwise / reduction launches forward and ~60 backward per minibatch, each
// moving a few MB; here one thread per row reads logits / value / action / old logprob / advantage / return / old
// value once, accumulates the 7 means (warp shuffle -> block -> one atomic per block and statistic, fp64) and writes
// the ANALYTIC gradients dloss/dlogits and dloss/dvalue (already scaled by 1/M), which the host feeds to autograd
// for the network backward.  Tie rules follow ATen (maximum: ties split the gradient; clamp: inclusive bounds).
// HBM traffic per row: 4*A + 28 B read, 4*A + 4 B written.
#include "pb_common.cuh"

namespace {

constexpr int PL_MAX_ACT = 32;
constexpr int PL_THREADS = 256;

struct PpoParams {
    const float* logits; int64_t lstride;
    const float* value; int64_t vstride;
    const int64_t* actions;
    const float* old_logprobs;
    const float* adv;
    const float* returns;
    const float* old_values;
    float* grad_logits; int64_t glstride;
    float* grad_value; int64_t gvstride;
    double* stats;   // [8]: sum pg, sum v (before the 0.5), sum entropy, sum -logratio, sum (ratio-1)-logratio, sum clipped, unused, unused
    int64_t m;
    int n_act;
    float clip, vclip, vf_coef, ent_coef;
    int clip_vloss;
};

// PACKED: logits / value / grads all live in [m][8] rows (n_act logits | value | zero pad): 128-bit row accesses
template <bool PACKED>
__global__ void __launch_bounds__(PL_THREADS) k_ppo_loss(PpoParams p) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double s_pg = 0, s_v = 0, s_ent = 0, s_okl = 0, s_kl = 0, s_clip = 0;
    if (i < p.m) {
        float z[PL_MAX_ACT];
        float mx = -INFINITY;
        float v_packed = 0.f;
        if (PACKED) {   // one 32-byte row: two 128-bit loads
            const float4 a0 = *reinterpret_cast<const float4*>(p.logits + i * 8);
            const float4 a1 = *reinterpret_cast<const float4*>(p.logits + i * 8 + 4);
            const float row[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                z[k] = row[k];
                if (k == p.n_act) v_packed = row[k];
            }
        }
#pragma unroll
        for (int k = 0; k < PL_MAX_ACT; ++k)
            if (k < p.n_act) {
                if (!PACKED) z[k] = p.logits[i * p.lstride + k];
                mx = fmaxf(mx, z[k]);
            }
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < PL_MAX_ACT; ++k)
            if (k < p.n_act) sum += expf(z[k] - mx);
        const float lse = mx + logf(sum);
        int a = (int)p.actions[i];
        a = a < 0 ? 0 : (a >= p.n_act ? p.n_act - 1 : a);
        float ent = 0.f, nl_a = 0.f;
#pragma unroll
        for (int k = 0; k < PL_MAX_ACT; ++k)
            if (k < p.n_act) {
                const float nl = z[k] - lse, pk = expf(nl);
                ent -= pk * nl;
                if (k == a) nl_a = nl;
                z[k] = nl;   // keep the normalised logit
            }
        const float logratio = nl_a - p.old_logprobs[i];
        const float ratio = expf(logratio);
        const float adv = p.adv[i];
        const float pg1 = -adv * ratio;
        const float rc = fminf(fmaxf(ratio, 1.f - p.clip), 1.f + p.clip);
        const float pg2 = -adv * rc;
        const float pg = fmaxf(pg1, pg2);
        // d pg / d ratio: maximum() sends the gradient to the larger branch, ties split it; clamp passes the gradient
        // inside [1-clip, 1+clip] (inclusive) and blocks it outside
        const float in_range = (ratio >= 1.f - p.clip && ratio <= 1.f + p.clip) ? 1.f : 0.f;
        float g_ratio;
        if (pg1 > pg2) g_ratio = -adv;
        else if (pg1 < pg2) g_ratio = -adv * in_range;
        else g_ratio = 0.5f * (-adv) + 0.5f * (-adv * in_range);
        const float inv_m = 1.0f / (float)p.m;
        const float g_nlp = g_ratio * ratio * inv_m;          // d loss / d newlogprob
        // value loss
        const float v = PACKED ? v_packed : p.value[i * p.vstride], ret = p.returns[i];
        const float dv = v - ret;
        float vl, g_v;
        if (p.clip_vloss) {
            const float ov = p.old_values[i];
            const float d = v - ov;
            const float dc = fminf(fmaxf(d, -p.vclip), p.vclip);
            const float vc = ov + dc;
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
        if (!PACKED) p.grad_value[i * p.gvstride] = gv_out;
        // d loss / d logits_j = g_nlp * (delta_ja - p_j) + ent_coef/M * p_j * (nl_j + H)
        const float g_ent = p.ent_coef * inv_m;
        float gro[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < PL_MAX_ACT; ++k)
            if (k < p.n_act) {
                const float pk = expf(z[k]);
                const float gk = g_nlp * ((k == a ? 1.f : 0.f) - pk) + g_ent * pk * (z[k] + ent);
                if (PACKED) { if (k < 8) gro[k] = gk; }
                else p.grad_logits[i * p.glstride + k] = gk;
            }
        if (PACKED) {   // the whole 8-column gradient row (zero padding included) in two 128-bit stores
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (k == p.n_act) gro[k] = gv_out;
            *reinterpret_cast<float4*>(p.grad_logits + i * 8) = make_float4(gro[0], gro[1], gro[2], gro[3]);
            *reinterpret_cast<float4*>(p.grad_logits + i * 8 + 4) = make_float4(gro[4], gro[5], gro[6], gro[7]);
        }
        s_pg = pg; s_v = vl; s_ent = ent; s_okl = -logratio; s_kl = (ratio - 1.f) - logratio;
        s_clip = fabsf(ratio - 1.f) > p.clip ? 1.0 : 0.0;
    }
    // block reduction of the six sums (fp64), one atomic per block and statistic
    __shared__ double sh[6][PL_THREADS / 32];
    double vals[6] = {s_pg, s_v, s_ent, s_okl, s_kl, s_clip};
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        double x = vals[q];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
        if ((threadIdx.x & 31) == 0) sh[q][threadIdx.x >> 5] = x;
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        double t = 0;
        for (int w = 0; w < PL_THREADS / 32; ++w) t += sh[threadIdx.x][w];
        atomicAdd(p.stats + threadIdx.x, t);
    }
}

}  // namespace

extern "C" int pb_ppo_loss(const float* logits, int64_t logits_stride, const float* value, int64_t value_stride,
                           const int64_t* actions, const float* old_logprobs, const float* advantages,
                           const float* returns, const float* old_values, int64_t m, int32_t n_act, float clip_coef,
                           int32_t clip_vloss, float vf_clip_coef, float vf_coef, float ent_coef, float* grad_logits,
                           int64_t grad_logits_stride, float* grad_value, int64_t grad_value_stride, double* stats8,
                           void* stream) {
    PB_REQUIRE(m >= 1, PB_ERR_INVALID, "pb_ppo_loss: m must be positive");
    PB_REQUIRE(n_act >= 1 && n_act <= PL_MAX_ACT, PB_ERR_UNSUPPORTED, "pb_ppo_loss: n_act must be in [1, %d]", PL_MAX_ACT);
    PB_REQUIRE(logits && value && actions && old_logprobs && advantages && returns && grad_logits && grad_value && stats8,
               PB_ERR_INVALID, "pb_ppo_loss: null pointer");
    PB_REQUIRE(!clip_vloss || old_values, PB_ERR_INVALID, "pb_ppo_loss: clip_vloss needs old_values");
    PB_REQUIRE(logits_stride >= n_act && grad_logits_stride >= n_act && value_stride >= 1 && grad_value_stride >= 1,
               PB_ERR_INVALID, "pb_ppo_loss: bad strides");
    cudaStream_t s = (cudaStream_t)stream;
    PB_CUDA(cudaMemsetAsync(stats8, 0, 8 * sizeof(double), s));
    PpoParams p{logits, logits_stride, value, value_stride, actions, old_logprobs, advantages, returns, old_values,
                grad_logits, grad_logits_stride, grad_value, grad_value_stride, stats8, m, n_act, clip_coef, vf_clip_coef,
                vf_coef, ent_coef, clip_vloss};
    // packed rows: logits, value, and both gradients share [m][8] buffers (value = column n_act of the logits rows)
    const bool packed = logits_stride == 8 && grad_logits_stride == 8 && n_act <= 7 && value == logits + n_act &&
                        value_stride == 8 && grad_value == grad_logits + n_act && grad_value_stride == 8 &&
                        ((uintptr_t)logits & 15) == 0 && ((uintptr_t)grad_logits & 15) == 0;
    if (packed) k_ppo_loss<true><<<(unsigned)pb_ceil_div(m, PL_THREADS), PL_THREADS, 0, s>>>(p);
    else k_ppo_loss<false><<<(unsigned)pb_ceil_div(m, PL_THREADS), PL_THREADS, 0, s>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
