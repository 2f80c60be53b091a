// sample.cu -- fused categorical sampling epilogue for one Discrete head (sm_90a).
//
// Replaces, for the sampling case, reference pufferlib/frameworks/cleanrl.py:25-47 (sample_logits):
//   normalized = logits - logsumexp(logits);  action ~ multinomial(softmax(normalized));
//   logprob = normalized[action];  entropy = -sum(softmax * normalized)          (cleanrl.py:12-23)
// and, optionally, the policy-output part of Experience.store (clean_pufferl.py:443-446) by writing action /
// logprob / value straight into their rollout rows.  One thread per row (n_act is 4..18 on this path, a row is
// 16..72 B, so a warp reads a contiguous 0.5..2.3 KB span); the ~8 ATen launches of the reference become one.
// Sampling uses inverse-CDF on a counter-based uniform (seed, offset, row): reproducible, but not the same stream
// as torch.multinomial -- action sampling is not a parity surface (parity runs feed an action tape, SURVEY §8c-4).
#include "pb_common.cuh"

namespace {

constexpr int MAX_ACT = 32;

__global__ void __launch_bounds__(256) k_sample_logits(const float* __restrict__ logits, int64_t lstride, int64_t n, int n_act,
                                                      uint64_t seed, uint64_t offset, const uint64_t* __restrict__ offset_dev,
                                                      int64_t* actions, float* logprobs, float* entropies, const float* value, int64_t vstride,
                                                      float* values_row, float* logprobs_row, int64_t* actions_row) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float l[MAX_ACT];
    float m = -INFINITY;
#pragma unroll
    for (int k = 0; k < MAX_ACT; ++k)
        if (k < n_act) { l[k] = logits[i * lstride + k]; m = fmaxf(m, l[k]); }
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < MAX_ACT; ++k)
        if (k < n_act) sum += expf(l[k] - m);
    const float lse = m + logf(sum);
    // uniform in [0,1) from the counter-based generator; inverse CDF over the probabilities
    if (offset_dev) offset += *offset_dev;
    const uint32_t r = pb_mix32(seed * 0x9E3779B97F4A7C15ull + offset * 0xD1B54A32D192ED03ull + (uint64_t)i * 0x2545F4914F6CDD1Dull);
    const float u = (float)(r >> 8) * (1.0f / 16777216.0f);
    float cdf = 0.f, ent = 0.f, lp_a = 0.f;
    int a = -1;
#pragma unroll
    for (int k = 0; k < MAX_ACT; ++k) {
        if (k < n_act) {
            const float nl = l[k] - lse;
            const float pk = expf(nl);
            ent -= pk * fmaxf(nl, -3.4028234663852886e38f);
            cdf += pk;
            if (a < 0 && u < cdf) { a = k; lp_a = nl; }
        }
    }
    if (a < 0) {  // rounding left cdf a hair below u: take the last action with non-zero probability
        for (int k = n_act - 1; k >= 0; --k)
            if (l[k] - lse > -80.f) { a = k; lp_a = l[k] - lse; break; }
        if (a < 0) { a = n_act - 1; lp_a = l[a] - lse; }
    }
    if (actions) actions[i] = a;
    if (logprobs) logprobs[i] = lp_a;
    if (entropies) entropies[i] = ent;
    if (actions_row) actions_row[i] = a;
    if (logprobs_row) logprobs_row[i] = lp_a;
    if (values_row && value) values_row[i] = value[i * vstride];
}

}  // namespace

extern "C" int pb_sample_logits(const float* logits, int64_t logits_stride, int64_t n, int32_t n_act, uint64_t seed,
                                uint64_t offset, const uint64_t* offset_dev, int64_t* actions, float* logprobs,
                                float* entropies, const float* value, int64_t value_stride,
                                float* values_row, float* logprobs_row, int64_t* actions_row, void* stream) {
    PB_REQUIRE(n >= 0, PB_ERR_INVALID, "pb_sample_logits: negative n");
    if (n == 0) return PB_OK;
    PB_REQUIRE(logits, PB_ERR_INVALID, "pb_sample_logits: null logits");
    PB_REQUIRE(n_act >= 1 && n_act <= MAX_ACT, PB_ERR_UNSUPPORTED, "pb_sample_logits: n_act must be in [1, %d]", MAX_ACT);
    PB_REQUIRE(!values_row || value, PB_ERR_INVALID, "pb_sample_logits: values_row given without value");
    PB_REQUIRE(logits_stride >= n_act, PB_ERR_INVALID, "pb_sample_logits: logits_stride < n_act");
    k_sample_logits<<<(unsigned)pb_ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(
        logits, logits_stride, n, n_act, seed, offset, offset_dev, actions, logprobs, entropies, value, value_stride,
        values_row, logprobs_row, actions_row);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
