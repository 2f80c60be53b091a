// sample.cu -- fused categorical sampling epilogue for one Discrete head (sm_90a).
//
// Replaces, for the sampling case, reference pufferlib/frameworks/cleanrl.py:25-47 (sample_logits):
//   normalized = logits - logsumexp(logits);  action ~ multinomial(softmax(normalized));
//   logprob = normalized[action];  entropy = -sum(softmax * normalized)          (cleanrl.py:12-23)
// and, optionally, the policy-output part of Experience.store (clean_pufferl.py:443-446) by writing action /
// logprob / value straight into their rollout rows.  One thread per row (n_act is 1..32, a row is 4..128 B); the ~8
// ATen launches of the reference become one.
// The row's epilogue is pb_sample_row (policy_sample.cuh), the one the fused policy kernels use: inverse CDF,
// renormalised when lse was rounded on a coarse grid, with the counter-based uniform u = pb_policy_uniform(seed, offset
// (+ *offset_dev), row).  Reproducible, but not the same stream as torch.multinomial -- action sampling is not a parity
// surface (parity runs feed an action tape, SURVEY §8c-4).
#include "pb_common.cuh"
#include "policy_sample.cuh"

namespace {

constexpr int MAX_ACT = 32;

// NC: the logit registers of a row, 8, 16 or MAX_ACT (the smallest that holds n_act): at NC = MAX_ACT the logits and
// their weights take 64 registers, so the narrower rows get instances of their own
template <int NC>
__global__ void __launch_bounds__(256) k_sample_logits(const float* __restrict__ logits, int64_t lstride, int64_t n, int n_act,
                                                      uint64_t seed, uint64_t offset, const uint64_t* __restrict__ offset_dev,
                                                      int64_t* actions, float* logprobs, float* entropies, const float* value, int64_t vstride,
                                                      float* values_row, float* logprobs_row, int64_t* actions_row) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float l[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) l[k] = k < n_act ? logits[i * lstride + k] : 0.f;
    if (offset_dev) offset += *offset_dev;
    int a;
    float lp_a, ent, unused_value;
    pb_sample_row<NC>(l, n_act, pb_policy_uniform(seed, offset, i), a, lp_a, ent, unused_value);
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
    const unsigned blocks = (unsigned)pb_ceil_div(n, 256);
    cudaStream_t s = (cudaStream_t)stream;
    if (n_act <= 8)
        k_sample_logits<8><<<blocks, 256, 0, s>>>(logits, logits_stride, n, n_act, seed, offset, offset_dev, actions, logprobs,
                                                  entropies, value, value_stride, values_row, logprobs_row, actions_row);
    else if (n_act <= 16)
        k_sample_logits<16><<<blocks, 256, 0, s>>>(logits, logits_stride, n, n_act, seed, offset, offset_dev, actions, logprobs,
                                                   entropies, value, value_stride, values_row, logprobs_row, actions_row);
    else
        k_sample_logits<MAX_ACT><<<blocks, 256, 0, s>>>(logits, logits_stride, n, n_act, seed, offset, offset_dev, actions,
                                                        logprobs, entropies, value, value_stride, values_row, logprobs_row,
                                                        actions_row);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
