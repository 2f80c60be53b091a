// policy_sample.cuh -- pieces shared by the fused rollout-time policy kernels (policy_mlp.cu, policy_lstm.cu):
//   * to_tf32 / mma_tf32: round-to-nearest TF32 conversion (cvt.rna) and the mma.sync m16n8k8 TF32 tile product;
//   * pb_policy_uniform: the counter-based uniform of a row, u = mix(seed, step counter, row) in [0, 1), 24 bits;
//   * pb_sample_row<NC>: one row's sampling epilogue over NC padded head outputs z[0..NC) = n_act logits | value | pad:
//     logsumexp, the inverse CDF (first k with u < cdf_k), the fallback when rounding leaves cdf_{n_act-1} below u,
//     logprob of the sampled action and the entropy (reference frameworks/cleanrl.py:25-47).
// The bits of pb_sample_row<8> are those of the epilogue pb_policy_mlp_sample had before it moved here.
#pragma once
#include "pb_common.cuh"

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
    float cdf = 0.f, ent = 0.f, lp = 0.f, v = 0.f;
    int a = -1;
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        if (k < n_act) {
            const float nl = z[k] - lse, pk = expf(nl);
            ent -= pk * nl;
            cdf += pk;
            if (a < 0 && u < cdf) { a = k; lp = nl; }
        }
        if (k == n_act) v = z[k];
    }
    if (a < 0) {   // rounding left cdf a hair below u: last action with non-negligible probability
#pragma unroll
        for (int k = NC - 1; k >= 0; --k)
            if (a < 0 && k < n_act && z[k] - lse > -80.f) { a = k; lp = z[k] - lse; }
        if (a < 0) {
            a = n_act - 1;
#pragma unroll
            for (int k = 0; k < NC; ++k) if (k == a) lp = z[k] - lse;    // static indices: z stays in registers
        }
    }
    action = a;
    logprob = lp;
    entropy = ent;
    value = v;
}
