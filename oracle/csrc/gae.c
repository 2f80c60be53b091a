/* Plain-C restatement of the reference's GAE recurrence.  TEST INFRASTRUCTURE (see oracle/__init__.py).
 *
 * Follows reference c_gae.pyx:11-32: one backward chain over the flat, (env_id, step)-sorted batch,
 * all arithmetic in C `float`, association exactly as written there:
 *     nextnonterminal = 1.0 - dones[t+1]
 *     delta       = rewards[t+1] + gamma * values[t+1] * nextnonterminal - values[t]
 *     lastgaelam  = delta + gamma * gae_lambda * nextnonterminal * lastgaelam
 * advantages[num_steps-1] stays 0.  Compiled without FMA contraction (-ffp-contract=off) like the
 * pyximport build of the reference (no -march flags => no fused multiply-add on x86-64).
 */
#include <stddef.h>

void oracle_compute_gae(const float* dones, const float* values, const float* rewards,
                        float gamma, float gae_lambda, float* advantages, long num_steps) {
    float lastgaelam = 0;
    float nextnonterminal, delta;
    if (num_steps <= 0) return;
    advantages[num_steps - 1] = 0.0f;
    for (long t = 0; t < num_steps - 1; t++) {
        long t_cur = num_steps - 2 - t;
        long t_next = num_steps - 1 - t;
        nextnonterminal = 1.0f - dones[t_next];
        delta = rewards[t_next] + gamma * values[t_next] * nextnonterminal - values[t_cur];
        lastgaelam = delta + gamma * gae_lambda * nextnonterminal * lastgaelam;
        advantages[t_cur] = lastgaelam;
    }
}

/* The same recurrence in double: ground truth that puts the reference's fp32 rounding and the CUDA scan's
 * rounding on one scale in the tolerance tests (gamma / lambda are the fp32 values widened, like the C floats). */
void oracle_compute_gae_f64(const float* dones, const float* values, const float* rewards, float gamma,
                            float gae_lambda, double* advantages, long num_steps) {
    double last = 0.0, g = (double)gamma, l = (double)gae_lambda;
    if (num_steps <= 0) return;
    advantages[num_steps - 1] = 0.0;
    for (long t = num_steps - 2; t >= 0; t--) {
        double nnt = 1.0 - (double)dones[t + 1];
        double delta = (double)rewards[t + 1] + g * (double)values[t + 1] * nnt - (double)values[t];
        last = delta + g * l * nnt * last;
        advantages[t] = last;
    }
}
