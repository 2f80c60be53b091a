// optim.cu -- the optimizer step of clean_pufferl.train for small policies, ONE launch (sm_90a).
//
// Replaces reference clean_pufferl.py:240-244
//     torch.nn.utils.clip_grad_norm_(policy.parameters(), max_grad_norm);  optimizer.step()      (Adam, eps 1e-5)
// which for the 17k-parameter models.Default is ~12 short launches per minibatch (multi-tensor L2 norms,
// cleanup, reciprocal / clamp / multiply, fused Adam): latency, not work.  Here a single 1024-thread CTA makes two
// passes over the gradients (<= 1 M elements): global L2 norm -> clip coefficient, then the Adam update with the
// bias corrections of torch.optim.Adam(capturable=True): step counters, moments and parameters are the optimizer's
// own state tensors, updated in place, so state_dict() and a later fall-back to optimizer.step() stay valid.
//
// pb_pack_heads builds the 8-row head matrix (n_act logit rows | value row | zero pad) that the fused forward, the
// rollout-time policy kernel and pb_mlp_tail_backward consume, plus the TF32-rounded encoder weight, in one launch
// (the ATen formulation is 2 fills + 4 strided copies + 3 elementwise kernels per optimizer step).
#include "pb_common.cuh"
#include "peer.cuh"

namespace {

constexpr int CA_THREADS = 1024;
constexpr int CA_MAX_TENSORS = 8;

struct AdamArgs {
    pb_adam_tensor t[CA_MAX_TENSORS];
    int n;
    float max_norm, grad_scale, lr;
    const float* lr_dev;
    float beta1, beta2, eps;
    float* total_norm_out;
    pb_peer_comm peer;      // world <= 1: no exchange
    float* flat;            // the flat gradient buffer all `grad` pointers lie in (peer exchange only)
    int64_t flat_n;
};

__global__ void __launch_bounds__(CA_THREADS) k_clip_adam(AdamArgs a) {
    __shared__ double s_red[CA_THREADS / 32];
    __shared__ float s_coef;
    __shared__ float s_step_size[CA_MAX_TENSORS], s_bc2_sqrt[CA_MAX_TENSORS];
    const int tid = threadIdx.x;

    // ---- multi-GPU: sum the flat gradient buffer over all ranks through NVLink peer memory (peer.cuh)
    if (a.peer.world > 1) pb_peer_allreduce_sum(a.peer, a.flat, a.flat_n);

    // ---- pass 1: global L2 norm of the (scaled) gradients
    float ss = 0.f;
    for (int k = 0; k < a.n; ++k) {
        const float* g = a.t[k].grad;
        for (int64_t i = tid; i < a.t[k].numel; i += CA_THREADS) {
            const float x = g[i] * a.grad_scale;
            ss += x * x;
        }
    }
    double d = (double)ss;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
    if ((tid & 31) == 0) s_red[tid >> 5] = d;
    __syncthreads();
    if (tid == 0) {
        double tot = 0.0;
        for (int w = 0; w < CA_THREADS / 32; ++w) tot += s_red[w];
        const float norm = (float)sqrt(tot);
        // clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1 (max_norm <= 0: no clipping)
        float coef = 1.f;
        if (a.max_norm > 0.f) coef = fminf(a.max_norm / (norm + 1e-6f), 1.f);
        s_coef = coef * a.grad_scale;
        if (a.total_norm_out) *a.total_norm_out = norm;
    }
    // ---- step counters and bias corrections (torch.optim.Adam: step += 1 first; double math like ATen's fused kernel)
    if (tid < a.n) {
        const float step = *a.t[tid].step + 1.f;
        const double lr = a.lr_dev ? (double)*a.lr_dev : (double)a.lr;
        const double bc1 = 1.0 - pow((double)a.beta1, (double)step);
        const double bc2 = 1.0 - pow((double)a.beta2, (double)step);
        s_step_size[tid] = (float)(lr / bc1);
        s_bc2_sqrt[tid] = (float)sqrt(bc2);
        *a.t[tid].step = step;
    }
    __syncthreads();
    const float coef = s_coef;
    const float w1 = 1.f - a.beta1, w2 = 1.f - a.beta2;

    // ---- pass 2: Adam
    for (int k = 0; k < a.n; ++k) {
        const float* g = a.t[k].grad;
        float* p = a.t[k].param;
        float* m = a.t[k].exp_avg;
        float* v = a.t[k].exp_avg_sq;
        const float step_size = s_step_size[k], bc2_sqrt = s_bc2_sqrt[k];
        for (int64_t i = tid; i < a.t[k].numel; i += CA_THREADS) {
            const float x = g[i] * coef;
            const float mi = m[i] + w1 * (x - m[i]);                  // lerp(exp_avg, grad, 1 - beta1)
            const float vi = a.beta2 * v[i] + w2 * x * x;
            const float denom = sqrtf(vi) / bc2_sqrt + a.eps;
            m[i] = mi;
            v[i] = vi;
            p[i] -= step_size * mi / denom;
        }
    }
}

// Multi-CTA form for callers that already hold the gradient's sum of squares as partial sums (k_update_reduce of the fused
// update, or the sliced peer all-reduce): no norm pass, every CTA sums the partials in the same fixed order, then updates
// its share of the elements.  The step counters are advanced by the LAST CTA to finish (all others have read them).
constexpr int CAP_BLOCKS = 32;
// (one optimizer step in flight per device: the counters below are module-wide, like the trainer that owns the stream)
__device__ unsigned int g_cap_ticket = 0;

// PEER: the sliced NVLink all-reduce of the flat gradient (peer.cuh) runs first in the same kernel -- one CTA per slice, a grid
// barrier among the PB_PEER_SLICES co-resident CTAs, then clip + Adam: one launch per optimizer step for any world size.
__device__ unsigned int g_gb_count = 0;
__device__ volatile unsigned int g_gb_gen = 0;

template <int CAP_THREADS, bool PEER>
__global__ void __launch_bounds__(CAP_THREADS) k_clip_adam_parts(AdamArgs a, const double* __restrict__ parts, int n_parts,
                                                                unsigned long long* peer_epoch, pb_head_pack pack,
                                                                double* peer_parts) {
    __shared__ int s_last;
    __shared__ double s_red[CAP_THREADS / 32];
    if (PEER) {
        pb_peer_allreduce_slice(a.peer, a.flat, a.flat_n, peer_parts);       // flat slice summed over the ranks + its sum of squares
        __syncthreads();
        if (threadIdx.x == 0) {          // grid barrier: every slice and every partial sum is in global memory
            __threadfence();
            const unsigned int gen = g_gb_gen;
            if (atomicAdd(&g_gb_count, 1u) == gridDim.x - 1) {
                g_gb_count = 0;
                __threadfence();
                g_gb_gen = gen + 1;
            } else {
                const long long t0 = clock64();
                while (g_gb_gen == gen)
                    if (clock64() - t0 > 20000000000ll) __trap();
            }
            __threadfence();
        }
        __syncthreads();
        parts = peer_parts;
        n_parts = (int)gridDim.x;
    }
    __shared__ float s_coef;
    __shared__ float s_step_size[CA_MAX_TENSORS], s_bc2_sqrt[CA_MAX_TENSORS], s_new_step[CA_MAX_TENSORS];
    __shared__ int64_t s_first[CA_MAX_TENSORS + 1];
    const int tid = threadIdx.x;
    double d = 0.0;
    for (int i = tid; i < n_parts; i += CAP_THREADS) d += PEER ? ((volatile const double*)parts)[i] : parts[i];   // fixed assignment and order: same bits in every CTA
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
    if ((tid & 31) == 0) s_red[tid >> 5] = d;
    if (tid == 0) {
        int64_t acc = 0;
        for (int k = 0; k < a.n; ++k) { s_first[k] = acc; acc += a.t[k].numel; }
        s_first[a.n] = acc;
    }
    __syncthreads();
    if (tid == 0) {
        double tot = 0.0;
        for (int w = 0; w < CAP_THREADS / 32; ++w) tot += s_red[w];
        const float norm = (float)sqrt(tot) * a.grad_scale;                   // partials are of the unscaled (summed) gradient
        float coef = 1.f;
        if (a.max_norm > 0.f) coef = fminf(a.max_norm / (norm + 1e-6f), 1.f);
        s_coef = coef * a.grad_scale;
        if (a.total_norm_out && blockIdx.x == 0) *a.total_norm_out = norm;
    }
    if (tid < a.n) {
        const float step = *a.t[tid].step + 1.f;
        const double lr = a.lr_dev ? (double)*a.lr_dev : (double)a.lr;
        const double bc1 = 1.0 - pow((double)a.beta1, (double)step);
        const double bc2 = 1.0 - pow((double)a.beta2, (double)step);
        s_step_size[tid] = (float)(lr / bc1);
        s_bc2_sqrt[tid] = (float)sqrt(bc2);
        s_new_step[tid] = step;
    }
    __syncthreads();
    const float coef = s_coef;
    const float w1 = 1.f - a.beta1, w2 = 1.f - a.beta2;
    const int64_t total = s_first[a.n];
    for (int64_t j = (int64_t)blockIdx.x * CAP_THREADS + tid; j < total; j += (int64_t)gridDim.x * CAP_THREADS) {
        int k = 0;
        while (j >= s_first[k + 1]) ++k;
        const int64_t i = j - s_first[k];
        // PEER: the summed gradient was written by other CTAs of this launch: read it from L2 (an L1 line fetched while copying
        // this CTA's own slice may hold the neighbouring slice's pre-exchange values)
        const float x = (PEER ? __ldcg(a.t[k].grad + i) : a.t[k].grad[i]) * coef;
        float* m = a.t[k].exp_avg;
        float* v = a.t[k].exp_avg_sq;
        const float mi = m[i] + w1 * (x - m[i]);                  // lerp(exp_avg, grad, 1 - beta1)
        const float vi = a.beta2 * v[i] + w2 * x * x;
        const float denom = sqrtf(vi) / s_bc2_sqrt[k] + a.eps;
        m[i] = mi;
        v[i] = vi;
        a.t[k].param[i] -= s_step_size[k] * mi / denom;
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        const unsigned int t = atomicAdd(&g_cap_ticket, 1u);
        s_last = t == gridDim.x - 1;
        if (s_last) {                    // every CTA has read the step counters (and the peer epoch is no longer in use)
            for (int k = 0; k < a.n; ++k) *a.t[k].step = s_new_step[k];
            if (peer_epoch) *peer_epoch += 1ull;
            g_cap_ticket = 0;
        }
    }
    __syncthreads();
    if (s_last && pack.w_cat) {          // the last CTA sees every CTA's parameter updates: rebuild the 8-row head matrix (pb_pack_heads)
        __threadfence();
        for (int j = tid; j < 8 * pack.hid; j += CAP_THREADS) {
            const int r = j / pack.hid, c = j % pack.hid;
            pack.w_cat[j] = r < pack.n_act ? pack.w_dec[(int64_t)r * pack.hid + c] : (r == pack.n_act ? pack.w_val[c] : 0.f);
        }
        if (tid < 8) pack.b_cat[tid] = tid < pack.n_act ? pack.b_dec[tid] : (tid == pack.n_act ? pack.b_val[0] : 0.f);
    }
}

__global__ void __launch_bounds__(256) k_pack_heads(const float* __restrict__ w_dec, const float* __restrict__ b_dec,
                                                    const float* __restrict__ w_val, const float* __restrict__ b_val,
                                                    int n_act, int hid, float* __restrict__ w_cat,
                                                    float* __restrict__ b_cat, const float* __restrict__ w_enc,
                                                    float* __restrict__ w_enc_tf32, int64_t enc_numel) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = i; j < 8 * (int64_t)hid; j += stride) {
        const int r = (int)(j / hid), c = (int)(j % hid);
        w_cat[j] = r < n_act ? w_dec[(int64_t)r * hid + c] : (r == n_act ? w_val[c] : 0.f);
    }
    if (i < 8) b_cat[i] = i < n_act ? b_dec[i] : (i == n_act ? b_val[0] : 0.f);
    if (w_enc_tf32)
        for (int64_t j = i; j < enc_numel; j += stride) {   // cvt.rna.tf32.f32: round to nearest, ties away from zero
            uint32_t r;
            asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(w_enc[j]));
            w_enc_tf32[j] = __uint_as_float(r);
        }
}

}  // namespace

extern "C" int pb_clip_adam(const pb_adam_tensor* tensors, int32_t n_tensors, float max_grad_norm, float grad_scale,
                            float lr, const float* lr_dev, float beta1, float beta2, float eps, float* total_norm_out,
                            void* stream) {
    return pb_clip_adam_peer(tensors, n_tensors, max_grad_norm, grad_scale, lr, lr_dev, beta1, beta2, eps, total_norm_out,
                             nullptr, nullptr, 0, stream);
}

extern "C" int pb_clip_adam_peer(const pb_adam_tensor* tensors, int32_t n_tensors, float max_grad_norm, float grad_scale,
                                 float lr, const float* lr_dev, float beta1, float beta2, float eps, float* total_norm_out,
                                 const pb_peer_comm* comm, float* grad_flat, int64_t grad_flat_numel, void* stream) {
    PB_REQUIRE(tensors && n_tensors >= 1 && n_tensors <= CA_MAX_TENSORS, PB_ERR_INVALID,
               "pb_clip_adam: 1..%d tensors", CA_MAX_TENSORS);
    AdamArgs a{};
    int64_t total = 0;
    for (int k = 0; k < n_tensors; ++k) {
        const pb_adam_tensor& t = tensors[k];
        PB_REQUIRE(t.param && t.exp_avg && t.exp_avg_sq && t.step && t.grad && t.numel >= 1, PB_ERR_INVALID,
                   "pb_clip_adam: tensor %d has a null pointer or no elements", k);
        a.t[k] = t;
        total += t.numel;
    }
    PB_REQUIRE(total <= (1 << 20), PB_ERR_UNSUPPORTED,
               "pb_clip_adam: single-CTA kernel for small policies (%lld parameters > 1 Mi)", (long long)total);
    PB_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f && grad_scale > 0.f,
               PB_ERR_INVALID, "pb_clip_adam: bad hyper-parameters");
    a.n = n_tensors;
    a.max_norm = max_grad_norm;
    a.grad_scale = grad_scale;
    a.lr = lr;
    a.lr_dev = lr_dev;
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.total_norm_out = total_norm_out;
    if (comm && comm->world > 1) {
        PB_REQUIRE(comm->world <= PB_PEER_MAX_RANKS && comm->rank >= 0 && comm->rank < comm->world && comm->epoch &&
                       grad_flat && grad_flat_numel >= 1 && grad_flat_numel <= comm->capacity,
                   PB_ERR_INVALID, "pb_clip_adam_peer: bad communicator or flat gradient buffer");
        for (int r = 0; r < comm->world; ++r) PB_REQUIRE(comm->base[r], PB_ERR_INVALID, "pb_clip_adam_peer: peer %d not mapped", r);
        for (int k = 0; k < n_tensors; ++k)
            PB_REQUIRE(tensors[k].grad >= grad_flat && tensors[k].grad + tensors[k].numel <= grad_flat + grad_flat_numel,
                       PB_ERR_INVALID, "pb_clip_adam_peer: gradient %d lies outside the flat buffer", k);
        a.peer = *comm;
        a.flat = grad_flat;
        a.flat_n = grad_flat_numel;
    }
    k_clip_adam<<<1, CA_THREADS, 0, (cudaStream_t)stream>>>(a);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

// pb_clip_adam for callers that hold the sum of squares of the (already summed over ranks, unscaled) gradient as n_parts
// partial sums: the reduce step of pb_mlp_update_fused (pb_mlp_update_sumsq_offset / _parts) or pb_peer_allreduce_parts.
// peer_epoch (nullable): the communicator's epoch counter, advanced here after pb_peer_allreduce_parts.
extern "C" int pb_clip_adam_parts(const pb_adam_tensor* tensors, int32_t n_tensors, float max_grad_norm, float grad_scale,
                                  float lr, const float* lr_dev, float beta1, float beta2, float eps, float* total_norm_out,
                                  const double* sumsq_parts, int32_t n_parts, unsigned long long* peer_epoch,
                                  const pb_head_pack* pack, void* stream) {
    PB_REQUIRE(tensors && n_tensors >= 1 && n_tensors <= CA_MAX_TENSORS && sumsq_parts && n_parts >= 1, PB_ERR_INVALID,
               "pb_clip_adam_parts: bad arguments");
    AdamArgs a{};
    for (int k = 0; k < n_tensors; ++k) {
        const pb_adam_tensor& t = tensors[k];
        PB_REQUIRE(t.param && t.exp_avg && t.exp_avg_sq && t.step && t.grad && t.numel >= 1, PB_ERR_INVALID,
                   "pb_clip_adam_parts: tensor %d has a null pointer or no elements", k);
        a.t[k] = t;
    }
    PB_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f && grad_scale > 0.f,
               PB_ERR_INVALID, "pb_clip_adam_parts: bad hyper-parameters");
    a.n = n_tensors;
    a.max_norm = max_grad_norm;
    a.grad_scale = grad_scale;
    a.lr = lr;
    a.lr_dev = lr_dev;
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.total_norm_out = total_norm_out;
    pb_head_pack hp{};
    if (pack) {
        PB_REQUIRE(pack->w_dec && pack->b_dec && pack->w_val && pack->b_val && pack->w_cat && pack->b_cat && pack->n_act >= 1 &&
                       pack->n_act <= 7 && pack->hid >= 1,
                   PB_ERR_INVALID, "pb_clip_adam_parts: bad head-pack arguments");
        hp = *pack;
    }
    k_clip_adam_parts<256, false><<<CAP_BLOCKS, 256, 0, (cudaStream_t)stream>>>(a, sumsq_parts, n_parts, peer_epoch, hp, nullptr);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

// The same with the gradient all-reduce over NVLink peer memory in front, in ONE kernel (pb_peer_slices() CTAs): replaces the
// pair pb_peer_allreduce_parts + pb_clip_adam_parts.  sumsq_scratch: pb_peer_slices() doubles of device memory.
extern "C" int pb_clip_adam_peer_parts(const pb_adam_tensor* tensors, int32_t n_tensors, float max_grad_norm, float grad_scale,
                                       float lr, const float* lr_dev, float beta1, float beta2, float eps, float* total_norm_out,
                                       const pb_peer_comm* comm, float* grad_flat, int64_t grad_flat_numel, double* sumsq_scratch,
                                       const pb_head_pack* pack, void* stream) {
    PB_REQUIRE(tensors && n_tensors >= 1 && n_tensors <= CA_MAX_TENSORS && comm && grad_flat && sumsq_scratch, PB_ERR_INVALID,
               "pb_clip_adam_peer_parts: bad arguments");
    PB_REQUIRE(comm->world >= 2 && comm->world <= PB_PEER_MAX_RANKS && comm->rank >= 0 && comm->rank < comm->world && comm->epoch &&
                   grad_flat_numel >= 1 && grad_flat_numel <= comm->capacity,
               PB_ERR_INVALID, "pb_clip_adam_peer_parts: bad communicator or flat gradient buffer");
    for (int r = 0; r < comm->world; ++r) PB_REQUIRE(comm->base[r], PB_ERR_INVALID, "pb_clip_adam_peer_parts: peer %d not mapped", r);
    AdamArgs a{};
    for (int k = 0; k < n_tensors; ++k) {
        const pb_adam_tensor& t = tensors[k];
        PB_REQUIRE(t.param && t.exp_avg && t.exp_avg_sq && t.step && t.grad && t.numel >= 1, PB_ERR_INVALID,
                   "pb_clip_adam_peer_parts: tensor %d has a null pointer or no elements", k);
        PB_REQUIRE(t.grad >= grad_flat && t.grad + t.numel <= grad_flat + grad_flat_numel, PB_ERR_INVALID,
                   "pb_clip_adam_peer_parts: gradient %d lies outside the flat buffer", k);
        a.t[k] = t;
    }
    PB_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps >= 0.f && grad_scale > 0.f,
               PB_ERR_INVALID, "pb_clip_adam_peer_parts: bad hyper-parameters");
    a.n = n_tensors;
    a.max_norm = max_grad_norm;
    a.grad_scale = grad_scale;
    a.lr = lr;
    a.lr_dev = lr_dev;
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.total_norm_out = total_norm_out;
    a.peer = *comm;
    a.flat = grad_flat;
    a.flat_n = grad_flat_numel;
    pb_head_pack hp{};
    if (pack) {
        PB_REQUIRE(pack->w_dec && pack->b_dec && pack->w_val && pack->b_val && pack->w_cat && pack->b_cat && pack->n_act >= 1 &&
                       pack->n_act <= 7 && pack->hid >= 1,
                   PB_ERR_INVALID, "pb_clip_adam_peer_parts: bad head-pack arguments");
        hp = *pack;
    }
    k_clip_adam_parts<512, true><<<PB_PEER_SLICES, 512, 0, (cudaStream_t)stream>>>(
        a, nullptr, 0, reinterpret_cast<unsigned long long*>(comm->epoch), hp, sumsq_scratch);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_pack_heads(const float* w_dec, const float* b_dec, const float* w_val, const float* b_val,
                             int32_t n_act, int32_t hidden_size, float* w_cat, float* b_cat, const float* w_enc,
                             float* w_enc_tf32, int64_t enc_numel, void* stream) {
    PB_REQUIRE(w_dec && b_dec && w_val && b_val && w_cat && b_cat, PB_ERR_INVALID, "pb_pack_heads: null pointer");
    PB_REQUIRE(n_act >= 1 && n_act <= 7 && hidden_size >= 1, PB_ERR_INVALID, "pb_pack_heads: n_act in [1,7], hidden >= 1");
    PB_REQUIRE(!w_enc_tf32 || (w_enc && enc_numel >= 1), PB_ERR_INVALID, "pb_pack_heads: w_enc_tf32 needs w_enc");
    const int64_t work = w_enc_tf32 ? (enc_numel > 8 * (int64_t)hidden_size ? enc_numel : 8 * (int64_t)hidden_size)
                                    : 8 * (int64_t)hidden_size;
    int64_t blocks = pb_ceil_div(work, 256);
    if (blocks > 4 * PB_NUM_SMS) blocks = 4 * PB_NUM_SMS;
    k_pack_heads<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w_dec, b_dec, w_val, b_val, n_act, hidden_size, w_cat,
                                                                     b_cat, w_enc, w_enc_tf32, enc_numel);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
