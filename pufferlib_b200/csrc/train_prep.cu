// train_prep.cu -- rollout-buffer write, minibatch construction and advantage normalisation (sm_90a).
//
// Replaces, from reference clean_pufferl.py:
//   :443-446  Experience.store (value / logprob / action rows)        -> pb_rollout_store
//   :442      obs[ptr:end] = obs[indices] (all-True mask)            -> pb_copy_rows
//   :466-482  Experience.flatten_batch (scalar tensors)              -> pb_flatten_batch
//   :477      b_obs = obs[b_idxs_obs]                                 -> pb_minibatch_gather (LSU path; TMA path in image.cu)
//   :211-213  per-minibatch advantage normalisation                   -> pb_adv_norm
// All of these are HBM-bound byte movers: coalesced, vectorised, grid sized in multiples of the SM count.
#include "pb_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ store
__global__ void __launch_bounds__(256) k_rollout_store(const float* __restrict__ value,
                                                      const float* __restrict__ logprob,
                                                      const int64_t* __restrict__ action, float* values_row,
                                                      float* logprobs_row, int64_t* actions_row, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        if (values_row) values_row[i] = value[i];
        if (logprobs_row) logprobs_row[i] = logprob[i];
        if (actions_row) actions_row[i] = action[i];
    }
}

// ------------------------------------------------------------------------------------------------ row copies
template <typename V>
__device__ __forceinline__ void copy_row_warp(const char* src, char* dst, int row_vecs, int lane) {
    const V* s = reinterpret_cast<const V*>(src);
    V* d = reinterpret_cast<V*>(dst);
    for (int c = lane; c < row_vecs; c += 32) d[c] = __ldcs(s + c);
}

template <typename V>
__global__ void __launch_bounds__(256) k_copy_rows(const char* __restrict__ src, int64_t src_stride,
                                                  char* __restrict__ dst, int64_t dst_stride, int row_vecs,
                                                  int64_t n_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t row = warp; row < n_rows; row += nwarps)
        copy_row_warp<V>(src + row * src_stride, dst + row * dst_stride, row_vecs, lane);
}

// sorted row f = (r*n_mb + mb)*bptt + j  ->  arrival row t*N + e with e = f / H, t = f % H
struct GatherGeom {
    int64_t N, H, n_mb, rows, bptt, mb_begin;
};

// One warp moves 32 output rows per iteration.  Lane k does the (division-heavy) index arithmetic for row o0+k
// once; the row byte offsets are then shuffle-broadcast and every row is copied by all 32 lanes, UNROLL rows at a
// time with all loads issued before the first store (memory-level parallelism).
template <typename V, int UNROLL>
__global__ void __launch_bounds__(256) k_minibatch_gather(const char* __restrict__ obs, char* __restrict__ dst,
                                                         int64_t row_bytes, int row_vecs, int64_t n_out_rows,
                                                         GatherGeom g) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t mb_size = g.rows * g.bptt;
    for (int64_t o0 = warp * 32; o0 < n_out_rows; o0 += nwarps * 32) {
        const int64_t o = min(o0 + lane, n_out_rows - 1);
        const int64_t mb = g.mb_begin + o / mb_size, rem = o % mb_size;
        const int64_t r = rem / g.bptt, j = rem - r * g.bptt;
        const int64_t f = (r * g.n_mb + mb) * g.bptt + j;
        const int64_t e = f / g.H, t = f - e * g.H;
        const int64_t my_src = (t * g.N + e) * row_bytes;
        const int rows_here = (int)min((int64_t)32, n_out_rows - o0);
        for (int k0 = 0; k0 < rows_here; k0 += UNROLL) {
            const V* s[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
                s[u] = reinterpret_cast<const V*>(obs + __shfl_sync(0xffffffffu, my_src, min(k0 + u, rows_here - 1)));
            for (int c = lane; c < row_vecs; c += 32) {
                V tmp[UNROLL];
#pragma unroll
                for (int u = 0; u < UNROLL; ++u) tmp[u] = __ldcs(s[u] + c);
#pragma unroll
                for (int u = 0; u < UNROLL; ++u)
                    if (k0 + u < rows_here) reinterpret_cast<V*>(dst + (o0 + k0 + u) * row_bytes)[c] = tmp[u];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ flatten_batch
constexpr int FT = 32;  // tile: 32 envs x 32 steps

struct FlattenParams {
    const int64_t* actions;
    const float* logprobs;
    const float* dones;
    const float* values;
    const float* adv;  // sorted order
    int64_t* b_actions;
    float* b_logprobs;
    float* b_dones;
    float* b_values;
    float* b_adv;
    float* b_ret;
    float* returns_np;
    int N, H, n_mb, rows, bptt;
};

__global__ void __launch_bounds__(256) k_flatten_batch(FlattenParams p) {
    __shared__ float sL[FT][FT + 1], sD[FT][FT + 1], sV[FT][FT + 1];
    __shared__ int64_t sA[FT][FT + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int e0 = blockIdx.x * FT, t0 = blockIdx.y * FT;
    // load: lane = env (coalesced along e), warp strides over the tile's time rows
    for (int tl = warp; tl < FT; tl += 8) {
        const int t = t0 + tl, e = e0 + lane;
        if (t < p.H && e < p.N) {
            const int64_t i = (int64_t)t * p.N + e;
            const float v = p.values[i];
            sV[tl][lane] = v;
            sL[tl][lane] = p.logprobs ? p.logprobs[i] : 0.f;
            sD[tl][lane] = p.dones ? p.dones[i] : 0.f;
            sA[tl][lane] = p.actions ? p.actions[i] : 0;
            // clean_pufferl.py:476, literally: sorted-order advantages + arrival-order values, same flat index
            if (p.returns_np) p.returns_np[i] = p.adv[i] + v;
        }
    }
    __syncthreads();
    // store: lane = step (f contiguous along t), warp strides over the tile's envs
    const int mb_size = p.rows * p.bptt;
    for (int el = warp; el < FT; el += 8) {
        const int e = e0 + el, t = t0 + lane;
        if (e < p.N && t < p.H) {
            const int64_t f = (int64_t)e * p.H + t;
            const int64_t k = f / p.bptt;
            const int j = (int)(f - k * p.bptt);
            const int mb = (int)(k % p.n_mb), r = (int)(k / p.n_mb);
            const int64_t o = (int64_t)mb * mb_size + (int64_t)r * p.bptt + j;
            const float v = sV[lane][el];
            const float a = p.adv[f];
            if (p.b_actions) p.b_actions[o] = sA[lane][el];
            if (p.b_logprobs) p.b_logprobs[o] = sL[lane][el];
            if (p.b_dones) p.b_dones[o] = sD[lane][el];
            if (p.b_values) p.b_values[o] = v;
            if (p.b_adv) p.b_adv[o] = a;
            if (p.b_ret) p.b_ret[o] = a + v;
        }
    }
}

// ------------------------------------------------------------------------------------------------ adv norm
constexpr int AN_THREADS = 256;
constexpr int AN_MAX_PARTS = 64;

__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
    return x;
}

// grid (parts, n_mb): block (part, mb) reduces its slice of minibatch mb to (sum, sum of squares) in fp64
__global__ void __launch_bounds__(AN_THREADS) k_adv_stats(const float* __restrict__ adv, int64_t mb_size,
                                                         double2* __restrict__ partials) {
    const int part = blockIdx.x, parts = gridDim.x, mb = blockIdx.y;
    const float* a = adv + (int64_t)mb * mb_size;
    const int64_t chunk = pb_ceil_div_dev(mb_size, parts);
    const int64_t lo = (int64_t)part * chunk, hi = min(lo + chunk, mb_size);
    double s = 0.0, ss = 0.0;
    int64_t i = lo + threadIdx.x;
    if ((reinterpret_cast<uintptr_t>(a + lo) & 15) == 0) {
        const int64_t nv = (hi - lo) / 4;
        const float4* a4 = reinterpret_cast<const float4*>(a + lo);
        for (int64_t q = threadIdx.x; q < nv; q += AN_THREADS) {
            const float4 x = a4[q];
            s += (double)x.x + (double)x.y + (double)x.z + (double)x.w;
            ss += (double)x.x * x.x + (double)x.y * x.y + (double)x.z * x.z + (double)x.w * x.w;
        }
        i = lo + nv * 4 + threadIdx.x;
    }
    for (; i < hi; i += AN_THREADS) {
        const double x = a[i];
        s += x;
        ss += x * x;
    }
    __shared__ double sh_s[AN_THREADS / 32], sh_ss[AN_THREADS / 32];
    s = warp_sum(s);
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) {
        sh_s[threadIdx.x >> 5] = s;
        sh_ss[threadIdx.x >> 5] = ss;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ts = 0.0, tss = 0.0;
        for (int w = 0; w < AN_THREADS / 32; ++w) {
            ts += sh_s[w];
            tss += sh_ss[w];
        }
        partials[(int64_t)mb * parts + part] = make_double2(ts, tss);
    }
}

__global__ void __launch_bounds__(AN_THREADS) k_adv_apply(const float* __restrict__ adv, float* __restrict__ out,
                                                         int64_t mb_size, const double2* __restrict__ partials) {
    const int part = blockIdx.x, parts = gridDim.x, mb = blockIdx.y;
    __shared__ float s_mean, s_den;
    if (threadIdx.x == 0) {
        double ts = 0.0, tss = 0.0;
        for (int q = 0; q < parts; ++q) {
            const double2 v = partials[(int64_t)mb * parts + q];
            ts += v.x;
            tss += v.y;
        }
        const double n = (double)mb_size;
        const double mean = ts / n;
        double var = (tss - ts * mean) / (n - 1.0);  // unbiased (torch.Tensor.std default); n == 1 -> nan like torch
        if (var < 0.0) var = 0.0;
        s_mean = (float)mean;
        s_den = (float)sqrt(var) + 1e-8f;
    }
    __syncthreads();
    const float mean = s_mean, den = s_den;
    const float* a = adv + (int64_t)mb * mb_size;
    float* o = out + (int64_t)mb * mb_size;
    const int64_t chunk = pb_ceil_div_dev(mb_size, parts);
    const int64_t lo = (int64_t)part * chunk, hi = min(lo + chunk, mb_size);
    for (int64_t i = lo + threadIdx.x; i < hi; i += AN_THREADS) o[i] = (a[i] - mean) / den;
}

// Advantage statistics of the zero-copy slab minibatches (clean_pufferl.Experience.flatten_batch_slabs) straight from the
// ARRIVAL-order advantages: minibatch mb = slabs (g*n_mb + mb), g = 0..G-1, of R consecutive rows each.
// grid (parts, n_mb); partials[mb][part] = (sum, sum of squares) in fp64.
__global__ void __launch_bounds__(AN_THREADS) k_adv_stats_slabs(const float* __restrict__ adv, int64_t slab_rows, int n_slabs,
                                                               int n_mb, double2* __restrict__ partials) {
    const int part = blockIdx.x, parts = gridDim.x, mb = blockIdx.y;
    const int64_t total = slab_rows * n_slabs;
    const int64_t chunk = (pb_ceil_div_dev(total, parts) + 3) & ~(int64_t)3;
    const int64_t lo = (int64_t)part * chunk, hi = min(lo + chunk, total);
    double s = 0.0, ss = 0.0;
    const bool vec = (slab_rows & 3) == 0 && (reinterpret_cast<uintptr_t>(adv) & 15) == 0;
    if (vec) {
        for (int64_t i = lo + 4 * (int64_t)threadIdx.x; i < hi; i += 4 * AN_THREADS) {
            const int64_t g = i / slab_rows, r = i - g * slab_rows;
            const float4 x = *reinterpret_cast<const float4*>(adv + ((g * n_mb + mb) * slab_rows + r));
            s += (double)x.x + (double)x.y + (double)x.z + (double)x.w;
            ss += (double)x.x * x.x + (double)x.y * x.y + (double)x.z * x.z + (double)x.w * x.w;
        }
    } else {
        for (int64_t i = lo + threadIdx.x; i < hi; i += AN_THREADS) {
            const int64_t g = i / slab_rows, r = i - g * slab_rows;
            const double x = adv[(g * n_mb + mb) * slab_rows + r];
            s += x;
            ss += x * x;
        }
    }
    __shared__ double sh_s[AN_THREADS / 32], sh_ss[AN_THREADS / 32];
    s = warp_sum(s);
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) {
        sh_s[threadIdx.x >> 5] = s;
        sh_ss[threadIdx.x >> 5] = ss;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ts = 0.0, tss = 0.0;
        for (int w = 0; w < AN_THREADS / 32; ++w) {
            ts += sh_s[w];
            tss += sh_ss[w];
        }
        partials[(int64_t)mb * parts + part] = make_double2(ts, tss);
    }
}

// norm[mb] = (mean, 1 / (std + 1e-8)) with the unbiased std of clean_pufferl.py:211-213 (torch.Tensor.std default)
__global__ void k_adv_finalize(const double2* __restrict__ partials, int parts, int64_t mb_size, float2* __restrict__ norm) {
    const int mb = threadIdx.x;       // one block of n_mb threads
    double ts = 0.0, tss = 0.0;
    for (int q = 0; q < parts; ++q) {
        const double2 v = partials[(int64_t)mb * parts + q];
        ts += v.x;
        tss += v.y;
    }
    const double n = (double)mb_size;
    const double mean = ts / n;
    double var = (tss - ts * mean) / (n - 1.0);
    if (var < 0.0) var = 0.0;
    norm[mb] = make_float2((float)mean, 1.0f / ((float)sqrt(var) + 1e-8f));
}

template <typename V>
int launch_copy_rows(const void* src, int64_t ss, void* dst, int64_t ds, int64_t row_bytes, int64_t n_rows,
                     cudaStream_t s) {
    const int row_vecs = (int)(row_bytes / (int64_t)sizeof(V));
    const int64_t warps_needed = n_rows;
    int64_t blocks = pb_ceil_div(warps_needed, 8);
    const int64_t cap = (int64_t)PB_NUM_SMS * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    k_copy_rows<V><<<(unsigned)blocks, 256, 0, s>>>((const char*)src, ss, (char*)dst, ds, row_vecs, n_rows);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int vec_bytes_for(const void* a, const void* b, int64_t stride_a, int64_t stride_b, int64_t row_bytes) {
    const uintptr_t bits = (uintptr_t)a | (uintptr_t)b | (uintptr_t)stride_a | (uintptr_t)stride_b |
                           (uintptr_t)row_bytes;
    if ((bits & 15) == 0) return 16;
    if ((bits & 3) == 0) return 4;
    return 1;
}

}  // namespace

extern "C" int pb_rollout_store(const float* value, const float* logprob, const int64_t* action, float* values_row,
                                float* logprobs_row, int64_t* actions_row, int64_t n, void* stream) {
    PB_REQUIRE(n >= 0, PB_ERR_INVALID, "pb_rollout_store: negative n");
    if (n == 0) return PB_OK;
    PB_REQUIRE((!values_row || value) && (!logprobs_row || logprob) && (!actions_row || action), PB_ERR_INVALID,
               "pb_rollout_store: destination row given without its source");
    k_rollout_store<<<(unsigned)pb_ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(
        value, logprob, action, values_row, logprobs_row, actions_row, n);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_copy_rows(const void* src, int64_t src_stride, void* dst, int64_t dst_stride, int64_t row_bytes,
                            int64_t n_rows, void* stream) {
    PB_REQUIRE(row_bytes >= 0 && n_rows >= 0, PB_ERR_INVALID, "pb_copy_rows: negative size");
    if (row_bytes == 0 || n_rows == 0) return PB_OK;
    PB_REQUIRE(src && dst, PB_ERR_INVALID, "pb_copy_rows: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    switch (vec_bytes_for(src, dst, src_stride, dst_stride, row_bytes)) {
        case 16: return launch_copy_rows<uint4>(src, src_stride, dst, dst_stride, row_bytes, n_rows, s);
        case 4: return launch_copy_rows<uint32_t>(src, src_stride, dst, dst_stride, row_bytes, n_rows, s);
        default: return launch_copy_rows<unsigned char>(src, src_stride, dst, dst_stride, row_bytes, n_rows, s);
    }
}

int pb_minibatch_gather_tma(const void* obs, void* dst, int64_t row_bytes, int64_t N, int64_t H, int64_t n_mb,
                            int64_t rows, int64_t bptt, int64_t mb_begin, int64_t mb_count, cudaStream_t s);

extern "C" int pb_minibatch_gather(const void* obs, void* dst, int64_t row_bytes, int64_t num_envs,
                                   int64_t horizon, int64_t n_mb, int64_t rows, int64_t bptt, int64_t mb_begin,
                                   int64_t mb_count, void* stream) {
    PB_REQUIRE(row_bytes > 0 && num_envs > 0 && horizon > 0 && n_mb > 0 && rows > 0 && bptt > 0, PB_ERR_INVALID,
               "pb_minibatch_gather: sizes must be positive");
    PB_REQUIRE(n_mb * rows * bptt == num_envs * horizon, PB_ERR_INVALID,
               "pb_minibatch_gather: n_mb*rows*bptt (%lld) != num_envs*horizon (%lld)",
               (long long)(n_mb * rows * bptt), (long long)(num_envs * horizon));
    PB_REQUIRE(mb_begin >= 0 && mb_count >= 0 && mb_begin + mb_count <= n_mb, PB_ERR_INVALID,
               "pb_minibatch_gather: minibatch range out of bounds");
    if (mb_count == 0) return PB_OK;
    PB_REQUIRE(obs && dst, PB_ERR_INVALID, "pb_minibatch_gather: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const int vb = vec_bytes_for(obs, dst, row_bytes, row_bytes, row_bytes);
    if (vb == 16 && row_bytes >= 4096)
        return pb_minibatch_gather_tma(obs, dst, row_bytes, num_envs, horizon, n_mb, rows, bptt, mb_begin, mb_count, s);
    const int64_t n_out = mb_count * rows * bptt;
    GatherGeom g{num_envs, horizon, n_mb, rows, bptt, mb_begin};
    constexpr int RPI = 8;   // rows in flight per warp
    int64_t blocks = pb_ceil_div(pb_ceil_div(n_out, 32), 8);
    const int64_t cap = (int64_t)PB_NUM_SMS * 8;
    if (blocks > cap) blocks = cap;
    if (vb == 16)
        k_minibatch_gather<uint4, RPI><<<(unsigned)blocks, 256, 0, s>>>((const char*)obs, (char*)dst, row_bytes,
                                                                        (int)(row_bytes / 16), n_out, g);
    else if (vb == 4)
        k_minibatch_gather<uint32_t, RPI><<<(unsigned)blocks, 256, 0, s>>>((const char*)obs, (char*)dst, row_bytes,
                                                                           (int)(row_bytes / 4), n_out, g);
    else
        k_minibatch_gather<unsigned char, RPI><<<(unsigned)blocks, 256, 0, s>>>((const char*)obs, (char*)dst,
                                                                                row_bytes, (int)row_bytes, n_out, g);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_flatten_batch(const int64_t* actions, const float* logprobs, const float* dones,
                                const float* values, const float* advantages_sorted, int64_t* b_actions,
                                float* b_logprobs, float* b_dones, float* b_values, float* b_advantages,
                                float* b_returns, float* returns_np, int64_t num_envs, int64_t horizon,
                                int64_t n_mb, int64_t rows, int64_t bptt, void* stream) {
    PB_REQUIRE(num_envs > 0 && horizon > 0 && n_mb > 0 && rows > 0 && bptt > 0, PB_ERR_INVALID,
               "pb_flatten_batch: sizes must be positive");
    PB_REQUIRE(n_mb * rows * bptt == num_envs * horizon, PB_ERR_INVALID,
               "pb_flatten_batch: n_mb*rows*bptt != num_envs*horizon");
    PB_REQUIRE(num_envs * horizon < (1ll << 31), PB_ERR_INVALID, "pb_flatten_batch: batch must be < 2^31 rows");
    PB_REQUIRE(values && advantages_sorted, PB_ERR_INVALID, "pb_flatten_batch: values/advantages required");
    PB_REQUIRE((!b_actions || actions) && (!b_logprobs || logprobs) && (!b_dones || dones), PB_ERR_INVALID,
               "pb_flatten_batch: output given without its input");
    FlattenParams p{actions, logprobs, dones, values, advantages_sorted, b_actions, b_logprobs, b_dones,
                    b_values, b_advantages, b_returns, returns_np,
                    (int)num_envs, (int)horizon, (int)n_mb, (int)rows, (int)bptt};
    dim3 grid((unsigned)pb_ceil_div(num_envs, FT), (unsigned)pb_ceil_div(horizon, FT));
    PB_REQUIRE(grid.y <= 65535, PB_ERR_INVALID, "pb_flatten_batch: horizon too large");
    k_flatten_batch<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

static int adv_norm_parts(int64_t n_mb, int64_t mb_size) {
    int64_t parts = pb_ceil_div((int64_t)PB_NUM_SMS * 4, n_mb);      // ~4 blocks per SM overall
    const int64_t max_by_work = pb_ceil_div(mb_size, 2048);           // at least 2048 elements per block
    if (parts > max_by_work) parts = max_by_work;
    if (parts > AN_MAX_PARTS) parts = AN_MAX_PARTS;
    if (parts < 1) parts = 1;
    return (int)parts;
}

extern "C" size_t pb_adv_norm_workspace_bytes(int64_t n_mb, int64_t mb_size) {
    if (n_mb <= 0 || mb_size <= 0) return 16;
    return (size_t)n_mb * adv_norm_parts(n_mb, mb_size) * sizeof(double2);
}

extern "C" int pb_adv_norm(const float* adv, float* out, int64_t n_mb, int64_t mb_size, void* workspace,
                           size_t workspace_bytes, void* stream) {
    PB_REQUIRE(n_mb >= 0 && mb_size >= 0, PB_ERR_INVALID, "pb_adv_norm: negative size");
    if (n_mb == 0 || mb_size == 0) return PB_OK;
    PB_REQUIRE(adv && out, PB_ERR_INVALID, "pb_adv_norm: null pointer");
    PB_REQUIRE(n_mb <= 65535, PB_ERR_INVALID, "pb_adv_norm: too many minibatches");
    const int parts = adv_norm_parts(n_mb, mb_size);
    PB_REQUIRE(workspace && workspace_bytes >= (size_t)n_mb * parts * sizeof(double2), PB_ERR_INVALID,
               "pb_adv_norm: workspace too small");
    dim3 grid((unsigned)parts, (unsigned)n_mb);
    cudaStream_t s = (cudaStream_t)stream;
    k_adv_stats<<<grid, AN_THREADS, 0, s>>>(adv, mb_size, (double2*)workspace);
    PB_LAUNCH_CHECK();
    k_adv_apply<<<grid, AN_THREADS, 0, s>>>(adv, out, mb_size, (const double2*)workspace);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_adv_stats_slabs(const float* advantages_time_major, int64_t slab_rows, int32_t n_slabs, int32_t n_minibatches,
                                  float* norm_out, void* workspace, size_t workspace_bytes, void* stream) {
    PB_REQUIRE(advantages_time_major && norm_out && workspace, PB_ERR_INVALID, "pb_adv_stats_slabs: null pointer");
    PB_REQUIRE(slab_rows >= 1 && n_slabs >= 1 && n_minibatches >= 1 && n_minibatches <= 65535, PB_ERR_INVALID,
               "pb_adv_stats_slabs: bad sizes");
    const int64_t mb_size = slab_rows * n_slabs;
    PB_REQUIRE(workspace_bytes >= pb_adv_norm_workspace_bytes(n_minibatches, mb_size), PB_ERR_INVALID,
               "pb_adv_stats_slabs: workspace too small");
    PB_REQUIRE(n_minibatches <= 1024, PB_ERR_UNSUPPORTED, "pb_adv_stats_slabs: at most 1024 minibatches");
    const int parts = adv_norm_parts(n_minibatches, mb_size);
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)parts, (unsigned)n_minibatches);
    k_adv_stats_slabs<<<grid, AN_THREADS, 0, s>>>(advantages_time_major, slab_rows, n_slabs, n_minibatches,
                                                   (double2*)workspace);
    PB_LAUNCH_CHECK();
    k_adv_finalize<<<1, n_minibatches, 0, s>>>((const double2*)workspace, parts, mb_size, (float2*)norm_out);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
