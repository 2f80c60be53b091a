// env_squared.cu -- N instances of ocean.Squared behind vector.Serial semantics, on the device (sm_90a).
//
// Bit-exact restatement of (paths under reference pufferlib/):
//   environments/ocean/ocean.py:406-513   Squared (grid (2d+1)^2 fp32 in {-1,0,1}; 8 moves; reward 1 - Linf/d;
//                                         done when tick >= d; one perimeter target; teleport to centre on the rim)
//   environments/ocean/environment.py:28-31  distance_to_target=3, num_targets=1
//   postprocess.py:8-54                   EpisodeStats (episode_return, episode_length, score on the done row)
//   emulation.py:169-228                  buffer rows: reset -> r=0, term=False, trunc=False, mask=True
//   vector.py:112-156, 639-641            Serial: seeds seed+i; `if env.done: reset() else: step()` per send
//
// RNG parity: the reference draws targets from CPython's process-global `random` (MT19937).  async_reset seeds
// it per env (init_by_array(seed+i)) and takes one randbelow(8d); every later auto-reset draws the NEXT
// randbelow from the stream left by the last seeded env, in env order.  k_sq_seed does the per-env seeding with
// a thread-local MT state (env N-1 publishes its state as the global stream); k_sq_prepare, one block, ranks the
// envs that reset on this send and regenerates the stream in parallel (4-phase twist, tempering, rejection
// `getrandbits(k) < 8d`, block scan to compact accepted draws).  The stream does not depend on actions.
//
// Step kernel: one lane per env for the state update; the 32 envs of a warp then write their observation rows
// cooperatively (lanes stride across the (2d+1)^2 floats of one row: coalesced 128 B stores); reward / flag /
// done rows are [N]-contiguous stores.  Per-env state is 8 bytes in HBM.
#include "env_common.cuh"
#include "mt19937.cuh"

namespace {

struct SquaredState {
    int d, g, n_targets, bits;  // distance_to_target, grid size, 8d perimeter cells, bit_length(8d)
    uint32_t* d_cell;           // [N] packed: x | y<<8 | tick<<16 | hit<<24
    uint16_t* d_target;         // [N] tx | ty<<8
    uint32_t* d_mt;             // [625] global stream: mt[624] + idx
    int32_t* d_rank;            // [N] rank among the envs that reset on this send (-1 otherwise)
    int32_t* d_draws;           // [N] accepted draws for ranks 0..R-1
    float* d_reward_f32;        // [2d+1] fp32(1 - k/d)
    double* d_reward_f64;       // [2d+1] 1 - k/d in double (EpisodeStats sums python floats)
};

__host__ __device__ inline void target_from_index(int j, int g, int& x, int& y) {
    // ocean.py:444-446: x-major scan of the grid keeping perimeter cells
    if (j < g) { x = 0; y = j; }
    else if (j >= g + 2 * (g - 2)) { x = g - 1; y = j - (g + 2 * (g - 2)); }
    else { const int m = j - g; x = 1 + (m >> 1); y = (m & 1) ? g - 1 : 0; }
}

// async_reset: env i <- random.seed(seed + i); target = possible_targets[randbelow(8d)]
__global__ void __launch_bounds__(64) k_sq_seed(SquaredState st, int n, uint64_t seed_base, uint8_t* done) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t mt[MT_N];
    mt_seed_by_array(mt, seed_base + (uint64_t)i);   // random.seed(int)
    int idx = MT_N;
    int draw;
    do {
        draw = (int)(mt_next(mt, idx) >> (32 - st.bits));
    } while (draw >= st.n_targets);
    int tx, ty;
    target_from_index(draw, st.g, tx, ty);
    st.d_target[i] = (uint16_t)(tx | (ty << 8));
    st.d_cell[i] = (uint32_t)(st.d | (st.d << 8));  // centre, tick 0, not hit
    done[i] = 0;
    if (i == n - 1) {  // the stream every later reset draws from (vector.py:147-149 passes seed=None)
        for (int k = 0; k < MT_N; ++k) st.d_mt[k] = mt[k];
        st.d_mt[MT_N] = (uint32_t)idx;
    }
}

// One block: rank the envs that reset on this send and produce their draws from the global stream.
constexpr int PREP_THREADS = 256;

__global__ void __launch_bounds__(PREP_THREADS) k_sq_prepare(SquaredState st, int n, const uint8_t* done) {
    __shared__ uint32_t mt[MT_N];
    __shared__ int s_warp[PREP_THREADS / 32];
    __shared__ int s_idx, s_newidx;
    const int tid = threadIdx.x;
    const int R = rank_resets<PREP_THREADS>(done, n, st.d_rank, s_warp);   // ranks in env order
    if (R == 0) return;
    for (int k = tid; k < MT_N; k += PREP_THREADS) mt[k] = st.d_mt[k];
    if (tid == 0) s_idx = (int)st.d_mt[MT_N];
    __syncthreads();
    int accepted = 0;
    while (accepted < R) {
        if (s_idx >= MT_N) {
            mt_twist_block<PREP_THREADS>(mt);
            if (tid == 0) s_idx = 0;
            __syncthreads();
        }
        const int start = s_idx;
        const int pos = start + tid;
        const bool valid = pos < MT_N;
        int draw = 0;
        if (valid) draw = (int)(mt_temper(mt[pos]) >> (32 - st.bits));
        const int acc = (valid && draw < st.n_targets) ? 1 : 0;
        int tot;
        const int off = block_exclusive_scan<PREP_THREADS>(acc, &tot, s_warp);
        if (acc && accepted + off < R) {
            st.d_draws[accepted + off] = draw;
            if (accepted + off == R - 1) s_newidx = pos + 1;  // stream position just after the last used output
        }
        __syncthreads();
        if (accepted + tot >= R) {
            accepted = R;
            if (tid == 0) s_idx = s_newidx;
        } else {
            accepted += tot;
            if (tid == 0) s_idx = min(start + PREP_THREADS, MT_N);
        }
        __syncthreads();
    }
    for (int k = tid; k < MT_N; k += PREP_THREADS) st.d_mt[k] = mt[k];
    if (tid == 0) st.d_mt[MT_N] = (uint32_t)s_idx;
}

struct SqOut {
    float* obs;
    int64_t obs_stride_f;  // in floats
    float* rewards;
    uint8_t* terminals;
    uint8_t* truncations;
    uint8_t* masks;
    float* dones_f32;
    bool write_const;
};

// mode 0: write reset rows for every env (after k_sq_seed); mode 1: vectoriser send (reset-or-step)
template <int MODE>
__global__ void __launch_bounds__(128) k_sq_step(SquaredState st, int n, const int64_t* __restrict__ actions,
                                                uint8_t* done, SqOut out, EpisodeAcc acc) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool active = e < n;
    int x = 0, y = 0, tick = 0, hit = 0, tx = 0, ty = 0;
    float reward = 0.f;
    double reward_d = 0.0;
    bool terminal = false, reset_row = true;
    if (active) {
        const uint32_t c = st.d_cell[e];
        x = c & 0xff; y = (c >> 8) & 0xff; tick = (c >> 16) & 0xff; hit = (c >> 24) & 1;
        const uint16_t t = st.d_target[e];
        tx = t & 0xff; ty = t >> 8;
        if (MODE == 1) {
            if (done[e]) {  // vector.py:147-149: reset, action ignored
                target_from_index(st.d_draws[st.d_rank[e]], st.g, tx, ty);
                x = y = st.d; tick = 0; hit = 0;
            } else {        // ocean.py:465-513
                reset_row = false;
                int a = (int)actions[e];
                a = a < 0 ? 0 : (a > 7 ? 7 : a);
                // MOVES = [(0,-1),(0,1),(-1,0),(1,0),(1,-1),(-1,-1),(1,1),(-1,1)]   ocean.py:424
                const int dx = ((0x2285 >> (2 * a)) & 3) - 1;   // dx+1 packed 2 bits per action
                const int dy = ((0xA058 >> (2 * a)) & 3) - 1;   // dy+1 packed 2 bits per action
                x += dx; y += dy;
                const int k = max(abs(x - tx), abs(y - ty));
                reward = st.d_reward_f32[k];
                reward_d = st.d_reward_f64[k];
                if (x == tx && y == ty) hit = 1;
                if (max(abs(x - st.d), abs(y - st.d)) >= st.d) { x = st.d; y = st.d; }
                tick += 1;
                terminal = tick >= st.d;  // max_ticks = num_targets * distance_to_target
            }
            st.d_cell[e] = (uint32_t)(x | (y << 8) | (tick << 16) | (hit << 24));
            st.d_target[e] = (uint16_t)(tx | (ty << 8));
            done[e] = terminal ? 1 : 0;
        }
        out.rewards[e] = reward;
        out.terminals[e] = terminal ? 1 : 0;
        if (out.write_const) out.truncations[e] = 0;
        if (out.write_const) out.masks[e] = 1;
        if (out.dones_f32) out.dones_f32[e] = terminal ? 1.f : 0.f;
    }
    episode_update(acc, e, active, reset_row, reward_d, terminal, (float)hit);
    // cooperative observation rows: the warp walks its 32 envs, lanes stride over the g*g cells of one row
    const int cells = st.g * st.g;
    const int agent_cell = x * st.g + y, target_cell = tx * st.g + ty;
    const int e_base = e - lane;
    for (int j = 0; j < 32; ++j) {
        const int ej = e_base + j;
        if (ej >= n) break;
        const int ac = __shfl_sync(0xffffffffu, agent_cell, j);
        const int tc = __shfl_sync(0xffffffffu, target_cell, j);
        float* row = out.obs + (int64_t)ej * out.obs_stride_f;
        for (int c = lane; c < cells; c += 32) row[c] = (c == ac) ? -1.f : ((c == tc) ? 1.f : 0.f);
    }
}

int squared_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    SquaredState* st = (SquaredState*)env->kind;
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 4 == 0 && ((uintptr_t)out->obs & 3) == 0, PB_ERR_INVALID,
               "squared: obs pointer/stride must be 4-byte aligned");
    SqOut o{(float*)out->obs, out->obs_stride / 4, out->rewards, out->terminals, out->truncations, out->masks,
            out->dones_f32,
            env->write_const};
    const int blocks = (int)pb_ceil_div(n, 128);
    if (mode == 0)
        k_sq_step<0><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, o, pb_episode_acc(env));
    else
        k_sq_step<1><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, o, pb_episode_acc(env));
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int squared_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    SquaredState* st = (SquaredState*)env->kind;
    const int n = env->cfg.num_envs;
    k_sq_seed<<<(int)pb_ceil_div(n, 64), 64, 0, s>>>(*st, n, seed + (uint64_t)env->cfg.env_index_offset, env->d_done);
    PB_LAUNCH_CHECK();
    return squared_launch(env, 0, nullptr, out, s);
}

int squared_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    SquaredState* st = (SquaredState*)env->kind;
    k_sq_prepare<<<1, PREP_THREADS, 0, s>>>(*st, env->cfg.num_envs, env->d_done);
    PB_LAUNCH_CHECK();
    return squared_launch(env, 1, actions, out, s);
}

void squared_destroy(pb_env* env) {
    SquaredState* st = (SquaredState*)env->kind;
    if (!st) return;
    cudaFree(st->d_cell); cudaFree(st->d_target); cudaFree(st->d_mt); cudaFree(st->d_rank); cudaFree(st->d_draws);
    cudaFree(st->d_reward_f32); cudaFree(st->d_reward_f64);
    delete st;
    env->kind = nullptr;
}

const pb_env_vtable SQUARED_VT = {squared_reset, squared_step, squared_destroy};

}  // namespace

int pb_squared_create(pb_env* env) {
    const int d = env->cfg.iparam[0] > 0 ? env->cfg.iparam[0] : 3;
    PB_REQUIRE(d >= 1 && d <= 15, PB_ERR_INVALID, "squared: distance_to_target must be in [1, 15]");
    SquaredState* st = new SquaredState();
    env->kind = st;
    env->vt = &SQUARED_VT;
    st->d = d;
    st->g = 2 * d + 1;
    st->n_targets = 8 * d;
    st->bits = 0;
    while ((1 << st->bits) <= st->n_targets) ++st->bits;  // int.bit_length(8d)
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&st->d_cell, n * sizeof(uint32_t)));
    PB_CUDA(cudaMalloc(&st->d_target, n * sizeof(uint16_t)));
    PB_CUDA(cudaMalloc(&st->d_mt, (MT_N + 1) * sizeof(uint32_t)));
    PB_CUDA(cudaMalloc(&st->d_rank, n * sizeof(int32_t)));
    PB_CUDA(cudaMalloc(&st->d_draws, n * sizeof(int32_t)));
    PB_CUDA(cudaMalloc(&st->d_reward_f32, (2 * d + 1) * sizeof(float)));
    PB_CUDA(cudaMalloc(&st->d_reward_f64, (2 * d + 1) * sizeof(double)));
    PB_CUDA(cudaMemset(st->d_cell, 0, n * sizeof(uint32_t)));
    PB_CUDA(cudaMemset(st->d_target, 0, n * sizeof(uint16_t)));
    PB_CUDA(cudaMemset(st->d_mt, 0, (MT_N + 1) * sizeof(uint32_t)));
    float rf[31];
    double rd[31];
    for (int k = 0; k <= 2 * d; ++k) {
        rd[k] = 1.0 - (double)k / (double)d;  // python: 1 - min_dist / distance_to_target (ocean.py:477)
        rf[k] = (float)rd[k];                 // fp32 store into buf.rewards (emulation.py:221)
    }
    PB_CUDA(cudaMemcpy(st->d_reward_f32, rf, (2 * d + 1) * sizeof(float), cudaMemcpyHostToDevice));
    PB_CUDA(cudaMemcpy(st->d_reward_f64, rd, (2 * d + 1) * sizeof(double), cudaMemcpyHostToDevice));
    env->info.obs_dtype = PB_DTYPE_F32;
    env->info.obs_ndim = 2;
    env->info.obs_shape[0] = st->g;
    env->info.obs_shape[1] = st->g;
    env->info.obs_bytes = (int64_t)st->g * st->g * 4;
    env->info.num_actions = 8;
    env->info.obs_low = -1.f;
    env->info.obs_high = 1.f;
    return PB_OK;
}
