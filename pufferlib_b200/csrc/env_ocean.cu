// env_ocean.cu -- the reference's ocean test envs Memory, Password, Stochastic, Bandit and Multiagent, N instances
// each behind vector.Serial semantics, on the device (sm_90a).  Each env probes one learning ability: recall (memory),
// exploration (password), a stochastic optimum (stochastic), credit assignment under reward noise (bandit), one
// policy serving two agents that need different actions (multiagent: two agent rows per env, see multiagent_step).
//
// Bit-exact restatement of (paths under reference pufferlib/):
//   environments/ocean/ocean.py:64-123    Memory      (obs = digit on ticks < L else 0; reward for 0 on the
//                                                      show ticks, for the digit on the answer ticks; horizon 2L+D)
//   environments/ocean/ocean.py:228-281   Password    (obs = guesses so far, -1 elsewhere; reward on the last tick)
//   environments/ocean/ocean.py:529-582   Stochastic  (reward 1 - (p - count/tick)**2 when the action moves the
//                                                      action-0 share towards p; 100 ticks)
//   environments/ocean/ocean.py:8-62      Bandit      (one-step episodes; (correct + randn*scale)*scale)
//   environments/ocean/environment.py:33-46, 67-70   creator defaults: memory L=2 D=2, password 5, stochastic
//                                                      p=0.7 horizon=100, bandit 10 arms scale 1 noise 1
//   environments/ocean/ocean.py:149-208   Multiagent  (agent 1 rewarded for action 0, agent 2 for action 1; every
//                                                      step terminal for both, so every second send resets)
//   postprocess.py:8-54 EpisodeStats, emulation.py:169-228 buffer rows, vector.py:112-156 Serial
//   postprocess.py:147-179 MultiagentEpisodeStats (per-agent infos only), emulation.py:236-420 PettingZooPufferEnv
//
// RNG parity (numpy's legacy process-global np.random, MT19937 seeded by init_genrand):
//   memory     async_reset seeds env i with seed+i and draws 2L+D digits (randint(0, 2) = genrand & 1); every later
//              reset draws the next 2L+D outputs of the stream left by the last seeded env, in env order.  k_mem_seed
//              seeds one env per thread (env N-1 publishes its state); k_mem_prepare, one block, ranks the resetting
//              envs and regenerates R*(2L+D) outputs with a block-parallel twist.  Only the first L digits are kept.
//   password   reseeds 42 on every reset: the solution is a constant, computed once per handle.
//   bandit     reseeds 42 on every reset and every episode lasts one step, so on every step-send env j of a shard
//              draws the same gaussian G[j] (legacy polar method from the state "seed(42), one randint").  G is
//              computed once per handle on the device, in fp64.
//   stochastic draws nothing.  Its reward table 1 - (p - c/t)**2 is built on the host with libm pow, the function
//              python's float ** calls: pow(x, 2) is not always x*x rounded (it differs in 5 of the 5151 cells at
//              p = 0.7 with glibc 2.39), so only pow itself reproduces the reference's bits.
//   memory and stochastic pass seed+i to np.random.seed, which refuses seeds >= 2**32: so does the reset here.
//
// Envelope (refused in pb_env_create before any launch): mem_length in [1, 64], mem_delay in [0, 1024],
// password_length in [1, 128], num_actions in [1, 32768], finite p / reward_scale / reward_noise.
//
// Kernels: one lane per env for all four kinds; observation rows (1 float, or L floats for password), reward,
// terminal and dones_f32 rows go straight to the caller's pb_env_out.  HBM state per env: memory 12 B
// (tick + L digits), password 20 B (tick + guess bits), stochastic 4 B (tick + count), bandit 8 B (G[j]).
#include <math.h>

#include <vector>

#include "env_common.cuh"
#include "mt19937.cuh"

namespace {

constexpr int MEM_MAX_L = 64, MEM_MAX_D = 1024, PW_MAX_L = 128, BANDIT_MAX_ARMS = 1 << 15;
constexpr int STOCH_HORIZON = 100;   // make_stochastic passes horizon=100 whatever it is given
constexpr int PREP_THREADS = 256;

struct OceanState {
    int kind;
    int L, D, h;                 // memory: mem_length, mem_delay, 2L + D;  password: L = password_length
    int n_act;
    double p, scale, noise;      // stochastic p; bandit reward_scale, reward_noise
    int solution;                // bandit: the winning arm
    uint32_t pw_solution[4];     // password: solution bits
    uint32_t* d_tick;            // [N] memory: tick | wrong<<16;  password: tick;  stochastic: tick | count<<8
    uint64_t* d_bits;            // [N] memory: the L digits it reads
    uint4* d_guess;              // [N] password: guess bits
    uint32_t* d_mt;              // [625] memory: the global stream mt[624] + idx
    int32_t* d_rank;             // [N] memory: rank among the envs that reset on this send (-1 otherwise)
    uint8_t* d_digits;           // [N * L] memory: digits for ranks 0..R-1
    double* d_gauss;             // [N] bandit: G[j]
    double* d_prox;              // [101*102/2] stochastic: 1 - (p - c/t)**2 at t*(t+1)/2 + c
    double* d_score64;           // [N] fp64 episode score
    unsigned long long* d_agent_stats;   // [4] multiagent: env steps, agent 1 / agent 2 score sums, 0
};

// -- memory RNG -------------------------------------------------------------------------------------------------

// async_reset: env i <- np.random.seed(seed + i); solution = randint(0, 2, size=2L+D), first L digits kept
__global__ void __launch_bounds__(64) k_mem_seed(OceanState st, int n, uint64_t seed_base) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t mt[MT_N];
    mt_seed_genrand(mt, (uint32_t)(seed_base + (uint64_t)i));
    int idx = MT_N;
    uint64_t bits = 0;
    for (int j = 0; j < st.h; ++j) {
        const uint64_t b = mt_next(mt, idx) & 1u;
        if (j < st.L) bits |= b << j;
    }
    st.d_bits[i] = bits;
    if (i == n - 1) {  // the stream every later reset draws from (vector.py:147-149 passes seed=None)
        for (int k = 0; k < MT_N; ++k) st.d_mt[k] = mt[k];
        st.d_mt[MT_N] = (uint32_t)idx;
    }
}

// One block: rank the envs that reset on this send and regenerate their R*(2L+D) outputs of the global stream.
__global__ void __launch_bounds__(PREP_THREADS) k_mem_prepare(OceanState st, int n, const uint8_t* done) {
    __shared__ uint32_t mt[MT_N];
    __shared__ int s_warp[PREP_THREADS / 32];
    const int tid = threadIdx.x;
    const int R = rank_resets<PREP_THREADS>(done, n, st.d_rank, s_warp);
    if (R == 0) return;
    for (int k = tid; k < MT_N; k += PREP_THREADS) mt[k] = st.d_mt[k];
    int idx = (int)st.d_mt[MT_N];   // uniform across the block
    __syncthreads();
    const int64_t total = (int64_t)R * st.h;
    for (int64_t produced = 0; produced < total;) {
        if (idx >= MT_N) {
            mt_twist_block<PREP_THREADS>(mt);
            idx = 0;
        }
        const int take = (int)min((int64_t)(MT_N - idx), total - produced);
        for (int k = tid; k < take; k += PREP_THREADS) {
            const int64_t q = produced + k;
            const int r = (int)(q / st.h), j = (int)(q % st.h);
            if (j < st.L) st.d_digits[(int64_t)r * st.L + j] = (uint8_t)(mt_temper(mt[idx + k]) & 1u);
        }
        produced += take;
        idx += take;
        __syncthreads();   // every read of this state is done before the next twist
    }
    for (int k = tid; k < MT_N; k += PREP_THREADS) st.d_mt[k] = mt[k];
    if (tid == 0) st.d_mt[MT_N] = (uint32_t)idx;
}

// -- password / bandit constants: np.random.seed(42) then the first draws --------------------------------------

__device__ double legacy_double(uint32_t* mt, int& idx) {   // numpy legacy_double / mt19937_next_double
    const int32_t a = (int32_t)(mt_next(mt, idx) >> 5), b = (int32_t)(mt_next(mt, idx) >> 6);
    return __ddiv_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)b), 9007199254740992.0);
}

// One thread: the bandit arm (legacy masked-rejection randint) and the gaussians G[0..n) of numpy's legacy polar
// method (legacy_gauss: the second value of each pair is cached and returned next), fp64 without contraction.
__global__ void k_bandit_init(OceanState st, int n, int* solution_out) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    uint32_t mt[MT_N];
    mt_seed_genrand(mt, 42u);
    int idx = MT_N;
    const uint32_t rng = (uint32_t)(st.n_act - 1);
    uint32_t sol = 0;
    if (rng != 0) {
        uint32_t mask = rng;
        mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
        while ((sol = mt_next(mt, idx) & mask) > rng) {}
    }
    *solution_out = (int)sol;
    for (int j = 0; j < n; j += 2) {
        double x1, x2, r2;
        do {
            x1 = __dadd_rn(__dmul_rn(2.0, legacy_double(mt, idx)), -1.0);
            x2 = __dadd_rn(__dmul_rn(2.0, legacy_double(mt, idx)), -1.0);
            r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));
        } while (r2 >= 1.0 || r2 == 0.0);
        const double f = __dsqrt_rn(__ddiv_rn(__dmul_rn(-2.0, log(r2)), r2));
        st.d_gauss[j] = __dmul_rn(f, x2);
        if (j + 1 < n) st.d_gauss[j + 1] = __dmul_rn(f, x1);
    }
}

// -- step ---------------------------------------------------------------------------------------------------------

struct OcOut {
    char* obs;
    int64_t obs_stride;   // bytes
    float* rewards;
    uint8_t* terminals;
    uint8_t* truncations;
    uint8_t* masks;
    float* dones_f32;
    bool write_const;
};

// Multiagent behind PettingZooPufferEnv: env e owns agent rows 2e (agent 1) and 2e + 1 (agent 2).  Every step ends
// with both agents terminal (ocean.py:163-166, returned unchanged by step), so all_done holds and the next send
// resets: sends alternate between reset rows and step rows.  One lane per env; the caller's warp is whole.
template <int MODE>
__device__ __forceinline__ void multiagent_step(const OceanState& st, int e, bool active,
                                                const int64_t* __restrict__ actions, uint8_t* done, const OcOut& out) {
    const bool step = active && MODE == 1 && !done[e];   // done[e]: all agents' previous rows were terminal
    bool r0 = false, r1 = false;
    if (active) {
        if (step) {            // ocean.py:186-208: agent 1 is rewarded for action 0, agent 2 for action 1
            const int64_t a0 = actions[2 * (int64_t)e], a1 = actions[2 * (int64_t)e + 1];
            r0 = a0 <= 0;      // clamped into [0, 2) like every kind's actions
            r1 = a1 >= 1;
        }
        const int64_t row = 2 * (int64_t)e;
        // the observation is the constant dict {1: [0], 2: [1]}; written on every send because a bound rollout gives
        // every send fresh rows (emulation.py:340-345 reset rows, 395-406 step rows)
        *(float*)(out.obs + row * out.obs_stride) = 0.f;
        *(float*)(out.obs + (row + 1) * out.obs_stride) = 1.f;
        out.rewards[row] = r0 ? 1.f : 0.f;
        out.rewards[row + 1] = r1 ? 1.f : 0.f;
        out.terminals[row] = out.terminals[row + 1] = step ? 1 : 0;
        if (out.write_const) {
            out.truncations[row] = out.truncations[row + 1] = 0;
            out.masks[row] = out.masks[row + 1] = 1;
        }
        if (out.dones_f32) out.dones_f32[row] = out.dones_f32[row + 1] = step ? 1.f : 0.f;
        done[e] = step ? 1 : 0;
    }
    // per-agent statistics (the score info of each agent equals its reward): one integer atomic per warp and quantity
    const unsigned m = __ballot_sync(0xffffffffu, step);
    const unsigned s0 = __ballot_sync(0xffffffffu, r0), s1 = __ballot_sync(0xffffffffu, r1);
    if (m && (threadIdx.x & 31) == 0) {
        atomicAdd(st.d_agent_stats + 0, (unsigned long long)__popc(m));
        if (s0) atomicAdd(st.d_agent_stats + 1, (unsigned long long)__popc(s0));
        if (s1) atomicAdd(st.d_agent_stats + 2, (unsigned long long)__popc(s1));
    }
}

// mode 0: write reset rows for every env (after async_reset); mode 1: vectoriser send (reset-or-step)
template <int KIND, int MODE>
__global__ void __launch_bounds__(128) k_ocean_step(OceanState st, int n, const int64_t* __restrict__ actions,
                                                   uint8_t* done, OcOut out, EpisodeAcc acc) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = e < n;
    if constexpr (KIND == PB_ENV_MULTIAGENT) {
        multiagent_step<MODE>(st, e, active, actions, done, out);   // no EpisodeStats (postprocess.py:147-179)
        return;
    }
    float reward = 0.f;
    double reward_d = 0.0, score = 0.0;
    bool terminal = false, reset_row = true;
    if (active) {
        const bool reset = MODE == 0 || done[e];
        int a = 0;
        if (!reset) {
            reset_row = false;
            a = (int)actions[e];
            const int hi = KIND == PB_ENV_BANDIT ? st.n_act - 1 : 1;
            a = a < 0 ? 0 : (a > hi ? hi : a);
        }
        float* row = (float*)(out.obs + (int64_t)e * out.obs_stride);
        if (KIND == PB_ENV_MEMORY) {
            uint32_t t = 1, wrong = 0;
            uint64_t bits;
            if (reset) {       // ocean.py:87-97: tick 1, obs = solution[0]
                if (MODE == 0) {
                    bits = st.d_bits[e];
                } else {
                    const uint8_t* d = st.d_digits + (int64_t)st.d_rank[e] * st.L;
                    bits = 0;
                    for (int j = 0; j < st.L; ++j) bits |= (uint64_t)d[j] << j;
                    st.d_bits[e] = bits;
                }
                row[0] = (float)(bits & 1u);
            } else {           // ocean.py:99-123
                const uint32_t s = st.d_tick[e];
                t = s & 0xffffu;
                wrong = s >> 16;
                bits = st.d_bits[e];
                float ob = 0.f;
                if ((int)t < st.L) {
                    ob = (float)((bits >> t) & 1u);
                    reward_d = a == 0 ? 1.0 : 0.0;
                }
                if ((int)t >= st.L + st.D) {
                    const int sol = (int)((bits >> (t - st.L - st.D)) & 1u);
                    reward_d = a == sol ? 1.0 : 0.0;
                    wrong |= a != sol;
                }
                t += 1;
                terminal = (int)t == st.h;
                score = wrong ? 0.0 : 1.0;   // np.all(solution[:L] == submission[-L:])
                row[0] = ob;
            }
            st.d_tick[e] = t | (wrong << 16);
        } else if (KIND == PB_ENV_PASSWORD) {
            uint32_t t = 0;
            uint4 g = make_uint4(0, 0, 0, 0);
            if (!reset) {      // ocean.py:266-281
                t = st.d_tick[e];
                g = st.d_guess[e];
                const uint32_t bit = (uint32_t)a << (t & 31), k = t >> 5;   // observation[tick] = action
                g.x |= k == 0 ? bit : 0u; g.y |= k == 1 ? bit : 0u; g.z |= k == 2 ? bit : 0u; g.w |= k == 3 ? bit : 0u;
                t += 1;
                terminal = (int)t == st.L;
                if (terminal) {
                    const bool ok = g.x == st.pw_solution[0] && g.y == st.pw_solution[1] && g.z == st.pw_solution[2]
                                    && g.w == st.pw_solution[3];
                    reward_d = ok ? 1.0 : 0.0;
                    score = reward_d;
                }
            }
            st.d_tick[e] = t;
            st.d_guess[e] = g;
            for (int j = 0; j < st.L; ++j) {   // ocean.py:259: -1 where no guess was made yet
                const uint32_t w = j < 32 ? g.x : (j < 64 ? g.y : (j < 96 ? g.z : g.w));
                row[j] = j < (int)t ? (float)((w >> (j & 31)) & 1u) : -1.f;
            }
        } else if (KIND == PB_ENV_STOCHASTIC) {
            uint32_t t = 0, c = 0;
            if (!reset) {      // ocean.py:562-582
                const uint32_t s = st.d_tick[e];
                t = (s & 0xffu) + 1;
                c = (s >> 8) + (a == 0 ? 1u : 0u);
                terminal = t == STOCH_HORIZON;
                const double frac = __ddiv_rn((double)c, (double)t);
                const double prox = st.d_prox[t * (t + 1) / 2 + c];
                reward_d = ((a == 0 && frac < st.p) || (a == 1 && frac >= st.p)) ? prox : 0.0;
                score = prox;
            }
            st.d_tick[e] = t | (c << 8);
            row[0] = 0.f;
        } else {               // PB_ENV_BANDIT, ocean.py:33-62
            if (!reset) {
                const double correct = a == st.solution ? 1.0 : 0.0;
                reward_d = st.noise != 0.0
                    ? __dmul_rn(__dadd_rn(correct, __dmul_rn(st.d_gauss[e], st.scale)), st.scale)
                    : __dmul_rn(correct, st.scale);
                terminal = true;
                score = correct;
            }
            row[0] = 1.f;
        }
        reward = (float)reward_d;   // fp32 store into buf.rewards (emulation.py:221)
        done[e] = terminal ? 1 : 0;
        out.rewards[e] = reward;
        out.terminals[e] = terminal ? 1 : 0;
        if (out.write_const) out.truncations[e] = 0;
        if (out.write_const) out.masks[e] = 1;
        if (out.dones_f32) out.dones_f32[e] = terminal ? 1.f : 0.f;
    }
    episode_update(acc, e, active, reset_row, reward_d, terminal, score);
}

template <int KIND>
void launch_kind(const OceanState& st, int mode, int n, const int64_t* actions, uint8_t* done, const OcOut& o,
                 const EpisodeAcc& acc, cudaStream_t s) {
    const int blocks = (int)pb_ceil_div(n, 128);
    if (mode == 0)
        k_ocean_step<KIND, 0><<<blocks, 128, 0, s>>>(st, n, actions, done, o, acc);
    else
        k_ocean_step<KIND, 1><<<blocks, 128, 0, s>>>(st, n, actions, done, o, acc);
}

int ocean_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    OceanState* st = (OceanState*)env->kind;
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 4 == 0 && ((uintptr_t)out->obs & 3) == 0, PB_ERR_INVALID,
               "ocean: obs pointer/stride must be 4-byte aligned");
    OcOut o{(char*)out->obs, out->obs_stride, out->rewards, out->terminals, out->truncations, out->masks,
            out->dones_f32, env->write_const};
    const EpisodeAcc acc = pb_episode_acc(env);
    switch (st->kind) {
        case PB_ENV_MEMORY: launch_kind<PB_ENV_MEMORY>(*st, mode, n, actions, env->d_done, o, acc, s); break;
        case PB_ENV_PASSWORD: launch_kind<PB_ENV_PASSWORD>(*st, mode, n, actions, env->d_done, o, acc, s); break;
        case PB_ENV_STOCHASTIC: launch_kind<PB_ENV_STOCHASTIC>(*st, mode, n, actions, env->d_done, o, acc, s); break;
        case PB_ENV_MULTIAGENT: launch_kind<PB_ENV_MULTIAGENT>(*st, mode, n, actions, env->d_done, o, acc, s); break;
        default: launch_kind<PB_ENV_BANDIT>(*st, mode, n, actions, env->d_done, o, acc, s); break;
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int ocean_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    OceanState* st = (OceanState*)env->kind;
    const int n = env->cfg.num_envs;
    const uint64_t base = seed + (uint64_t)env->cfg.env_index_offset;
    if (st->kind == PB_ENV_MEMORY || st->kind == PB_ENV_STOCHASTIC) {
        // np.random.seed(seed + i) raises for seeds outside [0, 2**32)
        PB_REQUIRE(base >= seed && base < (1ull << 32) && base + (uint64_t)(n - 1) < (1ull << 32), PB_ERR_INVALID,
                   "seed %llu + %lld + [0, %d): np.random.seed only takes seeds in [0, 2**32)",
                   (unsigned long long)seed, (long long)env->cfg.env_index_offset, n);
    }
    if (st->kind == PB_ENV_MEMORY) {
        k_mem_seed<<<(int)pb_ceil_div(n, 64), 64, 0, s>>>(*st, n, base);
        PB_LAUNCH_CHECK();
    }
    return ocean_launch(env, 0, nullptr, out, s);
}

int ocean_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    OceanState* st = (OceanState*)env->kind;
    if (st->kind == PB_ENV_MEMORY) {
        k_mem_prepare<<<1, PREP_THREADS, 0, s>>>(*st, env->cfg.num_envs, env->d_done);
        PB_LAUNCH_CHECK();
    }
    return ocean_launch(env, 1, actions, out, s);
}

void ocean_destroy(pb_env* env) {
    OceanState* st = (OceanState*)env->kind;
    if (!st) return;
    cudaFree(st->d_tick); cudaFree(st->d_bits); cudaFree(st->d_guess); cudaFree(st->d_mt); cudaFree(st->d_rank);
    cudaFree(st->d_digits); cudaFree(st->d_gauss); cudaFree(st->d_prox); cudaFree(st->d_score64);
    cudaFree(st->d_agent_stats);
    env->d_row_score64 = nullptr;
    env->d_agent_stats = nullptr;
    delete st;
    env->kind = nullptr;
}

const pb_env_vtable OCEAN_VT = {ocean_reset, ocean_step, ocean_destroy};

}  // namespace

int pb_ocean_create(pb_env* env, const double* dparam, int n_dparam) {
    const int kind = env->cfg.kind;
    const int32_t* ip = env->cfg.iparam;
    const auto dp = [&](int k, double dflt) { return (dparam && k < n_dparam) ? dparam[k] : dflt; };
    OceanState* st = new OceanState();
    env->kind = st;
    env->vt = &OCEAN_VT;
    st->kind = kind;
    const size_t n = (size_t)env->cfg.num_envs;
    int obs_len = 1;
    float lo = -1.f, hi = 1.f;
    st->n_act = 2;
    if (kind == PB_ENV_MEMORY) {
        st->L = ip[0] > 0 ? ip[0] : 2;
        st->D = ip[1] - 1 >= 0 ? ip[1] - 1 : 2;   // iparam[1] = mem_delay + 1 (0 = default)
        PB_REQUIRE(st->L >= 1 && st->L <= MEM_MAX_L, PB_ERR_INVALID, "memory: mem_length must be in [1, %d]",
                   MEM_MAX_L);
        PB_REQUIRE(st->D >= 0 && st->D <= MEM_MAX_D, PB_ERR_INVALID, "memory: mem_delay must be in [0, %d]",
                   MEM_MAX_D);
        st->h = 2 * st->L + st->D;
        PB_CUDA(cudaMalloc(&st->d_bits, n * sizeof(uint64_t)));
        PB_CUDA(cudaMalloc(&st->d_mt, (MT_N + 1) * sizeof(uint32_t)));
        PB_CUDA(cudaMalloc(&st->d_rank, n * sizeof(int32_t)));
        PB_CUDA(cudaMalloc(&st->d_digits, n * st->L));
        PB_CUDA(cudaMemset(st->d_bits, 0, n * sizeof(uint64_t)));
        PB_CUDA(cudaMemset(st->d_mt, 0, (MT_N + 1) * sizeof(uint32_t)));
    } else if (kind == PB_ENV_PASSWORD) {
        st->L = ip[0] > 0 ? ip[0] : 5;
        PB_REQUIRE(st->L >= 1 && st->L <= PW_MAX_L, PB_ERR_INVALID, "password: password_length must be in [1, %d]",
                   PW_MAX_L);
        uint32_t mt[MT_N];   // np.random.seed(42); randint(0, 2, size=L)  (ocean.py:254-261)
        mt_seed_genrand(mt, 42u);
        int idx = MT_N;
        for (int j = 0; j < st->L; ++j) st->pw_solution[j >> 5] |= (mt_next(mt, idx) & 1u) << (j & 31);
        PB_CUDA(cudaMalloc(&st->d_guess, n * sizeof(uint4)));
        PB_CUDA(cudaMemset(st->d_guess, 0, n * sizeof(uint4)));
        obs_len = st->L;
        lo = 0.f;
    } else if (kind == PB_ENV_STOCHASTIC) {
        st->p = dp(0, 0.7);
        PB_REQUIRE(isfinite(st->p), PB_ERR_INVALID, "stochastic: p must be finite");
        std::vector<double> prox((STOCH_HORIZON + 1) * (STOCH_HORIZON + 2) / 2, 0.0);
        const volatile double two = 2.0;   // keeps the compiler from folding pow(x, 2.0) into x * x
        for (int t = 1; t <= STOCH_HORIZON; ++t)
            for (int c = 0; c <= t; ++c)   // python: 1 - (p - count / tick)**2
                prox[t * (t + 1) / 2 + c] = 1.0 - pow(st->p - (double)c / (double)t, two);
        PB_CUDA(cudaMalloc(&st->d_prox, prox.size() * sizeof(double)));
        PB_CUDA(cudaMemcpy(st->d_prox, prox.data(), prox.size() * sizeof(double), cudaMemcpyHostToDevice));
        lo = 0.f;
    } else if (kind == PB_ENV_MULTIAGENT) {   // make_multiagent() takes no arguments (environment.py:69-72)
        for (int k = 0; k < 8; ++k)
            PB_REQUIRE(ip[k] == 0, PB_ERR_INVALID, "multiagent: takes no parameters (iparam[%d] = %d)", k, ip[k]);
        PB_REQUIRE(n_dparam == 0, PB_ERR_INVALID, "multiagent: takes no parameters (%d dparam given)", n_dparam);
        env->agents_per_env = 2;
        PB_CUDA(cudaMalloc(&st->d_agent_stats, 4 * sizeof(unsigned long long)));
        PB_CUDA(cudaMemset(st->d_agent_stats, 0, 4 * sizeof(unsigned long long)));
        env->d_agent_stats = st->d_agent_stats;
        lo = 0.f;              // Box(0, 1, (1,)) for both agents (ocean.py:171-173)
    } else {
        st->n_act = ip[0] > 0 ? ip[0] : 10;
        st->scale = dp(0, 1.0);
        st->noise = dp(1, 1.0);
        PB_REQUIRE(st->n_act >= 1 && st->n_act <= BANDIT_MAX_ARMS, PB_ERR_INVALID,
                   "bandit: num_actions must be in [1, %d]", BANDIT_MAX_ARMS);
        PB_REQUIRE(isfinite(st->scale) && isfinite(st->noise), PB_ERR_INVALID,
                   "bandit: reward_scale and reward_noise must be finite");
        PB_CUDA(cudaMalloc(&st->d_gauss, n * sizeof(double)));
        int* d_sol = nullptr;
        PB_CUDA(cudaMalloc(&d_sol, sizeof(int)));
        k_bandit_init<<<1, 1>>>(*st, (int)n, d_sol);
        PB_LAUNCH_CHECK();
        const cudaError_t err = cudaMemcpy(&st->solution, d_sol, sizeof(int), cudaMemcpyDeviceToHost);
        cudaFree(d_sol);
        PB_CUDA(err);
    }
    if (kind != PB_ENV_MULTIAGENT) {   // multiagent keeps no state but the per-env done flag
        if (kind != PB_ENV_BANDIT) {
            PB_CUDA(cudaMalloc(&st->d_tick, n * sizeof(uint32_t)));
            PB_CUDA(cudaMemset(st->d_tick, 0, n * sizeof(uint32_t)));
        }
        PB_CUDA(cudaMalloc(&st->d_score64, n * sizeof(double)));
        PB_CUDA(cudaMemset(st->d_score64, 0, n * sizeof(double)));
        env->d_row_score64 = st->d_score64;
    }
    env->info.obs_dtype = PB_DTYPE_F32;
    env->info.obs_ndim = 1;
    env->info.obs_shape[0] = obs_len;
    env->info.obs_bytes = (int64_t)obs_len * 4;
    env->info.num_actions = st->n_act;
    env->info.obs_low = lo;
    env->info.obs_high = hi;
    return PB_OK;
}
