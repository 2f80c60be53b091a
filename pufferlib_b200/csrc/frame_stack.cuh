// frame_stack.cuh -- the TMA ring that writes (S,84,84) uint8 frame-stack observation rows, S = 4 (the default) or 1,
// shared by the pixel env kinds (pong: env_pong.cu, breakout_pixels: env_breakout_pixels.cu).  The game is a template
// parameter; the ring, its mbarrier phases, the store / refill order, the reward / flag rows and EpisodeStats are this
// one body.
//
// The 28,224-byte observation row is moved by the TMA engine, never by the LSU: per env one cp.async.bulk pulls the
// three surviving frames of row t-1 (21,168 B) into a shared-memory stage while the CTA renders the new 84x84 frame
// into the same stage, then ONE cp.async.bulk pushes the whole 28,224 B row to row t.  A reset row is one rendered
// frame stored to all 4 slots.  A ring of FS_STAGES stages per CTA keeps 4 envs in flight; 2 CTAs per SM.
// S = 1 (pb_env_config.iparam[6] = 1, the one-frame observation of a recurrent policy) loads nothing: every row is the
// rendered frame, 7,056 B, stored by one cp.async.bulk.
//
// A game G provides
//   G::State                                           per-env SoA state in HBM (passed by value to the kernel)
//   G::Env                                             one env's unpacked state (every thread holds a copy)
//   G::reset(st, e, seed_e, keep_ctr, p)               reset state (keep_ctr: keep the draw counter, the send path)
//   G::step(st, e, action, seed_e, p, reward, terminal, score)   load state and run one step of the dynamics
//   G::render(p, frame, tid)                           all FS_THREADS threads draw the 84x84 frame into shared memory
//   G::store(st, e, p)                                 thread 0 writes the state back
// and, for the Atari preprocessing layer (oracle/SPEC_PIXEL_PREPROCESSING.md), which runs only in the FsPre instances:
//   G::load(st, e, p)                                  load one env's state
//   G::tick(st, p, action, seed_e, reward, terminal, score)   one tick of the dynamics on loaded state (reward: 0 on entry)
//   G::render2(a, b, frame, tid)                       the frame drawn from the objects of both states: the pixel-wise
//                                                      max of render(a) and render(b), in one pass
//   G::NOOP, G::kLives (and G::lives(p) where kLives)  the no-op action; whether the game has lives
// Every thread runs reset / step redundantly on the same inputs (broadcast loads), so no barrier is needed before render.
//
// A game with several agents per env (G::kAgents = A > 1; absent means 1, and the preprocessing layer is single-agent)
// writes A observation rows per env, agent a of env e at row e * A + a, every output row array indexed the same way.
// Its ring items are those rows: a CTA runs the A items of one env back to back, and the dynamics step once per env,
// at item 0, from all A actions, before any of its rows renders; the later items render from the same registers.  So
// no two items load and store one env's state.  Such a game provides, in place of step / render:
//   G::step(st, e, acts, seed_e, p, reward, terminal, score)   acts = the env's A actions; reward is agent 0's
//   G::render(p, frame, tid, a)                        agent a's frame
//   G::seat_reward(reward, a)                          agent a's reward, from agent 0's
//   G::game_over(st, length, score)                    thread 0, where a game ends: the per-agent statistics
#pragma once
#include <type_traits>

#include "env_common.cuh"
#include "tma.cuh"

// A, the agents per env of a frame-stack game: G::kAgents, or 1 where the game has no such member
template <class G, class = void>
struct fs_agents : std::integral_constant<int, 1> {};
template <class G>
struct fs_agents<G, std::void_t<decltype(G::kAgents)>> : std::integral_constant<int, G::kAgents> {};

constexpr int FS_STAGES = 4;
constexpr uint32_t FS_FRAME = 84 * 84;      // 7056 = 441 * 16
constexpr uint32_t FS_ROW = 4 * FS_FRAME;   // 28224
constexpr uint32_t FS_STAGE_BYTES = 28672;  // FS_ROW rounded up to 1 KiB
constexpr int FS_THREADS = 128;
// the stage and the ring of an S-frame row: a stage is S frames rounded up to 1 KiB
template <int S>
constexpr uint32_t FS_STAGE_OF = S == 4 ? FS_STAGE_BYTES : 7168u;
template <int S>
constexpr size_t FS_SMEM_OF = (size_t)FS_STAGES * FS_STAGE_OF<S>;

struct FsOut {
    unsigned char* obs;
    int64_t stride;
    float* rewards;
    uint8_t* terminals;
    uint8_t* truncations;
    uint8_t* masks;
    float* dones_f32;
    bool write_const;
};

static inline FsOut fs_out(const pb_env* env, const pb_env_out* out) {
    return FsOut{(unsigned char*)out->obs, out->obs_stride, out->rewards, out->terminals, out->truncations, out->masks,
                 out->dones_f32, env->write_const};
}

// The Atari preprocessing options of the pixel kinds (pb_env_config.iparam[2..5]; oracle/SPEC_PIXEL_PREPROCESSING.md).
// `word` [N] is the wrapper's per-env word: bit 31 = a soft reset (episodic life) is pending, bits 0..30 = real resets
// since async_reset (the key of the no-op draw).  `ended` [N] = 1 where the row ended a game (only with episodic_life,
// where a terminal row may not have); it is pb_env.d_ended.
struct FsPre {
    uint32_t* word;
    uint8_t* ended;
    int frameskip, noop_max, episodic_life, clip_rewards;
};
constexpr uint32_t FS_SOFT = 0x80000000u;

static inline bool fs_pre_on(const FsPre& p) {
    return p.frameskip > 1 || p.noop_max > 0 || p.episodic_life || p.clip_rewards;
}

// Range check of iparam[2..5] for PONG / BREAKOUT_PIXELS, before anything is allocated.  A skipping game lasts at least
// four full agent steps, one per frame-stack slot: max_ticks >= 4 * frameskip.  No-ops must not end a game:
// noop_max < max_ticks, and pong needs max_score >= 2 (a point takes at least 21 ticks from the serve, so 30 no-op ticks
// hold at most one).
static inline int fs_pre_check(const pb_env_config* cfg) {
    const bool pong = cfg->kind == PB_ENV_PONG;
    const int* ip = cfg->iparam;
    PB_REQUIRE(ip[6] == 0 || ip[6] == 1 || ip[6] == 4, PB_ERR_INVALID, "framestack must be 1 or 4, got %d", ip[6]);
    const int max_ticks = ip[pong ? 1 : 0] > 0 ? ip[pong ? 1 : 0] : 4096;
    const int max_score = ip[0] > 0 ? ip[0] : 5;
    PB_REQUIRE(ip[2] >= 0 && ip[2] <= 8, PB_ERR_INVALID, "frameskip must be in [1, 8], got %d", ip[2]);
    PB_REQUIRE(ip[2] <= 1 || max_ticks >= 4 * ip[2], PB_ERR_INVALID, "frameskip %d needs max_ticks >= %d, got %d", ip[2],
               4 * ip[2], max_ticks);
    PB_REQUIRE(ip[3] >= 0 && ip[3] <= 30 && ip[3] < max_ticks, PB_ERR_INVALID,
               "noop_max must be in [0, 30] and below max_ticks %d, got %d", max_ticks, ip[3]);
    PB_REQUIRE(ip[4] == 0 || (ip[4] == 1 && !pong), PB_ERR_INVALID,
               "episodic_life must be 0 or 1, and 0 for pong (no lives), got %d", ip[4]);
    PB_REQUIRE(ip[5] == 0 || ip[5] == 1, PB_ERR_INVALID, "clip_rewards must be 0 or 1, got %d", ip[5]);
    PB_REQUIRE(!pong || ip[3] == 0 || max_score >= 2, PB_ERR_INVALID, "pong: noop_max needs max_score >= 2");
    return PB_OK;
}

// The frames per observation row, S, of a checked config: iparam[6], 0 = the default 4.
static inline int fs_frames(const pb_env_config* cfg) { return cfg->iparam[6] == 1 ? 1 : 4; }

// Reads the (checked) options; allocates the per-env word, and pb_env.d_ended with episodic_life, when any is set.
static inline int fs_pre_create(pb_env* env, FsPre& pre) {
    const int* ip = env->cfg.iparam;
    pre = FsPre{nullptr, nullptr, ip[2] > 0 ? ip[2] : 1, ip[3], ip[4], ip[5]};
    if (!fs_pre_on(pre)) return PB_OK;
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&pre.word, n * 4));
    PB_CUDA(cudaMemset(pre.word, 0, n * 4));
    if (pre.episodic_life) {
        PB_CUDA(cudaMalloc(&env->d_ended, n));
        PB_CUDA(cudaMemset(env->d_ended, 0, n));
        pre.ended = env->d_ended;
    }
    return PB_OK;
}

static inline void fs_pre_destroy(pb_env* env, FsPre& pre) {
    cudaFree(pre.word);
    cudaFree(env->d_ended);
    pre.word = nullptr;
    env->d_ended = nullptr;
}

#ifdef __CUDACC__
// The no-op count draw of a real reset: its own key, so the game's counter stream is untouched; k = real resets of env
// e since async_reset.
__device__ __forceinline__ int fs_noops(uint64_t seed_e, uint32_t k, int noop_max) {
    const uint32_t r = pb_mix32((seed_e ^ 0x6E6F6F705F726E64ull) * 0x9E3779B97F4A7C15ull +
                                (uint64_t)k * 0xD1B54A32D192ED03ull);
    return 1 + (int)(r % (uint32_t)noop_max);
}

// MODE 0: async_reset;  MODE 1: vectoriser send.  The body of a __launch_bounds__(FS_THREADS) kernel with FS_SMEM_OF<S>
// bytes of dynamic shared memory.  PP: the Atari preprocessing layer (`pre`); PP = false is the plain game, one tick per
// step.  S: frames per row, 4 or 1.
template <int MODE, class G, bool PP = false, int S = 4>
__device__ __forceinline__ void frame_stack_run(const typename G::State& st, int n, const int64_t* __restrict__ actions,
                                                uint8_t* done, const unsigned char* __restrict__ prev, int64_t prev_stride,
                                                const FsOut& out, const EpisodeAcc& acc, FsPre pre = FsPre{}) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bars[FS_STAGES];
    const int tid = threadIdx.x;
    const int64_t step = gridDim.x;
    uint32_t phase[FS_STAGES] = {0, 0, 0, 0};

    static_assert(S == 4 || S == 1, "frame stacks of 4 or 1 frames");
    constexpr int A = fs_agents<G>::value;
    static_assert(A == 1 || !PP, "the preprocessing layer is single-agent");
    constexpr uint32_t STAGE = FS_STAGE_OF<S>;
    auto needs_load = [&](int64_t e) -> bool { return MODE == 1 && done[e] == 0; };
    auto issue_load = [&](int s, int64_t e, int a) {  // thread 0 only; the item of agent a of env e
        if (S == 4 && needs_load(e)) {
            mbar_expect_tx(&bars[s], 3 * FS_FRAME);
            tma_load_1d(smem + (size_t)s * STAGE, prev + (e * A + a) * prev_stride + FS_FRAME, 3 * FS_FRAME, &bars[s]);
        }
    };

    if (tid == 0) {
        for (int s = 0; s < FS_STAGES; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
        int64_t e = blockIdx.x;
        for (int s = 0; s < FS_STAGES && e < n; ++s) {   // item s: agent s % A of the (s / A)-th env
            issue_load(s, e, s % A);
            if ((s + 1) % A == 0) e += step;
        }
    }
    __syncthreads();

    int it = 0;
    for (int64_t e = blockIdx.x; e < n; e += step) {
        // the env's state, stepped at its first item; A > 1: its later items render from it
        typename G::Env p;
        float reward = 0.f, score = 0.f;
        bool terminal = false, loaded_env = false;
#pragma unroll
        for (int seat = 0; seat < A; ++seat, ++it) {
            const int s = it % FS_STAGES;
            unsigned char* buf = smem + (size_t)s * STAGE;
            unsigned char* frame = buf + (S - 1) * FS_FRAME;
            if constexpr (S == 1) {
                // no refill load waits for the bulk store that last read this stage (FS_STAGES iterations ago, the oldest of
                // the groups this thread committed): wait for it here, and let the barrier hold every thread back from
                // rendering into the stage until it has
                if (tid == 0 && it >= FS_STAGES) tma_wait_read<FS_STAGES - 1>();
                __syncthreads();
            }
            // refill the stage that was stored one iteration ago: by now its bulk store has long read shared memory, so
            // this wait does not stall, and the load gets FS_STAGES - 1 iterations of lead time
            if (S == 4 && tid == 0 && it > 0) {
                const int k = seat + FS_STAGES - 1;   // the item FS_STAGES - 1 ahead: k / A envs on, agent k % A
                const int64_t e_next = e + step * (k / A);
                if (e_next < n) {
                    tma_wait_read<0>();
                    issue_load((it - 1) % FS_STAGES, e_next, k % A);
                }
            }
            // ---- integer dynamics, computed redundantly by every thread (same inputs: broadcast loads)
            const uint64_t seed_e = st.seed + (uint64_t)e;
            // false -> this row is a reset row (PP: a real or a soft reset); read once per env, before its item 0
            // writes done[e]
            const bool loaded = (A == 1 || seat == 0) ? needs_load(e) : loaded_env;
            loaded_env = loaded;
            // PP: `raw` / `ticks` = the unclipped reward sum / the game ticks of this row, `ended` = the game ended,
            // `fresh` = a real reset, `word` = the wrapper word to store
            float raw = 0.f;
            int ticks = 0;
            bool ended = false, fresh = !loaded;
            uint32_t word = 0u;
            if constexpr (!PP) {
                if (seat == 0) {
                    if (!loaded) G::reset(st, e, seed_e, MODE == 1, p);
                    else if constexpr (A == 1) G::step(st, e, actions[e], seed_e, p, reward, terminal, score);
                    else G::step(st, e, actions + e * A, seed_e, p, reward, terminal, score);
                }
                // ---- render the new frame into the stage
                if constexpr (A == 1) G::render(p, frame, tid);
                else G::render(p, frame, tid, seat);
            } else {
                const uint32_t w = MODE == 1 ? pre.word[e] : 0u;
                fresh = !loaded && !(w & FS_SOFT);
                typename G::Env q;                 // the state after the second-to-last tick (max-pooling)
                if (fresh) {
                    // reset, then 1 + draw % noop_max ticks of NOOP; the frame is the last tick's
                    G::reset(st, e, seed_e, MODE == 1, p);
                    const int noops = pre.noop_max > 0 ? fs_noops(seed_e, w, pre.noop_max) : 0;
                    for (; ticks < noops; ++ticks) {
                        float r = 0.f;
                        G::tick(st, p, G::NOOP, seed_e, r, ended, score);
                        raw += r;
                    }
                    q = p;
                    word = (w + 1u) & ~FS_SOFT;
                } else {
                    // an agent step, or (soft reset) a NOOP step: up to frameskip ticks, stopping where the game ends
                    G::load(st, e, p);
                    const int a = loaded ? (int)actions[e] : G::NOOP;
                    int lives0 = 0;
                    if constexpr (G::kLives) lives0 = G::lives(p);
                    for (ticks = 0; ticks < pre.frameskip && !ended; ++ticks) {
                        q = p;
                        float r = 0.f;
                        G::tick(st, p, a, seed_e, r, ended, score);
                        raw += r;
                    }
                    if (ticks == 1) q = p;
                    bool life_lost = false;
                    if constexpr (G::kLives) life_lost = loaded && pre.episodic_life && G::lives(p) < lives0 && G::lives(p) > 0;
                    terminal = ended || life_lost;
                    if (loaded) reward = pre.clip_rewards ? (float)((raw > 0.f) - (raw < 0.f)) : raw;
                    word = (w & ~FS_SOFT) | (life_lost && !ended ? FS_SOFT : 0u);
                }
                G::render2(q, p, frame, tid);
            }
            fence_proxy_async_smem();
            __syncthreads();
            // ---- thread 0: bookkeeping + the bulk stores
            if (tid == 0) {
                const int64_t orow = e * A + seat;   // the observation / output row
                float reward_a = reward;
                if constexpr (A > 1) reward_a = G::seat_reward(reward, seat);
                if (seat == 0) {
                    G::store(st, e, p);
                    done[e] = terminal ? 1 : 0;
                }
                out.rewards[orow] = reward_a;
                out.terminals[orow] = terminal ? 1 : 0;
                if (out.write_const) out.truncations[orow] = 0;
                if (out.write_const) out.masks[orow] = 1;
                if (out.dones_f32) out.dones_f32[orow] = terminal ? 1.f : 0.f;
                if constexpr (PP) {
                    pre.word[e] = word;
                    if (pre.ended) pre.ended[e] = ended ? 1 : 0;
                }
                // EpisodeStats (postprocess.py:22-54), scalar form; PP: over every tick of the game, raw rewards, reported
                // where the game ends.  A > 1: per env, from agent 0's rewards, and the game's per-agent statistics
                if (A > 1 && seat != 0) {
                    // an env's statistics are kept at its item 0
                } else if (!PP && !loaded) { acc.ep_return[e] = 0.0; acc.ep_length[e] = 0; }
                else if constexpr (A > 1) {
                    const double ret = acc.ep_return[e] + (double)reward;
                    const int len = acc.ep_length[e] + 1;
                    acc.ep_return[e] = ret; acc.ep_length[e] = len;
                    if (terminal) {
                        acc.row_return[e] = ret; acc.row_length[e] = len; acc.row_score[e] = score;
                        G::game_over(st, len, score);
                    }
                } else {
                    const double ret = PP ? (fresh ? 0.0 : acc.ep_return[e]) + (double)raw : acc.ep_return[e] + (double)reward;
                    const int len = PP ? (fresh ? 0 : acc.ep_length[e]) + ticks : acc.ep_length[e] + 1;
                    acc.ep_return[e] = ret; acc.ep_length[e] = len;
                    if (PP ? ended : terminal) {
                        acc.row_return[e] = ret; acc.row_length[e] = len; acc.row_score[e] = score;
                        double* slot = acc.stats + 4 * (blockIdx.x & (PB_STAT_SLOTS - 1));
                        atomicAdd(slot + 0, 1.0); atomicAdd(slot + 1, ret);
                        atomicAdd(slot + 2, (double)len); atomicAdd(slot + 3, (double)score);
                    }
                }
                unsigned char* row = out.obs + orow * out.stride;
                if (S == 1) {
                    tma_store_1d(row, frame, FS_FRAME);
                } else if (loaded) {
                    mbar_wait(&bars[s], phase[s]);     // the three old frames have landed
                    tma_store_1d(row, buf, FS_ROW);
                } else {
                    for (int k = 0; k < 4; ++k) tma_store_1d(row + (size_t)k * FS_FRAME, frame, FS_FRAME);
                }
                tma_commit();
            }
            if (S == 4 && loaded) phase[s] ^= 1;
            // no trailing barrier: the next iteration uses another stage; this stage is refilled by thread 0 at the top of
            // the next iteration (after wait_read) and rendered into FS_STAGES iterations later, behind block barriers
        }
    }
    if (tid == 0) tma_wait_all<0>();
}

// The obs pointer / stride check and the launch: 2 CTAs per SM, at most one per env.  `k0` / `k1` are the game's MODE 0 / 1
// kernels (__global__ wrappers of frame_stack_run) for S frames per row, `p0` / `p1` its preprocessing instances,
// launched when `pre` sets any option.
template <int S, class State, class K0, class K1, class P0, class P1>
int fs_launch(pb_env* env, int mode, const State& st, const int64_t* actions, const pb_env_out* out, cudaStream_t s,
              K0* k0, K1* k1, P0* p0, P1* p1, const FsPre& pre, const char* who) {
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 16 == 0 && ((uintptr_t)out->obs & 15) == 0, PB_ERR_INVALID,
               "%s: obs pointer/stride must be 16-byte aligned", who);
    const FsOut o = fs_out(env, out);
    constexpr size_t SMEM = FS_SMEM_OF<S>;
    int grid = PB_NUM_SMS * 2;
    if (grid > n) grid = n;
    if (fs_pre_on(pre)) {
        const unsigned char* prev = mode == 0 ? nullptr : (const unsigned char*)env->cur_obs;
        const int64_t prev_stride = mode == 0 ? 0 : env->cur_obs_stride;
        if (mode == 0) {
            PB_CUDA(cudaFuncSetAttribute(p0, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
            p0<<<grid, FS_THREADS, SMEM, s>>>(st, n, actions, env->d_done, prev, prev_stride, o, pb_episode_acc(env), pre);
        } else {
            PB_CUDA(cudaFuncSetAttribute(p1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
            p1<<<grid, FS_THREADS, SMEM, s>>>(st, n, actions, env->d_done, prev, prev_stride, o, pb_episode_acc(env), pre);
        }
    } else if (mode == 0) {
        PB_CUDA(cudaFuncSetAttribute(k0, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
        k0<<<grid, FS_THREADS, SMEM, s>>>(st, n, actions, env->d_done, nullptr, 0, o, pb_episode_acc(env));
    } else {
        PB_CUDA(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
        k1<<<grid, FS_THREADS, SMEM, s>>>(st, n, actions, env->d_done, (const unsigned char*)env->cur_obs,
                                             env->cur_obs_stride, o, pb_episode_acc(env));
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}
#endif
