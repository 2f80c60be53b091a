// env_pong_versus.cu -- N two-player Pong instances from pixels (oracle/SPEC_PONG_VERSUS.md), sm_90a: pong's game with
// the scripted left paddle replaced by a second agent, two agent rows per env (row e*2 + a), each an (S,84,84) uint8
// frame stack, S = 4 or 1, seen from that agent's side, so one shared policy plays both seats (self-play).
//
// The state (12 B of SoA per env), its packing, the ball and the serve are pong's (pong_game.cuh).  Agent 0 is the
// right paddle (ry) and sees pong's frame; agent 1 is the left paddle (ly) and sees the field mirrored in x with the
// paddle values swapped, so its own paddle is 192 on the right, as agent 0's is.  Rewards are zero-sum.
// Bit-exact against oracle/pong_versus.py (the restatement in oracle/csrc/pong_versus.c).
//
// Design: the rows are written by the TMA frame-stack ring of frame_stack.cuh with its ring items being agent rows
// (kAgents = 2).  The two items of one env run back to back in one CTA: item 0 steps the dynamics once, from both
// actions, and renders agent 0's row; item 1 renders agent 1's row from the same registers.  The alternative, one ring
// item per env whose stage holds both rows, needs 56 KiB stages at S = 4: four of them are 225 KiB, one CTA per SM
// with no room for a second, or two stages per CTA and half the loads in flight.  Items of one row each keep pong's
// 28 KiB (S = 4) or 7 KiB (S = 1) stages, its 2 CTAs per SM and its load lead of three items; the cost is that the
// ring holds two envs instead of four.  Neither item loads or stores state the other wrote, and no env's items ever
// run in two CTAs.
//
// ptxas (sm_90a, -O3) for k_pong_versus<MODE, S>: <0,4> 22 registers, <1,4> 38, <0,1> 22, <1,1> 30; no spills; <1,4>
// keeps its four mbarrier phase words in a 16-byte stack frame, as k_pong<1,4> does (40 registers).  128 B of static
// shared memory plus the ring, 112 KiB (S = 4) or 28 KiB (S = 1) of dynamic shared memory per CTA: 2 CTAs per SM.
#include "env_common.cuh"
#include "frame_stack.cuh"
#include "pong_game.cuh"

namespace {

struct PongVersusState : PongState {   // pong's state and seed
    unsigned long long* agent_stats;   // [4]: games ended, agent 0's and agent 1's score sums (two's complement),
                                       // game lengths in ticks
};

struct PongVersusGame {
    using State = PongVersusState;
    using Env = PongEnv;
    static constexpr int kAgents = 2;

    static __device__ __forceinline__ void reset(const State& st, int64_t e, uint64_t seed_e, bool keep_ctr, Env& p) {
        pong_reset(st.ctr, e, seed_e, keep_ctr, p);
    }

    // both paddles move (agent 0 = right, agent 1 = left), then the ball; reward and score are agent 0's
    static __device__ __forceinline__ void step(const State& st, int64_t e, const int64_t* acts, uint64_t seed_e, Env& p,
                                                float& reward, bool& terminal, float& score) {
        pong_load(st, e, p);
        p.ry = pong_paddle(p.ry, acts[0]);
        p.ly = pong_paddle(p.ly, acts[1]);
        pong_ball(st, p, seed_e, reward, terminal, score);
    }

    // zero fill, then the opponent's paddle (128, x = 4..5), the agent's own paddle (192, x = 78..79), the ball.  Agent 1
    // sees the field mirrored in x (column c -> 83 - c): its own paddle ly on the right, the ball's left edge at 82 - bx.
    // The ball is always inside the field after a step or a serve (0 <= bx, by <= 82), so the clip below never cuts it.
    static __device__ __forceinline__ void render(const Env& p, unsigned char* frame, int tid, int seat) {
        const int own = seat == 0 ? p.ry : p.ly, opp = seat == 0 ? p.ly : p.ry, bx = seat == 0 ? p.bx : 82 - p.bx;
        for (int k = tid; k < (int)(FS_FRAME / 16); k += FS_THREADS) reinterpret_cast<uint4*>(frame)[k] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        if (tid < 24) frame[(opp + (tid >> 1)) * 84 + 4 + (tid & 1)] = 128;
        else if (tid < 48) frame[(own + ((tid - 24) >> 1)) * 84 + 78 + (tid & 1)] = 192;
        __syncthreads();   // the ball is drawn last (it may overlap a paddle pixel)
        if (tid < 4) {
            const int x = bx + (tid & 1), y = p.by + (tid >> 1);
            if (x >= 0 && x < 84 && y >= 0 && y < 84) frame[y * 84 + x] = 255;
        }
    }

    // zero-sum; 0 - r keeps a zero reward +0.0f
    static __device__ __forceinline__ float seat_reward(float reward, int seat) { return seat == 0 ? reward : 0.f - reward; }

    // thread 0, where a game ends: score = agent 0's points minus agent 1's, agent 1's score is its negation
    static __device__ __forceinline__ void game_over(const State& st, int length, float score) {
        const long long s = (long long)score;
        atomicAdd(st.agent_stats + 0, 1ull);
        atomicAdd(st.agent_stats + 1, (unsigned long long)s);
        atomicAdd(st.agent_stats + 2, (unsigned long long)-s);
        atomicAdd(st.agent_stats + 3, (unsigned long long)length);
    }

    static __device__ __forceinline__ void store(const State& st, int64_t e, const Env& p) {
        pong_store(st, e, p);
    }
};

// MODE 0: async_reset;  MODE 1: vectoriser send;  S frames per row
template <int MODE, int S>
__global__ void __launch_bounds__(FS_THREADS) k_pong_versus(PongVersusState st, int n,
                                                            const int64_t* __restrict__ actions, uint8_t* done,
                                                            const unsigned char* __restrict__ prev, int64_t prev_stride,
                                                            FsOut out, EpisodeAcc acc) {
    frame_stack_run<MODE, PongVersusGame, false, S>(st, n, actions, done, prev, prev_stride, out, acc);
}

struct PongVersusKind {
    PongVersusState st;
    int frames;   // S, 4 or 1
};

template <int S>
int versus_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    const PongVersusKind* k = (const PongVersusKind*)env->kind;
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 16 == 0 && ((uintptr_t)out->obs & 15) == 0, PB_ERR_INVALID,
               "pong_versus: obs pointer/stride must be 16-byte aligned");
    const FsOut o = fs_out(env, out);
    constexpr size_t SMEM = FS_SMEM_OF<S>;
    int grid = PB_NUM_SMS * 2;   // 2 CTAs per SM, at most one per env
    if (grid > n) grid = n;
    auto* kern = mode == 0 ? k_pong_versus<0, S> : k_pong_versus<1, S>;
    PB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
    kern<<<grid, FS_THREADS, SMEM, s>>>(k->st, n, actions, env->d_done, mode == 0 ? nullptr : (const unsigned char*)env->cur_obs,
                                        mode == 0 ? 0 : env->cur_obs_stride, o, pb_episode_acc(env));
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int versus_launch_any(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return ((const PongVersusKind*)env->kind)->frames == 1 ? versus_launch<1>(env, mode, actions, out, s)
                                                           : versus_launch<4>(env, mode, actions, out, s);
}

int versus_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    PongVersusKind* k = (PongVersusKind*)env->kind;
    k->st.seed = seed + (uint64_t)env->cfg.env_index_offset;
    return versus_launch_any(env, 0, nullptr, out, s);
}

int versus_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return versus_launch_any(env, 1, actions, out, s);
}

void versus_destroy(pb_env* env) {
    PongVersusKind* k = (PongVersusKind*)env->kind;
    if (!k) return;
    cudaFree(k->st.s0); cudaFree(k->st.s1); cudaFree(k->st.ctr); cudaFree(k->st.agent_stats);
    env->d_agent_stats = nullptr;
    delete k;
    env->kind = nullptr;
}

const pb_env_vtable PONG_VERSUS_VT = {versus_reset, versus_step, versus_destroy};

}  // namespace

// iparam: [0] = max_score in [1, 15] (0 = 5), [1] = max_ticks in [1, 65535] (0 = 4096), [6] = framestack 1 or 4 (0 = 4);
// everything else 0: the Atari preprocessing options (iparam[2..5]) are single-agent.  Checked before any allocation.
int pb_pong_versus_check(const pb_env_config* cfg) {
    const int* ip = cfg->iparam;
    PB_REQUIRE(ip[0] >= 0 && ip[0] <= 15, PB_ERR_INVALID, "pong_versus: max_score must be in [1, 15], got %d", ip[0]);
    PB_REQUIRE(ip[1] >= 0 && ip[1] <= 65535, PB_ERR_INVALID, "pong_versus: max_ticks must be in [1, 65535], got %d",
               ip[1]);
    PB_REQUIRE(ip[6] == 0 || ip[6] == 1 || ip[6] == 4, PB_ERR_INVALID, "pong_versus: framestack must be 1 or 4, got %d",
               ip[6]);
    for (int k = 2; k < 8; ++k)
        PB_REQUIRE(k == 6 || ip[k] == 0, PB_ERR_INVALID,
                   "pong_versus: iparam[%d] = %d: the Atari preprocessing options are not supported", k, ip[k]);
    return PB_OK;
}

int pb_pong_versus_create(pb_env* env) {
    PongVersusKind* k = new PongVersusKind();
    PongState* st = &k->st;
    env->kind = k;
    env->vt = &PONG_VERSUS_VT;
    st->max_score = env->cfg.iparam[0] > 0 ? env->cfg.iparam[0] : 5;
    st->max_ticks = env->cfg.iparam[1] > 0 ? env->cfg.iparam[1] : 4096;
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&st->s0, n * 4));
    PB_CUDA(cudaMalloc(&st->s1, n * 4));
    PB_CUDA(cudaMalloc(&st->ctr, n * 4));
    PB_CUDA(cudaMemset(st->s0, 0, n * 4));
    PB_CUDA(cudaMemset(st->s1, 0, n * 4));
    PB_CUDA(cudaMemset(st->ctr, 0, n * 4));
    PB_CUDA(cudaMalloc(&k->st.agent_stats, 4 * sizeof(unsigned long long)));
    PB_CUDA(cudaMemset(k->st.agent_stats, 0, 4 * sizeof(unsigned long long)));
    env->d_agent_stats = k->st.agent_stats;
    env->agents_per_env = 2;
    k->frames = fs_frames(&env->cfg);
    env->info.obs_dtype = PB_DTYPE_U8;
    env->info.obs_ndim = 3;
    env->info.obs_shape[0] = k->frames;
    env->info.obs_shape[1] = 84;
    env->info.obs_shape[2] = 84;
    env->info.obs_bytes = k->frames * FS_FRAME;
    env->info.num_actions = 6;
    env->info.obs_low = 0.f;
    env->info.obs_high = 255.f;
    return PB_OK;
}
