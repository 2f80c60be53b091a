// env_pong.cu -- N Pong instances with (4,84,84) (or, framestack=1, (1,84,84)) uint8 frame-stack observations (oracle/SPEC.md §Pong), sm_90a.
//
// Dynamics are the builder's spec (the reference's pong is ALE behind third-party wrappers: SURVEY.md §0); the
// observation layout (4,84,84) uint8 NCHW, oldest frame first, is the reference's (atari/environment.py:37-39,
// environments/test/mock_environments.py:211) and so are the vectoriser / EpisodeStats conventions
// (vector.py:147-151, emulation.py:187-192, postprocess.py:22-54).  Bit-exact against oracle/csrc/envs.c.
//
// The 28,224-byte observation rows are written by the TMA frame-stack ring of frame_stack.cuh; this file is the game:
// the scripted opponent and the renderer (zero fill + 52 pixel stores); the state and the rest of the dynamics are
// pong_game.cuh's.
#include "env_common.cuh"
#include "frame_stack.cuh"
#include "pong_game.cuh"

namespace {

// the game behind the frame-stack ring (frame_stack.cuh)
struct PongGame {
    using State = PongState;
    using Env = PongEnv;

    static __device__ __forceinline__ void reset(const State& st, int64_t e, uint64_t seed_e, bool keep_ctr, Env& p) {
        pong_reset(st.ctr, e, seed_e, keep_ctr, p);
    }

    static constexpr int NOOP = 0;
    static constexpr bool kLives = false;

    static __device__ __forceinline__ void load(const State& st, int64_t e, Env& p) {
        pong_load(st, e, p);
    }

    static __device__ __forceinline__ void tick(const State& st, Env& p, int64_t action, uint64_t seed_e, float& reward,
                                                bool& terminal, float& score) {
        int a = (int)action;
        a = a < 0 ? 0 : (a > 5 ? 5 : a);
        // dy+3 per action, 3 bits each: NOOP, FIRE -> 0; UP(2,4) -> -3; DOWN(3,5) -> +3   (oracle/SPEC.md §Pong)
        p.ry = min(max(p.ry + (int)((0x30C1Bu >> (3 * a)) & 7u) - 3, 0), 72);
        const int tgt = min(max(p.by - 5, 0), 72);
        if (p.ly < tgt) p.ly = min(p.ly + 2, tgt);
        else if (p.ly > tgt) p.ly = max(p.ly - 2, tgt);
        pong_ball(st, p, seed_e, reward, terminal, score);
    }

    static __device__ __forceinline__ void step(const State& st, int64_t e, int64_t action, uint64_t seed_e, Env& p,
                                                float& reward, bool& terminal, float& score) {
        load(st, e, p);
        tick(st, p, action, seed_e, reward, terminal, score);
    }

    // zero fill, then opponent paddle, agent paddle, ball
    static __device__ __forceinline__ void render(const Env& p, unsigned char* frame, int tid) {
        for (int k = tid; k < (int)(FS_FRAME / 16); k += FS_THREADS) reinterpret_cast<uint4*>(frame)[k] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        if (tid < 24) frame[(p.ly + (tid >> 1)) * 84 + 4 + (tid & 1)] = 128;
        else if (tid < 48) frame[(p.ry + ((tid - 24) >> 1)) * 84 + 78 + (tid & 1)] = 192;
        __syncthreads();   // ball is drawn last (it may overlap a paddle pixel)
        if (tid < 4) {
            const int x = p.bx + (tid & 1), y = p.by + (tid >> 1);
            if (x >= 0 && x < 84 && y >= 0 && y < 84) frame[y * 84 + x] = 255;
        }
    }

    // render's rule over the objects of both states (every pixel is the max over the objects covering it: 128 < 192 <
    // 255, drawn in that order): four paddles, then two balls
    static __device__ __forceinline__ void render2(const Env& a, const Env& b, unsigned char* frame, int tid) {
        for (int k = tid; k < (int)(FS_FRAME / 16); k += FS_THREADS) reinterpret_cast<uint4*>(frame)[k] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        const bool pa = tid < 48;                        // fields picked by value: a pointer pick puts Env in local memory
        const int t = pa ? tid : tid - 48, ly = pa ? a.ly : b.ly, ry = pa ? a.ry : b.ry;
        if (t < 24) frame[(ly + (t >> 1)) * 84 + 4 + (t & 1)] = 128;
        else if (t < 48) frame[(ry + ((t - 24) >> 1)) * 84 + 78 + (t & 1)] = 192;
        __syncthreads();
        if (tid < 8) {
            const int x = (tid < 4 ? a.bx : b.bx) + (tid & 1), y = (tid < 4 ? a.by : b.by) + ((tid >> 1) & 1);
            if (x >= 0 && x < 84 && y >= 0 && y < 84) frame[y * 84 + x] = 255;
        }
    }

    static __device__ __forceinline__ void store(const State& st, int64_t e, const Env& p) {
        pong_store(st, e, p);
    }
};

// MODE 0: async_reset;  MODE 1: vectoriser send;  S frames per row
template <int MODE, int S>
__global__ void __launch_bounds__(FS_THREADS) k_pong(PongState st, int n, const int64_t* __restrict__ actions,
                                                    uint8_t* done, const unsigned char* __restrict__ prev,
                                                    int64_t prev_stride, FsOut out, EpisodeAcc acc) {
    frame_stack_run<MODE, PongGame, false, S>(st, n, actions, done, prev, prev_stride, out, acc);
}

// the same with the Atari preprocessing layer (oracle/SPEC_PIXEL_PREPROCESSING.md)
template <int MODE, int S>
__global__ void __launch_bounds__(FS_THREADS, 2) k_pong_pp(PongState st, int n, const int64_t* __restrict__ actions,
                                                       uint8_t* done, const unsigned char* __restrict__ prev,
                                                       int64_t prev_stride, FsOut out, EpisodeAcc acc, FsPre pre) {
    frame_stack_run<MODE, PongGame, true, S>(st, n, actions, done, prev, prev_stride, out, acc, pre);
}

struct PongKind {
    PongState st;
    FsPre pre;
    int frames;   // S, 4 or 1
};

int pong_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    const PongKind* k = (const PongKind*)env->kind;
    if (k->frames == 1)
        return fs_launch<1>(env, mode, k->st, actions, out, s, k_pong<0, 1>, k_pong<1, 1>, k_pong_pp<0, 1>, k_pong_pp<1, 1>,
                            k->pre, "pong");
    return fs_launch<4>(env, mode, k->st, actions, out, s, k_pong<0, 4>, k_pong<1, 4>, k_pong_pp<0, 4>, k_pong_pp<1, 4>,
                        k->pre, "pong");
}

int pong_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    PongState* st = &((PongKind*)env->kind)->st;
    st->seed = seed + (uint64_t)env->cfg.env_index_offset;
    return pong_launch(env, 0, nullptr, out, s);
}

int pong_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return pong_launch(env, 1, actions, out, s);
}

void pong_destroy(pb_env* env) {
    PongKind* k = (PongKind*)env->kind;
    if (!k) return;
    cudaFree(k->st.s0); cudaFree(k->st.s1); cudaFree(k->st.ctr);
    fs_pre_destroy(env, k->pre);
    delete k;
    env->kind = nullptr;
}

const pb_env_vtable PONG_VT = {pong_reset, pong_step, pong_destroy};

}  // namespace

int pb_pong_create(pb_env* env) {
    PongKind* k = new PongKind();
    PongState* st = &k->st;
    env->kind = k;
    env->vt = &PONG_VT;
    st->max_score = env->cfg.iparam[0] > 0 ? env->cfg.iparam[0] : 5;
    st->max_ticks = env->cfg.iparam[1] > 0 ? env->cfg.iparam[1] : 4096;
    PB_REQUIRE(st->max_score <= 15 && st->max_ticks <= 65535, PB_ERR_INVALID,
               "pong: max_score must be <= 15 and max_ticks <= 65535");
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&st->s0, n * 4));
    PB_CUDA(cudaMalloc(&st->s1, n * 4));
    PB_CUDA(cudaMalloc(&st->ctr, n * 4));
    PB_CUDA(cudaMemset(st->s0, 0, n * 4));
    PB_CUDA(cudaMemset(st->s1, 0, n * 4));
    PB_CUDA(cudaMemset(st->ctr, 0, n * 4));
    const int rc = fs_pre_create(env, k->pre);
    if (rc != PB_OK) return rc;
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
