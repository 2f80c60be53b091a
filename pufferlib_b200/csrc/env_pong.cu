// env_pong.cu -- N Pong instances with (4,84,84) uint8 frame-stack observations (oracle/SPEC.md §Pong), sm_90a.
//
// Dynamics are the builder's spec (the reference's pong is ALE behind third-party wrappers: SURVEY.md §0); the
// observation layout (4,84,84) uint8 NCHW, oldest frame first, is the reference's (atari/environment.py:37-39,
// environments/test/mock_environments.py:211) and so are the vectoriser / EpisodeStats conventions
// (vector.py:147-151, emulation.py:187-192, postprocess.py:22-54).  Bit-exact against oracle/csrc/envs.c.
//
// The 28,224-byte observation rows are written by the TMA frame-stack ring of frame_stack.cuh; this file is the game:
// the integer dynamics and the renderer (zero fill + 52 pixel stores).  Per-env state is 12 B of SoA.
#include "env_common.cuh"
#include "frame_stack.cuh"

namespace {

struct PongState {
    uint32_t* s0;   // ly(8) | ry(8)<<8 | (bx+2)(8)<<16 | (by)(8)<<24
    uint32_t* s1;   // (vx+2)(3) | (vy+2)(3)<<3 | score_l(4)<<6 | score_r(4)<<10 | tick(16)<<16
    uint32_t* ctr;
    uint64_t seed;
    int max_score, max_ticks;
};

struct PongEnv {
    int ly, ry, bx, by, vx, vy, score_l, score_r, tick;
    uint32_t ctr;
};

__device__ __forceinline__ void pong_serve(PongEnv& s, uint64_t seed_e) {
    const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull + (uint64_t)s.ctr * 0xD1B54A32D192ED03ull);
    s.ctr += 1;
    s.bx = 41; s.by = 41;
    s.vx = (r & 1u) ? 2 : -2;
    s.vy = (int)((r >> 1) % 5u) - 2;
}

// the game behind the frame-stack ring (frame_stack.cuh)
struct PongGame {
    using State = PongState;
    using Env = PongEnv;

    static __device__ __forceinline__ void reset(const State& st, int64_t e, uint64_t seed_e, bool keep_ctr, Env& p) {
        p.ctr = keep_ctr ? st.ctr[e] : 0u;
        p.ly = 36; p.ry = 36; p.score_l = 0; p.score_r = 0; p.tick = 0;
        pong_serve(p, seed_e);
    }

    static __device__ __forceinline__ void step(const State& st, int64_t e, int64_t action, uint64_t seed_e, Env& p,
                                                float& reward, bool& terminal, float& score) {
        const uint32_t a0 = st.s0[e], a1 = st.s1[e];
        p.ly = a0 & 0xff; p.ry = (a0 >> 8) & 0xff; p.bx = (int)((a0 >> 16) & 0xff) - 2; p.by = (a0 >> 24) & 0xff;
        p.vx = (int)(a1 & 7) - 2; p.vy = (int)((a1 >> 3) & 7) - 2;
        p.score_l = (a1 >> 6) & 15; p.score_r = (a1 >> 10) & 15; p.tick = a1 >> 16;
        p.ctr = st.ctr[e];
        int a = (int)action;
        a = a < 0 ? 0 : (a > 5 ? 5 : a);
        // dy+3 per action, 3 bits each: NOOP, FIRE -> 0; UP(2,4) -> -3; DOWN(3,5) -> +3   (oracle/SPEC.md §Pong)
        p.ry = min(max(p.ry + (int)((0x30C1Bu >> (3 * a)) & 7u) - 3, 0), 72);
        const int tgt = min(max(p.by - 5, 0), 72);
        if (p.ly < tgt) p.ly = min(p.ly + 2, tgt);
        else if (p.ly > tgt) p.ly = max(p.ly - 2, tgt);
        p.bx += p.vx; p.by += p.vy;
        if (p.by < 0) { p.by = -p.by; p.vy = -p.vy; }
        if (p.by > 82) { p.by = 164 - p.by; p.vy = -p.vy; }
        if (p.vx > 0 && p.bx >= 76 && p.bx <= 78 && p.by + 2 > p.ry && p.by < p.ry + 12) {
            p.vx = -2; p.bx = 76; p.vy = (p.by + 1 - p.ry - 6) / 3;
        } else if (p.vx < 0 && p.bx >= 4 && p.bx <= 6 && p.by + 2 > p.ly && p.by < p.ly + 12) {
            p.vx = 2; p.bx = 6; p.vy = (p.by + 1 - p.ly - 6) / 3;
        }
        if (p.bx < 0) { p.score_r += 1; reward = 1.f; pong_serve(p, seed_e); }
        else if (p.bx > 82) { p.score_l += 1; reward = -1.f; pong_serve(p, seed_e); }
        p.tick += 1;
        terminal = p.score_l >= st.max_score || p.score_r >= st.max_score || p.tick >= st.max_ticks;
        score = (float)(p.score_r - p.score_l);
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

    static __device__ __forceinline__ void store(const State& st, int64_t e, const Env& p) {
        st.s0[e] = (uint32_t)p.ly | ((uint32_t)p.ry << 8) | ((uint32_t)(p.bx + 2) << 16) | ((uint32_t)p.by << 24);
        st.s1[e] = (uint32_t)(p.vx + 2) | ((uint32_t)(p.vy + 2) << 3) | ((uint32_t)p.score_l << 6) |
                   ((uint32_t)p.score_r << 10) | ((uint32_t)p.tick << 16);
        st.ctr[e] = p.ctr;
    }
};

// MODE 0: async_reset;  MODE 1: vectoriser send
template <int MODE>
__global__ void __launch_bounds__(FS_THREADS) k_pong(PongState st, int n, const int64_t* __restrict__ actions,
                                                    uint8_t* done, const unsigned char* __restrict__ prev,
                                                    int64_t prev_stride, FsOut out, EpisodeAcc acc) {
    frame_stack_run<MODE, PongGame>(st, n, actions, done, prev, prev_stride, out, acc);
}

int pong_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return fs_launch(env, mode, *(PongState*)env->kind, actions, out, s, k_pong<0>, k_pong<1>, "pong");
}

int pong_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    PongState* st = (PongState*)env->kind;
    st->seed = seed + (uint64_t)env->cfg.env_index_offset;
    return pong_launch(env, 0, nullptr, out, s);
}

int pong_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return pong_launch(env, 1, actions, out, s);
}

void pong_destroy(pb_env* env) {
    PongState* st = (PongState*)env->kind;
    if (!st) return;
    cudaFree(st->s0); cudaFree(st->s1); cudaFree(st->ctr);
    delete st;
    env->kind = nullptr;
}

const pb_env_vtable PONG_VT = {pong_reset, pong_step, pong_destroy};

}  // namespace

int pb_pong_create(pb_env* env) {
    PongState* st = new PongState();
    env->kind = st;
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
    env->info.obs_dtype = PB_DTYPE_U8;
    env->info.obs_ndim = 3;
    env->info.obs_shape[0] = 4;
    env->info.obs_shape[1] = 84;
    env->info.obs_shape[2] = 84;
    env->info.obs_bytes = FS_ROW;
    env->info.num_actions = 6;
    env->info.obs_low = 0.f;
    env->info.obs_high = 255.f;
    return PB_OK;
}
