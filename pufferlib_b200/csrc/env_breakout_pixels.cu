// env_breakout_pixels.cu -- N Breakout instances seen as (4,84,84) (or, framestack=1, (1,84,84)) uint8 frame stacks
// (oracle/SPEC_BREAKOUT_PIXELS.md),
// sm_90a: the policy input of the reference's Atari breakout (atari/environment.py:37-39, NatureCNN at atari/torch.py).
//
// The game is breakout's, step for step: bk_physics and the 28 B of SoA state from env_breakout.cuh, the same RNG,
// rewards, terminals and EpisodeStats score.  The rows are written by the TMA frame-stack ring of frame_stack.cuh (one
// bulk load of the three surviving frames, one bulk store of the 28,224-byte row per env).  The renderer evaluates the
// spec's rule per frame pixel -- the max over the pixel's field rectangle of ball 255 > paddle 192 > brick row gray >
// 0 -- with no zero fill and no scatter: each thread builds whole 16-byte runs of the frame (441 uint4 per frame).
// Bit-exact against oracle/breakout_pixels.py (the breakout oracle of oracle/csrc/envs.c + oracle/csrc/breakout_pixels.c).
#include "env_breakout.cuh"
#include "env_common.cuh"
#include "frame_stack.cuh"

namespace {

struct BkEnv {
    int px, lives, in_play, wait, vx, vy, bx, by, tick;
    uint4 bricks;
    uint32_t ctr;
};

// What a frame row r (field rows [200r/84, 200(r+1)/84): 2 or 3 of them) sees of the objects: whether the ball's and the
// paddle's rows meet it, and the alive bits of the first and last brick row it meets (20 bits, bit = brick column)
// with their gray levels.  A frame row meets at most two brick rows (6 field rows each).
struct BkRowView {
    bool ball, paddle;
    uint32_t bits_a, bits_b;
    uint32_t gray_a, gray_b;
};

__device__ __forceinline__ uint32_t bkp_brick_row_bits(const uint4& b, int row) {
    const int bit = 20 * row, w = bit >> 5, sh = bit & 31;    // 20 bits from word w, spilling into w + 1 (w <= 3)
    const uint32_t lo = w == 0 ? b.x : (w == 1 ? b.y : (w == 2 ? b.z : b.w));
    const uint32_t hi = w == 0 ? b.y : (w == 1 ? b.z : (w == 2 ? b.w : 0u));
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> sh) & 0xFFFFFu;
}

__device__ __forceinline__ BkRowView bkp_row_view(const BkEnv& p, int r) {
    const int y0 = (200 * r) / 84, y1 = (200 * (r + 1)) / 84;
    BkRowView v;
    v.ball = p.by < y1 && p.by + 2 > y0;
    v.paddle = 190 < y1 && 192 > y0;
    v.bits_a = v.bits_b = 0u;
    v.gray_a = v.gray_b = 0u;
    if (y1 > 30 && y0 < 66) {
        const int ra = (max(y0, 30) - 30) / 6, rb = (min(y1, 66) - 1 - 30) / 6;
        v.bits_a = bkp_brick_row_bits(p.bricks, ra);
        v.bits_b = bkp_brick_row_bits(p.bricks, rb);
        v.gray_a = 176u - 16u * (uint32_t)ra;
        v.gray_b = 176u - 16u * (uint32_t)rb;
    }
    return v;
}

// frame pixel (r, c): its field columns [160c/84, 160(c+1)/84) (1 or 2 of them, so at most two brick columns)
__device__ __forceinline__ uint32_t bkp_pixel(const BkEnv& p, const BkRowView& v, int c) {
    const int x0 = (160 * c) / 84, x1 = (160 * (c + 1)) / 84;
    if (v.ball && p.bx < x1 && p.bx + 2 > x0) return 255u;
    if (v.paddle && p.px < x1 && p.px + 24 > x0) return 192u;
    const uint32_t cols = (1u << (x0 >> 3)) | (1u << ((x1 - 1) >> 3));
    if (v.bits_a & cols) return v.gray_a;
    if (v.bits_b & cols) return v.gray_b;
    return 0u;
}

// frame pixel (r, c) of the union of two states' objects (render2): `va` is the row view of a with the OR of both brick
// bitmaps, `vb` that of b (only its ball test is read)
__device__ __forceinline__ uint32_t bkp_pixel2(const BkEnv& a, const BkEnv& b, const BkRowView& va, const BkRowView& vb,
                                               int c) {
    const int x0 = (160 * c) / 84, x1 = (160 * (c + 1)) / 84;
    if ((va.ball && a.bx < x1 && a.bx + 2 > x0) || (vb.ball && b.bx < x1 && b.bx + 2 > x0)) return 255u;
    if (va.paddle && ((a.px < x1 && a.px + 24 > x0) || (b.px < x1 && b.px + 24 > x0))) return 192u;
    const uint32_t cols = (1u << (x0 >> 3)) | (1u << ((x1 - 1) >> 3));
    if (va.bits_a & cols) return va.gray_a;
    if (va.bits_b & cols) return va.gray_b;
    return 0u;
}

// the game behind the frame-stack ring (frame_stack.cuh)
struct BreakoutPixelsGame {
    using State = BreakoutState;
    using Env = BkEnv;

    static __device__ __forceinline__ void reset(const State& st, int64_t e, uint64_t, bool keep_ctr, Env& p) {
        p.ctr = keep_ctr ? st.ctr[e] : 0u;
        p.px = 68; p.lives = 5; p.in_play = 0; p.wait = 0; p.vx = 0; p.vy = 0; p.bx = 79; p.by = 188; p.tick = 0;
        p.bricks = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0x00ffffffu);
    }

    static constexpr int NOOP = 0;
    static constexpr bool kLives = true;

    static __device__ __forceinline__ int lives(const Env& p) { return p.lives; }

    static __device__ __forceinline__ void load(const State& st, int64_t e, Env& p) {
        p.ctr = st.ctr[e];
        bk_unpack(st.s0[e], st.s1[e], p.px, p.lives, p.in_play, p.wait, p.vx, p.vy, p.bx, p.by, p.tick);
        p.bricks = st.bricks[e];
    }

    static __device__ __forceinline__ void tick(const State& st, Env& p, int64_t action, uint64_t seed_e, float& reward,
                                                bool& terminal, float& score) {
        // the game on plain locals (bk_physics picks the bitmap word by pointer: on a struct member that would put the
        // whole Env in local memory)
        uint32_t ctr = p.ctr;
        int px = p.px, lives = p.lives, in_play = p.in_play, wait = p.wait, vx = p.vx, vy = p.vy, bx = p.bx, by = p.by,
            tick = p.tick;
        uint4 bricks = p.bricks;
        int r = 0;
        bk_physics(px, lives, in_play, wait, vx, vy, bx, by, tick, bricks, ctr, (int)action, seed_e, st.max_ticks, r, terminal,
                   score);
        reward = (float)r;
        p.px = px; p.lives = lives; p.in_play = in_play; p.wait = wait; p.vx = vx; p.vy = vy; p.bx = bx; p.by = by;
        p.tick = tick; p.bricks = bricks; p.ctr = ctr;
    }

    static __device__ __forceinline__ void step(const State& st, int64_t e, int64_t action, uint64_t seed_e, Env& p,
                                                float& reward, bool& terminal, float& score) {
        load(st, e, p);
        tick(st, p, action, seed_e, reward, terminal, score);
    }

    // thread k builds the 16-byte runs k, k + 128, ...: frame bytes 16k .. 16k + 15 span frame rows r0 and r0 + 1 at most
    static __device__ __forceinline__ void render(const Env& p, unsigned char* frame, int tid) {
        for (int k = tid; k < (int)(FS_FRAME / 16); k += FS_THREADS) {
            const int r0 = (16 * k) / 84, c0 = 16 * k - 84 * r0;
            const BkRowView v0 = bkp_row_view(p, r0), v1 = bkp_row_view(p, r0 + 1);
            uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = c0 + j;
                const uint32_t px = c < 84 ? bkp_pixel(p, v0, c) : bkp_pixel(p, v1, c - 84);
                w[j >> 2] |= px << (8 * (j & 3));
            }
            reinterpret_cast<uint4*>(frame)[k] = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }

    // render's rule over the objects of both states: two balls, two paddles, the OR of the brick bitmaps (each frame pixel
    // is a max over objects, so this is the pixel-wise max of the two frames)
    static __device__ __forceinline__ void render2(const Env& a, const Env& b, unsigned char* frame, int tid) {
        Env u = a;
        u.bricks = make_uint4(a.bricks.x | b.bricks.x, a.bricks.y | b.bricks.y, a.bricks.z | b.bricks.z,
                              a.bricks.w | b.bricks.w);
        for (int k = tid; k < (int)(FS_FRAME / 16); k += FS_THREADS) {
            const int r0 = (16 * k) / 84, c0 = 16 * k - 84 * r0;
            const BkRowView a0 = bkp_row_view(u, r0), a1 = bkp_row_view(u, r0 + 1);
            const BkRowView b0 = bkp_row_view(b, r0), b1 = bkp_row_view(b, r0 + 1);
            uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = c0 + j;
                const uint32_t px = c < 84 ? bkp_pixel2(u, b, a0, b0, c) : bkp_pixel2(u, b, a1, b1, c - 84);
                w[j >> 2] |= px << (8 * (j & 3));
            }
            reinterpret_cast<uint4*>(frame)[k] = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }

    static __device__ __forceinline__ void store(const State& st, int64_t e, const Env& p) {
        st.s0[e] = bk_pack_s0(p.px, p.lives, p.in_play, p.wait, p.vx, p.vy);
        st.s1[e] = bk_pack_s1(p.bx, p.by, p.tick);
        st.bricks[e] = p.bricks;
        st.ctr[e] = p.ctr;
    }
};

// MODE 0: async_reset;  MODE 1: vectoriser send
template <int MODE, int S>
__global__ void __launch_bounds__(FS_THREADS) k_breakout_pixels(BreakoutState st, int n, const int64_t* __restrict__ actions,
                                                               uint8_t* done, const unsigned char* __restrict__ prev,
                                                               int64_t prev_stride, FsOut out, EpisodeAcc acc) {
    frame_stack_run<MODE, BreakoutPixelsGame, false, S>(st, n, actions, done, prev, prev_stride, out, acc);
}

// the same with the Atari preprocessing layer (oracle/SPEC_PIXEL_PREPROCESSING.md)
template <int MODE, int S>
__global__ void __launch_bounds__(FS_THREADS, 2) k_breakout_pixels_pp(BreakoutState st, int n, const int64_t* __restrict__ actions,
                                                                  uint8_t* done, const unsigned char* __restrict__ prev,
                                                                  int64_t prev_stride, FsOut out, EpisodeAcc acc, FsPre pre) {
    frame_stack_run<MODE, BreakoutPixelsGame, true, S>(st, n, actions, done, prev, prev_stride, out, acc, pre);
}

struct BkpKind {
    BreakoutState st;
    FsPre pre;
    int frames;   // S, 4 or 1
};

int bkp_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    const BkpKind* k = (const BkpKind*)env->kind;
    if (k->frames == 1)
        return fs_launch<1>(env, mode, k->st, actions, out, s, k_breakout_pixels<0, 1>, k_breakout_pixels<1, 1>,
                            k_breakout_pixels_pp<0, 1>, k_breakout_pixels_pp<1, 1>, k->pre, "breakout_pixels");
    return fs_launch<4>(env, mode, k->st, actions, out, s, k_breakout_pixels<0, 4>, k_breakout_pixels<1, 4>,
                        k_breakout_pixels_pp<0, 4>, k_breakout_pixels_pp<1, 4>, k->pre, "breakout_pixels");
}

int bkp_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    BreakoutState* st = &((BkpKind*)env->kind)->st;
    st->seed = seed + (uint64_t)env->cfg.env_index_offset;
    return bkp_launch(env, 0, nullptr, out, s);
}

int bkp_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return bkp_launch(env, 1, actions, out, s);
}

void bkp_destroy(pb_env* env) {
    BkpKind* k = (BkpKind*)env->kind;
    if (!k) return;
    cudaFree(k->st.s0); cudaFree(k->st.s1); cudaFree(k->st.bricks); cudaFree(k->st.ctr);
    fs_pre_destroy(env, k->pre);
    delete k;
    env->kind = nullptr;
}

const pb_env_vtable BREAKOUT_PIXELS_VT = {bkp_reset, bkp_step, bkp_destroy};

}  // namespace

int pb_breakout_pixels_create(pb_env* env) {
    BkpKind* k = new BkpKind();
    BreakoutState* st = &k->st;
    env->kind = k;
    env->vt = &BREAKOUT_PIXELS_VT;
    st->max_ticks = env->cfg.iparam[0] > 0 ? env->cfg.iparam[0] : 4096;
    PB_REQUIRE(st->max_ticks <= 65535, PB_ERR_INVALID, "breakout_pixels: max_ticks must be <= 65535");
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&st->s0, n * 4));
    PB_CUDA(cudaMalloc(&st->s1, n * 4));
    PB_CUDA(cudaMalloc(&st->bricks, n * 16));
    PB_CUDA(cudaMalloc(&st->ctr, n * 4));
    PB_CUDA(cudaMemset(st->s0, 0, n * 4));
    PB_CUDA(cudaMemset(st->s1, 0, n * 4));
    PB_CUDA(cudaMemset(st->bricks, 0, n * 16));
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
    env->info.num_actions = 4;
    env->info.obs_low = 0.f;
    env->info.obs_high = 255.f;
    return PB_OK;
}
