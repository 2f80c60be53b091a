// env_snake.cu -- N Snake instances (oracle/SPEC.md §Snake) behind the reference vectoriser semantics (sm_90a).
//
// Dynamics are the builder's spec (no snake exists in the reference: SURVEY.md §0); vectoriser / EpisodeStats
// conventions are the reference's (vector.py:147-151, emulation.py:187-192, postprocess.py:22-54).  Bit-exact
// against oracle/csrc/envs.c.
//
// The 16x16 uint8 observation IS the state: body cells carry their remaining life, so a step is "read row t-1,
// write row t" and nothing else but 12 B of scalars per env.  Half a warp (16 lanes) owns one env: lane y holds
// board row y as one uint4 (16 cells), i.e. an env row is ONE coalesced 256 B load and ONE coalesced 256 B store.
// Body decay is byte-SIMD (__vcmp*4 / __vsub4) on the 4 words of the lane; the target-cell probe and the
// "k-th empty cell" food placement are 16-lane shuffles (popcount + prefix sum), no loops over the board.
#include "env_common.cuh"

namespace {

struct SnakeState {
    uint32_t* s0;   // head(8) | dir(2)<<8 | len(8)<<16
    uint32_t* s1;   // tick(16)
    uint32_t* ctr;
    uint64_t seed;
    int max_ticks;
};

struct SnOut {
    uint8_t* obs;
    int64_t stride;
    float* rewards;
    uint8_t* terminals;
    uint8_t* truncations;
    uint8_t* masks;
    float* dones_f32;
    bool write_const;
};

__device__ __forceinline__ uint32_t get_word(const uint4& v, int i) {
    return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}
__device__ __forceinline__ void set_byte(uint4& v, int x, uint32_t val) {
    const uint32_t sh = (x & 3) * 8, m = ~(0xffu << sh), b = val << sh;
    switch (x >> 2) {
        case 0: v.x = (v.x & m) | b; break;
        case 1: v.y = (v.y & m) | b; break;
        case 2: v.z = (v.z & m) | b; break;
        default: v.w = (v.w & m) | b; break;
    }
}
__device__ __forceinline__ uint32_t zero_bytes(uint32_t w) { return __vcmpeq4(w, 0u) & 0x01010101u; }

// Place food (255) on the k-th empty cell in index order; 16 lanes cooperate (sub = lane within the group).
__device__ __forceinline__ void place_food(uint4& v, int sub, unsigned gmask, uint32_t k) {
    const int cnt = __popc(zero_bytes(v.x)) + __popc(zero_bytes(v.y)) + __popc(zero_bytes(v.z)) +
                    __popc(zero_bytes(v.w));
    int incl = cnt;
#pragma unroll
    for (int off = 1; off < 16; off <<= 1) {
        const int y = __shfl_up_sync(gmask, incl, off, 16);
        if (sub >= off) incl += y;
    }
    const int excl = incl - cnt;
    if ((int)k >= excl && (int)k < incl) {
        int r = (int)k - excl;
#pragma unroll
        for (int x = 0; x < 16; ++x) {
            const uint32_t b = (get_word(v, x >> 2) >> ((x & 3) * 8)) & 0xffu;
            if (b == 0u) {
                if (r == 0) { set_byte(v, x, 255u); r = -1; }
                else if (r > 0) --r;
            }
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(128) k_snake(SnakeState st, int n, const int64_t* __restrict__ actions,
                                              uint8_t* done, const uint8_t* __restrict__ prev, int64_t prev_stride,
                                              SnOut out, EpisodeAcc acc) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int e = tid >> 4, sub = tid & 15;
    const int lane = threadIdx.x & 31;
    const unsigned gmask = 0xffffu << (lane & 16);   // the 16 lanes of this env
    const bool valid = e < n;
    const bool leader = valid && sub == 0;
    uint4 v = make_uint4(0, 0, 0, 0);
    int head = 136, dir = 3, len = 2, tick = 0;
    uint32_t ctr = 0;
    float reward = 0.f;
    bool terminal = false, reset_row = true;
    if (valid) {
        const uint64_t seed_e = st.seed + (uint64_t)e;
        bool do_reset = true;
        uint32_t a0 = 0, a1 = 0;
        uint4 v_prev = v;
        int a = 0;
        if (MODE == 1) {   // every load is issued before the `done` branch: one DRAM latency, not two
            v_prev = *reinterpret_cast<const uint4*>(prev + (int64_t)e * prev_stride + sub * 16);
            ctr = st.ctr[e];
            a0 = st.s0[e]; a1 = st.s1[e];
            a = (int)actions[e];
            do_reset = done[e] != 0;
        }
        if (do_reset) {
            if (sub == 8) { set_byte(v, 8, 254u); set_byte(v, 7, 1u); }
            const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull + (uint64_t)ctr * 0xD1B54A32D192ED03ull);
            ctr += 1;
            place_food(v, sub, gmask, r % 254u);
        } else {
            reset_row = false;
            head = a0 & 0xff; dir = (a0 >> 8) & 3; len = (a0 >> 16) & 0xff; tick = a1 & 0xffff;
            v = v_prev;
            a = a < 0 ? 0 : (a > 3 ? 3 : a);
            if (a != (dir ^ 1)) dir = a;
            const int x = head & 15, y = head >> 4;
            const int nx = x + (dir == 3) - (dir == 2), ny = y + (dir == 1) - (dir == 0);
            bool dead = nx < 0 || nx > 15 || ny < 0 || ny > 15;
            const int cx = dead ? 0 : nx, cy = dead ? 0 : ny;
            const uint32_t mine = (get_word(v, cx >> 2) >> ((cx & 3) * 8)) & 0xffu;
            const uint32_t q = __shfl_sync(gmask, mine, cy, 16);
            if (!dead && q >= 2u && q <= 250u) dead = true;
            if (dead) {
                reward = -1.f;
                terminal = true;
            } else {
                const bool eat = q == 255u;
                if (eat) {
                    len += 1;
                    reward = 1.f;
                } else {  // every body value in [1,250] decays by one (byte SIMD)
#define SNAKE_DECAY(w) { const uint32_t m = __vcmpgeu4(w, 0x01010101u) & __vcmpleu4(w, 0xFAFAFAFAu); \
                         w = __vsub4(w, m & 0x01010101u); }
                    SNAKE_DECAY(v.x) SNAKE_DECAY(v.y) SNAKE_DECAY(v.z) SNAKE_DECAY(v.w)
#undef SNAKE_DECAY
                }
                if (sub == y) set_byte(v, x, (uint32_t)(len - 1));
                if (sub == ny) set_byte(v, nx, 254u);
                head = ny * 16 + nx;
                if (eat) {
                    if (len >= 250) terminal = true;
                    else {
                        const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull +
                                                    (uint64_t)ctr * 0xD1B54A32D192ED03ull);
                        ctr += 1;
                        place_food(v, sub, gmask, r % (uint32_t)(256 - len));
                    }
                }
            }
            tick += 1;
            if (tick >= st.max_ticks) terminal = true;
        }
        *reinterpret_cast<uint4*>(out.obs + (int64_t)e * out.stride + sub * 16) = v;
        if (leader) {
            st.s0[e] = (uint32_t)head | ((uint32_t)dir << 8) | ((uint32_t)len << 16);
            st.s1[e] = (uint32_t)tick;
            st.ctr[e] = ctr;
            done[e] = terminal ? 1 : 0;
            out.rewards[e] = reward;
            out.terminals[e] = terminal ? 1 : 0;
            if (out.write_const) out.truncations[e] = 0;
            if (out.write_const) out.masks[e] = 1;
            if (out.dones_f32) out.dones_f32[e] = terminal ? 1.f : 0.f;
        }
    }
    episode_update(acc, e, leader, reset_row, (double)reward, terminal, (float)(len - 2));
}


// ---------------------------------------------------------------------------------------------------------------
// k_snake4: 4 lanes per env (8 envs per warp) instead of 16.  Lane `sub` of an env owns board rows sub, 4+sub, 8+sub,
// 12+sub as four uint4, so load / store instruction j of the warp moves rows 4j .. 4j+3 of every env: 64 contiguous
// bytes per env, full sectors.  The per-env control work (state unpack, direction logic, RNG, flag / reward stores,
// EpisodeStats) is now shared by 8 envs per warp instead of 2 -- the 16-lane kernel spent ~370 warp instructions per
// 1056 bytes and was issue-bound at ~0.35 of the HBM roofline; this one moves 4224 bytes per warp pass.
// Same arithmetic as k_snake (oracle/SPEC.md §Snake), bit-exact.
__device__ __forceinline__ uint32_t row_zero_count(const uint4& v) {
    return (uint32_t)(__popc(zero_bytes(v.x)) + __popc(zero_bytes(v.y)) + __popc(zero_bytes(v.z)) + __popc(zero_bytes(v.w)));
}

// food (255) on the k-th empty cell in index order c = y*16 + x; the 4 lanes of the env cooperate
__device__ __forceinline__ void place_food4(uint4 (&v)[4], int sub, unsigned gmask, uint32_t k) {
    // per-row empty counts of my rows, one byte each: byte j = row 4j + sub
    const uint32_t mine = row_zero_count(v[0]) | (row_zero_count(v[1]) << 8) | (row_zero_count(v[2]) << 16) |
                          (row_zero_count(v[3]) << 24);
    uint32_t cnt[4];   // cnt[s]: the packed counts of lane s of this env
#pragma unroll
    for (int s = 0; s < 4; ++s) cnt[s] = __shfl_sync(gmask, mine, s, 4);
    // walk the 16 rows in index order r = 4j + s
    int excl = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int c = (int)((cnt[s] >> (8 * j)) & 0xffu);
            if (sub == s && (int)k >= excl && (int)k < excl + c) {
                int r = (int)k - excl;
#pragma unroll
                for (int x = 0; x < 16; ++x) {
                    const uint32_t b = (get_word(v[j], x >> 2) >> ((x & 3) * 8)) & 0xffu;
                    if (b == 0u) {
                        if (r == 0) { set_byte(v[j], x, 255u); r = -1; }
                        else if (r > 0) --r;
                    }
                }
            }
            excl += c;
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(128) k_snake4(SnakeState st, int n, const int64_t* __restrict__ actions,
                                               uint8_t* done, const uint8_t* __restrict__ prev, int64_t prev_stride,
                                               SnOut out, EpisodeAcc acc) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int e = tid >> 2, sub = tid & 3;
    const int lane = threadIdx.x & 31;
    const unsigned gmask = 0xfu << (lane & 28);      // the 4 lanes of this env
    const bool valid = e < n;
    const bool leader = valid && sub == 0;
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = make_uint4(0, 0, 0, 0);
    int head = 136, dir = 3, len = 2, tick = 0;
    uint32_t ctr = 0;
    float reward = 0.f;
    bool terminal = false, reset_row = true;
    if (valid) {
        const uint64_t seed_e = st.seed + (uint64_t)e;
        bool do_reset = true;
        uint32_t a0 = 0, a1 = 0;
        int a = 0;
        uint4 vp[4];
        if (MODE == 1) {
            const uint8_t* src = prev + (int64_t)e * prev_stride + sub * 16;
#pragma unroll
            for (int j = 0; j < 4; ++j) vp[j] = *reinterpret_cast<const uint4*>(src + j * 64);     // row 4j + sub
            ctr = st.ctr[e];
            a0 = st.s0[e]; a1 = st.s1[e];
            a = (int)actions[e];
            do_reset = done[e] != 0;
        }
        if (do_reset) {
            // row 8 = lane 0, slot 2: head 254 at x = 8, tail 1 at x = 7
            if (sub == 0) { set_byte(v[2], 8, 254u); set_byte(v[2], 7, 1u); }
            const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull + (uint64_t)ctr * 0xD1B54A32D192ED03ull);
            ctr += 1;
            place_food4(v, sub, gmask, r % 254u);
        } else {
            reset_row = false;
            head = a0 & 0xff; dir = (a0 >> 8) & 3; len = (a0 >> 16) & 0xff; tick = a1 & 0xffff;
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = vp[j];
            a = a < 0 ? 0 : (a > 3 ? 3 : a);
            if (a != (dir ^ 1)) dir = a;
            const int x = head & 15, y = head >> 4;
            const int nx = x + (dir == 3) - (dir == 2), ny = y + (dir == 1) - (dir == 0);
            bool dead = nx < 0 || nx > 15 || ny < 0 || ny > 15;
            const int cx = dead ? 0 : nx, cy = dead ? 0 : ny;
            // target cell: row cy lives in lane cy & 3, slot cy >> 2
            const int cj = cy >> 2;
            const uint4 vr = cj == 0 ? v[0] : (cj == 1 ? v[1] : (cj == 2 ? v[2] : v[3]));
            const uint32_t mine = (get_word(vr, cx >> 2) >> ((cx & 3) * 8)) & 0xffu;
            const uint32_t q = __shfl_sync(gmask, mine, cy & 3, 4);
            if (!dead && q >= 2u && q <= 250u) dead = true;
            if (dead) {
                reward = -1.f;
                terminal = true;
            } else {
                const bool eat = q == 255u;
                if (eat) {
                    len += 1;
                    reward = 1.f;
                } else {  // every body value in [1,250] decays by one (byte SIMD)
#define SNAKE_DECAY(w) { const uint32_t m = __vcmpgeu4(w, 0x01010101u) & __vcmpleu4(w, 0xFAFAFAFAu); \
                         w = __vsub4(w, m & 0x01010101u); }
#pragma unroll
                    for (int j = 0; j < 4; ++j) { SNAKE_DECAY(v[j].x) SNAKE_DECAY(v[j].y) SNAKE_DECAY(v[j].z) SNAKE_DECAY(v[j].w) }
#undef SNAKE_DECAY
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (sub == (y & 3) && j == (y >> 2)) set_byte(v[j], x, (uint32_t)(len - 1));
                    if (sub == (ny & 3) && j == (ny >> 2)) set_byte(v[j], nx, 254u);
                }
                head = ny * 16 + nx;
                if (eat) {
                    if (len >= 250) terminal = true;
                    else {
                        const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull +
                                                    (uint64_t)ctr * 0xD1B54A32D192ED03ull);
                        ctr += 1;
                        place_food4(v, sub, gmask, r % (uint32_t)(256 - len));
                    }
                }
            }
            tick += 1;
            if (tick >= st.max_ticks) terminal = true;
        }
        uint8_t* dst = out.obs + (int64_t)e * out.stride + sub * 16;
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<uint4*>(dst + j * 64) = v[j];
        if (leader) {
            st.s0[e] = (uint32_t)head | ((uint32_t)dir << 8) | ((uint32_t)len << 16);
            st.s1[e] = (uint32_t)tick;
            st.ctr[e] = ctr;
            done[e] = terminal ? 1 : 0;
            out.rewards[e] = reward;
            out.terminals[e] = terminal ? 1 : 0;
            if (out.write_const) out.truncations[e] = 0;
            if (out.write_const) out.masks[e] = 1;
            if (out.dones_f32) out.dones_f32[e] = terminal ? 1.f : 0.f;
        }
    }
    episode_update(acc, e, leader, reset_row, (double)reward, terminal, (float)(len - 2));
}

int g_snake_variant = 4;   // lanes per env: 4 (default) or 16 (round 1), for A/B measurements

int snake_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    SnakeState* st = (SnakeState*)env->kind;
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 16 == 0 && ((uintptr_t)out->obs & 15) == 0, PB_ERR_INVALID,
               "snake: obs pointer/stride must be 16-byte aligned");
    SnOut o{(uint8_t*)out->obs, out->obs_stride, out->rewards, out->terminals, out->truncations, out->masks,
            out->dones_f32,
            env->write_const};
    if (g_snake_variant == 4) {
        const int blocks = (int)pb_ceil_div((int64_t)n * 4, 128);
        if (mode == 0)
            k_snake4<0><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, nullptr, 0, o, pb_episode_acc(env));
        else
            k_snake4<1><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, (const uint8_t*)env->cur_obs,
                                               env->cur_obs_stride, o, pb_episode_acc(env));
    } else {
        const int blocks = (int)pb_ceil_div((int64_t)n * 16, 128);
        if (mode == 0)
            k_snake<0><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, nullptr, 0, o, pb_episode_acc(env));
        else
            k_snake<1><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, (const uint8_t*)env->cur_obs,
                                              env->cur_obs_stride, o, pb_episode_acc(env));
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int snake_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    SnakeState* st = (SnakeState*)env->kind;
    st->seed = seed + (uint64_t)env->cfg.env_index_offset;
    return snake_launch(env, 0, nullptr, out, s);
}

int snake_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return snake_launch(env, 1, actions, out, s);
}

void snake_destroy(pb_env* env) {
    SnakeState* st = (SnakeState*)env->kind;
    if (!st) return;
    cudaFree(st->s0); cudaFree(st->s1); cudaFree(st->ctr);
    delete st;
    env->kind = nullptr;
}

const pb_env_vtable SNAKE_VT = {snake_reset, snake_step, snake_destroy};

}  // namespace

int pb_snake_create(pb_env* env) {
    SnakeState* st = new SnakeState();
    env->kind = st;
    env->vt = &SNAKE_VT;
    st->max_ticks = env->cfg.iparam[0] > 0 ? env->cfg.iparam[0] : 1024;
    PB_REQUIRE(st->max_ticks <= 65535, PB_ERR_INVALID, "snake: max_ticks must be <= 65535");
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&st->s0, n * 4));
    PB_CUDA(cudaMalloc(&st->s1, n * 4));
    PB_CUDA(cudaMalloc(&st->ctr, n * 4));
    PB_CUDA(cudaMemset(st->s0, 0, n * 4));
    PB_CUDA(cudaMemset(st->s1, 0, n * 4));
    PB_CUDA(cudaMemset(st->ctr, 0, n * 4));
    env->info.obs_dtype = PB_DTYPE_U8;
    env->info.obs_ndim = 2;
    env->info.obs_shape[0] = 16;
    env->info.obs_shape[1] = 16;
    env->info.obs_bytes = 256;
    env->info.num_actions = 4;
    env->info.obs_low = 0.f;
    env->info.obs_high = 255.f;
    return PB_OK;
}

// lanes per env of the snake step kernel: 4 (default, 8 envs per warp) or 16 (the round-1 kernel), for A/B measurements
extern "C" int pb_snake_set_variant(int32_t lanes_per_env) {
    PB_REQUIRE(lanes_per_env == 4 || lanes_per_env == 16, PB_ERR_INVALID, "pb_snake_set_variant: 4 or 16");
    g_snake_variant = lanes_per_env;
    return PB_OK;
}
