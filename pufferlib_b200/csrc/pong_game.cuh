// pong_game.cuh -- pong's per-env state, its packing and its dynamics (oracle/SPEC.md §Pong), shared by the pong kind
// (env_pong.cu: the agent against the scripted tracker) and the pong_versus kind (env_pong_versus.cu: two agents).
// Per-env state is 12 B of SoA.
#pragma once
#include "env_common.cuh"

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

__device__ __forceinline__ void pong_reset(const uint32_t* ctr, int64_t e, uint64_t seed_e, bool keep_ctr, PongEnv& p) {
    p.ctr = keep_ctr ? ctr[e] : 0u;
    p.ly = 36; p.ry = 36; p.score_l = 0; p.score_r = 0; p.tick = 0;
    pong_serve(p, seed_e);
}

__device__ __forceinline__ void pong_load(const PongState& st, int64_t e, PongEnv& p) {
    const uint32_t a0 = st.s0[e], a1 = st.s1[e];
    p.ly = a0 & 0xff; p.ry = (a0 >> 8) & 0xff; p.bx = (int)((a0 >> 16) & 0xff) - 2; p.by = (a0 >> 24) & 0xff;
    p.vx = (int)(a1 & 7) - 2; p.vy = (int)((a1 >> 3) & 7) - 2;
    p.score_l = (a1 >> 6) & 15; p.score_r = (a1 >> 10) & 15; p.tick = a1 >> 16;
    p.ctr = st.ctr[e];
}

__device__ __forceinline__ void pong_store(const PongState& st, int64_t e, const PongEnv& p) {
    st.s0[e] = (uint32_t)p.ly | ((uint32_t)p.ry << 8) | ((uint32_t)(p.bx + 2) << 16) | ((uint32_t)p.by << 24);
    st.s1[e] = (uint32_t)(p.vx + 2) | ((uint32_t)(p.vy + 2) << 3) | ((uint32_t)p.score_l << 6) |
               ((uint32_t)p.score_r << 10) | ((uint32_t)p.tick << 16);
    st.ctr[e] = p.ctr;
}

// a paddle's top edge after action a: dy+3 per action, 3 bits each: NOOP, FIRE -> 0; UP(2,4) -> -3; DOWN(3,5) -> +3
// (oracle/SPEC.md §Pong), clamped to [0, 72].  env_pong.cu spells the same map out inline: as a call, its MODE 0
// preprocessing instances compile to a different (equivalent) schedule.
__device__ __forceinline__ int pong_paddle(int y, int64_t action) {
    int a = (int)action;
    a = a < 0 ? 0 : (a > 5 ? 5 : a);
    return min(max(y + (int)((0x30C1Bu >> (3 * a)) & 7u) - 3, 0), 72);
}

// everything after the paddles moved: the ball, its bounces and paddle hits, a point and its serve, the tick, the
// terminal and the score of the right paddle (reward: +1 / -1 for a point of the right / left paddle, else unchanged)
__device__ __forceinline__ void pong_ball(const PongState& st, PongEnv& p, uint64_t seed_e, float& reward,
                                          bool& terminal, float& score) {
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

}  // namespace
