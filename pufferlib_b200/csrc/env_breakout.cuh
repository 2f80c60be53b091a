// env_breakout.cuh -- the breakout game (oracle/SPEC.md §Breakout) shared by every kernel that steps it: the per-step
// kernel and the persistent rollout kernel of env_breakout.cu (128-float state rows) and the frame-stack kernel of
// env_breakout_pixels.cu ((4,84,84) uint8 frames).  One copy of the arithmetic, so the kinds play the same game.
//
// Per-env state is 28 B of SoA in HBM: two packed words, a uint4 brick bitmap and the RNG draw counter.
#pragma once
#include "env_common.cuh"

struct BreakoutState {
    uint32_t* s0;   // px(8) | lives(3)<<8 | in_play<<11 | wait(5)<<12 | (vx+3)(3)<<17 | (vy+2)(3)<<20
    uint32_t* s1;   // bx(8) | by(8)<<8 | tick(16)<<16
    uint4* bricks;  // 120 alive bits, brick i = row*20+col -> word i>>5, bit i&31
    uint32_t* ctr;  // RNG draw counter
    uint64_t seed;  // base seed + env_index_offset (env e uses seed + e)
    int max_ticks;
};

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t bk_draw(uint64_t seed_e, uint32_t& ctr) {
    const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull + (uint64_t)ctr * 0xD1B54A32D192ED03ull);
    ctr += 1;
    return r;
}

__device__ __forceinline__ void bk_unpack(uint32_t a0, uint32_t a1, int& px, int& lives, int& in_play, int& wait, int& vx,
                                          int& vy, int& bx, int& by, int& tick) {
    px = a0 & 0xff; lives = (a0 >> 8) & 7; in_play = (a0 >> 11) & 1; wait = (a0 >> 12) & 31;
    vx = (int)((a0 >> 17) & 7) - 3; vy = (int)((a0 >> 20) & 7) - 2;
    bx = a1 & 0xff; by = (a1 >> 8) & 0xff; tick = a1 >> 16;
}

__device__ __forceinline__ uint32_t bk_pack_s0(int px, int lives, int in_play, int wait, int vx, int vy) {
    return (uint32_t)px | ((uint32_t)lives << 8) | ((uint32_t)in_play << 11) | ((uint32_t)wait << 12) |
           ((uint32_t)(vx + 3) << 17) | ((uint32_t)(vy + 2) << 20);
}

__device__ __forceinline__ uint32_t bk_pack_s1(int bx, int by, int tick) {
    return (uint32_t)bx | ((uint32_t)by << 8) | ((uint32_t)tick << 16);
}

// One step of the dynamics (oracle/SPEC.md §Breakout) on unpacked state; shared by every breakout kernel so all of them
// are the same arithmetic.
__device__ __forceinline__ void bk_physics(int& px, int& lives, int& in_play, int& wait, int& vx, int& vy, int& bx, int& by,
                                           int& tick, uint4& bricks, uint32_t& ctr, int a, uint64_t seed_e, int max_ticks,
                                           int& reward, bool& terminal, float& score) {
    // actions are clamped to [0, 3] by the spec (a < 0 -> NOOP, a > 3 -> LEFT).  Written as three comparisons on the raw
    // value: ptxas 12.9 turned `a = clamp(a, 0, 3); if (a == 3) ..` into a VIMNMX.RELU with predicate outputs whose
    // predicate came out true for a == 2 when targeting sm_100a (the paddle moved left instead of right; caught by the oracle tests)
    const bool fire = a == 1, go_right = a == 2, go_left = a >= 3;
    if (go_right) px = min(px + 4, 136);
    if (go_left) px = max(px - 4, 0);
    if (!in_play) {
        wait += 1;
        bx = px + 11; by = 188;
        if (fire || wait >= 16) {
            in_play = 1; vy = -2;
            const int k = (int)(bk_draw(seed_e, ctr) & 3u);
            vx = k < 2 ? k - 2 : k - 1;   // {-2,-1,1,2}
        }
    } else {
        bx += vx; by += vy;
        if (bx < 0) { bx = -bx; vx = -vx; }
        if (bx > 158) { bx = 316 - bx; vx = -vx; }
        if (by < 0) { by = -by; vy = -vy; }
        const int cx = bx + 1, cy = by + 1;
        if (cy >= 30 && cy < 66) {
            const int row = (cy - 30) / 6, col = cx >> 3;
            const int i = row * 20 + col;
            uint32_t* w = (i < 32) ? &bricks.x : (i < 64) ? &bricks.y : (i < 96) ? &bricks.z : &bricks.w;
            const uint32_t bit = 1u << (i & 31);
            if (*w & bit) {
                *w &= ~bit;
                reward += row < 2 ? 7 : (row < 4 ? 4 : 1);
                vy = -vy;
            }
        }
        if (vy > 0 && by >= 188 && by <= 192 && bx + 2 > px && bx < px + 24) {
            int off = bx + 1 - px;
            off = off < 0 ? 0 : (off > 23 ? 23 : off);
            const int seg = off >> 2;
            vy = -2; by = 188;
            vx = seg < 3 ? seg - 3 : seg - 2;   // {-3,-2,-1,1,2,3}
        } else if (by >= 198) {
            lives -= 1; in_play = 0; wait = 0;
            bx = px + 11; by = 188; vx = 0; vy = 0;
        }
    }
    tick += 1;
    const int left = __popc(bricks.x) + __popc(bricks.y) + __popc(bricks.z) + __popc(bricks.w);
    terminal = lives == 0 || left == 0 || tick >= max_ticks;
    score = (float)(120 - left) / 120.0f;
}
#endif
