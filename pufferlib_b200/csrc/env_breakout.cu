// env_breakout.cu -- N Breakout instances (oracle/SPEC.md §Breakout) behind the reference vectoriser semantics.
//
// Dynamics are the builder's spec (the reference has no first-party breakout: SURVEY.md §0); conventions are the
// reference's: reset-on-next-send (vector.py:147-151), reset rows r=0/term=False/mask=True (emulation.py:187-192),
// EpisodeStats on the terminal row (postprocess.py:22-54).  Bit-exact against oracle/csrc/envs.c.
//
// Layout: per-env state is 28 B of SoA in HBM (two packed words, a uint4 brick bitmap, the draw counter),
// reloaded each step because the policy forward sits between steps.  One lane owns one env for the integer
// physics (EPW = 8 envs per warp, so N = 16384 still fills the chip with 2048 warps); the envs of a warp then emit
// their 512-byte observation rows cooperatively -- per row each lane builds one float4 (lane 0-1: the 8 header
// scalars, lanes 2-31: 4 bricks each from the shuffled bitmap) so every row is ONE fully coalesced 512 B warp store
// (4 x 128 B lines).  Reward / flag / done rows are [N]-contiguous.
#include <cuda.h>

#include "env_common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace {

struct BreakoutState {
    uint32_t* s0;   // px(8) | lives(3)<<8 | in_play<<11 | wait(5)<<12 | (vx+3)(3)<<17 | (vy+2)(3)<<20
    uint32_t* s1;   // bx(8) | by(8)<<8 | tick(16)<<16
    uint4* bricks;  // 120 alive bits, brick i = row*20+col -> word i>>5, bit i&31
    uint32_t* ctr;  // RNG draw counter
    uint64_t seed;  // base seed + env_index_offset (env e uses seed + e)
    int max_ticks;
};

struct BkOut {
    float* obs;
    int64_t stride_f;
    float* rewards;
    uint8_t* terminals;
    uint8_t* truncations;
    uint8_t* masks;
    float* dones_f32;
    bool write_const;
};

__device__ __forceinline__ uint32_t bk_draw(uint64_t seed_e, uint32_t& ctr) {
    const uint32_t r = pb_mix32(seed_e * 0x9E3779B97F4A7C15ull + (uint64_t)ctr * 0xD1B54A32D192ED03ull);
    ctr += 1;
    return r;
}

// One step of the dynamics (oracle/SPEC.md §Breakout) on unpacked state; shared by the per-step kernel and the persistent
// rollout kernel so both are the same arithmetic.
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

// MODE 0: async_reset rows for every env;  MODE 1: vectoriser send (reset-or-step)
constexpr int EPW = 8;   // envs per warp: lanes 0..7 own one env each, all 32 lanes write the rows

template <int MODE>
__global__ void __launch_bounds__(128) k_breakout(BreakoutState st, int n, const int64_t* __restrict__ actions,
                                                 uint8_t* done, BkOut out, EpisodeAcc acc) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int e_base = warp * EPW;
    const int e = e_base + lane;
    const bool active = lane < EPW && e < n;
    int px = 68, lives = 5, in_play = 0, wait = 0, vx = 0, vy = 0, bx = 79, by = 188, tick = 0;
    uint4 bricks = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0x00ffffffu);
    uint32_t ctr = 0;
    int reward = 0;
    bool terminal = false, reset_row = true;
    float score = 0.f;
    if (active) {
        const uint64_t seed_e = st.seed + (uint64_t)e;
        bool do_reset = true;
        uint32_t a0 = 0, a1 = 0;
        uint4 bricks_in = bricks;
        int a = 0;
        if (MODE == 1) {   // all state loads are issued together (independent of `done`): one latency, not two
            ctr = st.ctr[e];
            a0 = st.s0[e]; a1 = st.s1[e];
            bricks_in = st.bricks[e];
            a = (int)actions[e];
            do_reset = done[e] != 0;
        }
        if (!do_reset) {
            reset_row = false;
            px = a0 & 0xff; lives = (a0 >> 8) & 7; in_play = (a0 >> 11) & 1; wait = (a0 >> 12) & 31;
            vx = (int)((a0 >> 17) & 7) - 3; vy = (int)((a0 >> 20) & 7) - 2;
            bx = a1 & 0xff; by = (a1 >> 8) & 0xff; tick = a1 >> 16;
            bricks = bricks_in;
            bk_physics(px, lives, in_play, wait, vx, vy, bx, by, tick, bricks, ctr, a, seed_e, st.max_ticks, reward, terminal,
                       score);
        }
        st.s0[e] = (uint32_t)px | ((uint32_t)lives << 8) | ((uint32_t)in_play << 11) | ((uint32_t)wait << 12) |
                   ((uint32_t)(vx + 3) << 17) | ((uint32_t)(vy + 2) << 20);
        st.s1[e] = (uint32_t)bx | ((uint32_t)by << 8) | ((uint32_t)tick << 16);
        st.bricks[e] = bricks;
        st.ctr[e] = ctr;
        done[e] = terminal ? 1 : 0;
        out.rewards[e] = (float)reward;
        out.terminals[e] = terminal ? 1 : 0;
        if (out.write_const) out.truncations[e] = 0;
        if (out.write_const) out.masks[e] = 1;
        if (out.dones_f32) out.dones_f32[e] = terminal ? 1.f : 0.f;
    }
    episode_update(acc, e, active, reset_row, (double)reward, terminal, score);

    // ---- observation rows: 32 envs per warp, one coalesced 512 B store per env
    const int left_mine = __popc(bricks.x) + __popc(bricks.y) + __popc(bricks.z) + __popc(bricks.w);
    const int word_sel = (lane >= 2) ? ((4 * lane - 8) >> 5) : 0;   // which bitmap word this lane decodes
    const int bit0 = (4 * lane - 8) & 31;
#pragma unroll
    for (int j = 0; j < EPW; ++j) {
        if (e_base + j >= n) break;
        const int jpx = __shfl_sync(0xffffffffu, px, j), jbx = __shfl_sync(0xffffffffu, bx, j);
        const int jby = __shfl_sync(0xffffffffu, by, j), jvx = __shfl_sync(0xffffffffu, vx, j);
        const int jvy = __shfl_sync(0xffffffffu, vy, j), jlives = __shfl_sync(0xffffffffu, lives, j);
        const int jplay = __shfl_sync(0xffffffffu, in_play, j), jleft = __shfl_sync(0xffffffffu, left_mine, j);
        const uint32_t w0 = __shfl_sync(0xffffffffu, bricks.x, j), w1 = __shfl_sync(0xffffffffu, bricks.y, j);
        const uint32_t w2 = __shfl_sync(0xffffffffu, bricks.z, j), w3 = __shfl_sync(0xffffffffu, bricks.w, j);
        float4 v;
        if (lane == 0) {
            v = make_float4((float)jpx * (1.f / 256.f), (float)jbx * (1.f / 256.f), (float)jby * (1.f / 256.f),
                            (float)jvx * 0.25f);
        } else if (lane == 1) {
            v = make_float4((float)jvy * 0.25f, (float)jlives * 0.125f, (float)jplay, (float)jleft * (1.f / 128.f));
        } else {
            const uint32_t w = word_sel == 0 ? w0 : (word_sel == 1 ? w1 : (word_sel == 2 ? w2 : w3));
            const uint32_t b = w >> bit0;
            v = make_float4((float)(b & 1u), (float)((b >> 1) & 1u), (float)((b >> 2) & 1u), (float)((b >> 3) & 1u));
        }
        float4* row = reinterpret_cast<float4*>(out.obs + (int64_t)(e_base + j) * out.stride_f);
        row[lane] = v;
    }
}


// =====================================================================================================================
// Persistent rollout: H vectorised env steps WITH the policy in the loop in ONE launch (config C2 / C5: breakout +
// models.Default 128 -> 128 -> {n_act, 1}).  Replaces the H x (k_breakout + k_policy_mlp_sample) launches of
// clean_pufferl.evaluate (recv -> policy -> store -> send): the policy weights are frozen during a rollout and the envs are
// independent, so a CTA owns 128 envs for all H steps --
//   * env state lives in REGISTERS across steps (thread = env); HBM sees it once at the start and once at the end;
//   * the observation row is built once, into a SWIZZLE_128B K-major tile in shared memory, from where (a) four TMA tensor
//     stores (issued by warp 4) write it to the rollout tensor (fully coalesced 64 KB per tile) and (b) the Hopper tensor
//     core consumes it: the four env warps are one warpgroup and compute hidden = obs . W_enc^T as two wgmma chains
//     (M = 64 envs, N = 128, K = 8 per instruction, accumulators in registers), W_enc resident in shared memory for the
//     whole rollout (one TMA load per CTA instead of one 64 KB re-stage per CTA per env step);
//   * bias + ReLU on the accumulator, staged K-major in the observation tile that is not in flight; the two heads on
//     mma.sync fragments; then thread = env samples the action by inverse CDF on the counter-based uniform of
//     pb_policy_mlp_sample (same key: seed, step counter, env row), stores value / logprob / action rows, and steps its
//     env with that action -- no global round trip between policy and env.
// Observation values are k/256, k/8, k/4 or 0/1: exact in TF32, so only W_enc is rounded (truncated) by the tensor core.
// Rows follow the bound-rollout convention of vector.B200: row 0 = the carry-over of the previous rollout (reward / done
// copied from the vecenv's own buffers), step t's outputs go to row t+1, the step that closes the rollout writes the
// vecenv's own buffers again.
// =====================================================================================================================
constexpr int RO_ENVS = 128;                 // envs per CTA = two wgmma M blocks of 64
constexpr int RO_THREADS = 160;              // warps 0..3: env / policy threads (one warpgroup), warp 4: TMA issue
constexpr int RO_KBLK_BYTES = RO_ENVS * 32 * 4;          // 16 KiB: [128 rows][32 floats]
constexpr int RO_TILE_BYTES = 4 * RO_KBLK_BYTES;         // 64 KiB
constexpr int RO_SMEM_W = 0, RO_SMEM_X = RO_TILE_BYTES, RO_SMEM_BAR = 3 * RO_TILE_BYTES;
constexpr int RO_SMEM_TOTAL = RO_SMEM_BAR + 128;
constexpr int RO_HEADS = 5;                  // live rows of the 8-row head matrix: breakout has 4 actions + the value

__constant__ float c_ro_wh[8 * 128];
__constant__ float c_ro_benc[128];
__constant__ float c_ro_bh[8];

struct RolloutParams {
    BreakoutState st;
    EpisodeAcc acc;
    uint8_t* done;              // env.done flags [N]
    int n, horizon, n_act;
    float* rewards;             // rollout rows [H*N]
    float* dones;
    float* values;
    float* logprobs;
    int64_t* actions;
    const float* carry_rewards; // the vecenv's own buffers [N]: read for row 0, written by the closing step
    const float* carry_dones;
    float* out_rewards;
    uint8_t* out_terminals;
    float* out_dones;
    uint64_t seed;              // sampler seed
    const uint64_t* counter;    // sampler step counter at the start of the rollout (advanced by H afterwards)
    float* dbg_hidden;          // validation only: relu(h) of step 0, [N][128]
    float* dbg_out;             // validation only: head outputs of step 0, [N][8]
};

__device__ __forceinline__ void ro_tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void ro_tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* src) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                     reinterpret_cast<uint64_t>(map)),
                 "r"(c0), "r"(c1), "r"(smem_u32(src))
                 : "memory");
}

// the observation row of one env (same values as k_breakout's cooperative row write) into row r of a SW128 K-major tile
__device__ __forceinline__ void ro_write_obs(uint8_t* tile, int r, int px, int bx, int by, int vx, int vy, int lives,
                                             int in_play, const uint4& bricks) {
    const int left = __popc(bricks.x) + __popc(bricks.y) + __popc(bricks.z) + __popc(bricks.w);
    const uint32_t w[4] = {bricks.x, bricks.y, bricks.z, bricks.w};
#pragma unroll
    for (int c = 0; c < 32; ++c) {        // 16-byte chunk c = floats 4c .. 4c+3 of the row; K-block c >> 3
        float4 v;
        if (c == 0) v = make_float4((float)px * (1.f / 256.f), (float)bx * (1.f / 256.f), (float)by * (1.f / 256.f), (float)vx * 0.25f);
        else if (c == 1) v = make_float4((float)vy * 0.25f, (float)lives * 0.125f, (float)in_play, (float)left * (1.f / 128.f));
        else {
            const uint32_t b = w[(4 * c - 8) >> 5] >> ((4 * c - 8) & 31);
            v = make_float4((float)(b & 1u), (float)((b >> 1) & 1u), (float)((b >> 2) & 1u), (float)((b >> 3) & 1u));
        }
        *reinterpret_cast<float4*>(tile + (c >> 3) * RO_KBLK_BYTES + r * 128 + ((((c & 7) ^ (r & 7))) << 4)) = v;
    }
}

// mma.sync m16n8k8 TF32 (fp32 accumulate): a0 (g, t)  a1 (g + 8, t)  a2 (g, t + 4)  a3 (g + 8, t + 4);  b0 (k = t, n = g)  b1 (k = t + 4, n = g);
// c0 c1 (g, 2t + {0,1})  c2 c3 (g + 8, 2t + {0,1})      [g = lane >> 2, t = lane & 3]
__device__ __forceinline__ void ro_mma_tf32(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t ro_to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

template <bool DBG>      // DBG: step-0 dumps for the validation hook (pb_rollout_debug_buffers); compiled out of the product path
__global__ void __launch_bounds__(RO_THREADS, 1)
k_breakout_rollout(const __grid_constant__ CUtensorMap map_obs, const __grid_constant__ CUtensorMap map_carry,
                   const __grid_constant__ CUtensorMap map_w, const RolloutParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + RO_SMEM_BAR);
    uint64_t* w_full = bars;          // W_enc landed
    uint64_t* tile_full = bars + 1;   // [2] observation tile written by the 128 env threads
    uint64_t* tile_free = bars + 3;   // the tensor store of the previous step has finished reading its tile
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int e0 = blockIdx.x * RO_ENVS;
    const int H = p.horizon;

    if (threadIdx.x == 0) {
        mbar_init(w_full, 1);
        mbar_init(&tile_full[0], RO_ENVS);
        mbar_init(&tile_full[1], RO_ENVS);
        mbar_init(tile_free, 1);
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 4) {
        // ================= TMA issue (one thread) =================
        if (lane == 0) {
            mbar_expect_tx(w_full, RO_TILE_BYTES);
            for (int kb = 0; kb < 4; ++kb) ro_tma_load_2d(smem + RO_SMEM_W + kb * RO_KBLK_BYTES, &map_w, kb * 32, 0, w_full);
            for (int t = 0; t <= H; ++t) {
                const int s = t & 1;
                uint8_t* tile = smem + RO_SMEM_X + s * RO_TILE_BYTES;
                mbar_wait(&tile_full[s], (uint32_t)((t >> 1) & 1));     // all 128 rows of obs(t) are in the tile
                // the tensor store of obs(t-1) has finished READING the other tile: the env threads may stage relu(h) of
                // step t there and then overwrite it with obs(t+1); it had a whole step: no stall in practice
                tma_wait_read<0>();
                asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(tile_free)) : "memory");
                // the same tile goes to HBM: rollout row t, or the vecenv's own observation buffer for the closing step
                const CUtensorMap* map = t < H ? &map_obs : &map_carry;
                const int row0 = t < H ? t * p.n + e0 : e0;
                for (int kb = 0; kb < 4; ++kb) ro_tma_store_2d(map, kb * 32, row0, tile + kb * RO_KBLK_BYTES);
                tma_commit();
            }
            tma_wait_all<0>();
        }
    } else {
        // ================= env threads: thread = env; warps 0..3 = the warpgroup of the policy products =================
        const int r = threadIdx.x;                    // 0..127
        const int e = e0 + r;                         // n is a multiple of 128 (checked by the launcher)
        const uint64_t seed_e = p.st.seed + (uint64_t)e;
        const uint64_t offset0 = *p.counter;
        // ---- state in registers for the whole rollout
        uint32_t ctr = p.st.ctr[e];
        const uint32_t a0 = p.st.s0[e], a1 = p.st.s1[e];
        uint4 bricks = p.st.bricks[e];
        bool done = p.done[e] != 0;
        int px = a0 & 0xff, lives = (a0 >> 8) & 7, in_play = (a0 >> 11) & 1, wait = (a0 >> 12) & 31;
        int vx = (int)((a0 >> 17) & 7) - 3, vy = (int)((a0 >> 20) & 7) - 2;
        int bx = a1 & 0xff, by = (a1 >> 8) & 0xff, tick = a1 >> 16;
        double ep_ret = p.acc.ep_return[e];
        int ep_len = p.acc.ep_length[e];
        // row 0 = the carry-over of the previous rollout (vector.B200.recv with _pending_own)
        p.rewards[e] = p.carry_rewards[e];
        p.dones[e] = p.carry_dones[e];
        ro_write_obs(smem + RO_SMEM_X, r, px, bx, by, vx, vy, lives, in_play, bricks);
        fence_proxy_async_smem();
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&tile_full[0])) : "memory");

        // head products on mma.sync fragments (like k_mlp_update and k_policy_mlp_sample): out[32 rows][8] = relu(h) . W_heads^T
        // with the warp's relu(h) staged K-major ([hidden unit][row], 16-byte pieces XORed with unit & 7) in the observation
        // tile that is NOT in flight, W_heads fragments resident in registers (k = t + 4j <-> hidden unit 8kb + 2t + j), and the
        // m index permuted (m = g + 8h of block mb <-> row 4g + 2mb + h) so that an A fragment is one LDS.128.
        const int g = lane >> 2, tq = lane & 3;
        uint32_t hb[16][2];
        float benc[16][2];                            // b_enc of the accumulator columns 8j + 2tq + {0, 1}
#pragma unroll
        for (int kb = 0; kb < 16; ++kb) {
            hb[kb][0] = ro_to_tf32(c_ro_wh[g * 128 + 8 * kb + 2 * tq]);
            hb[kb][1] = ro_to_tf32(c_ro_wh[g * 128 + 8 * kb + 2 * tq + 1]);
            benc[kb][0] = c_ro_benc[8 * kb + 2 * tq];
            benc[kb][1] = c_ro_benc[8 * kb + 2 * tq + 1];
        }
        const float bh_row[8] = {c_ro_bh[0], c_ro_bh[1], c_ro_bh[2], c_ro_bh[3], c_ro_bh[4], c_ro_bh[5], c_ro_bh[6], c_ro_bh[7]};
        const uint32_t w_addr = smem_u32(smem + RO_SMEM_W);
        mbar_wait(w_full, 0);

        for (int t = 0; t < H; ++t) {
            // ---- policy on obs(t): hidden = obs . W_enc^T on the tensor core -> bias + ReLU -> heads -> sample
            asm volatile("bar.sync 1, 128;" ::: "memory");      // every row of obs(t) is in the tile (each writer fenced)
            const uint32_t x_addr = smem_u32(smem + RO_SMEM_X + (t & 1) * RO_TILE_BYTES);
            uint8_t* other = smem + RO_SMEM_X + ((t + 1) & 1) * RO_TILE_BYTES;
            mbar_wait(tile_free, (uint32_t)(t & 1));           // the other tile is no longer read by a tensor store
#pragma unroll 1
            for (int half = 0; half < 2; ++half) {             // envs 64 half .. 64 half + 63 of the CTA
                float acc[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int kb = 0; kb < 4; ++kb)
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_m64n128k8_ss(acc, wgmma_desc_sw128(x_addr + kb * RO_KBLK_BYTES + half * 8192 + k * 32),
                                           wgmma_desc_sw128(w_addr + kb * RO_KBLK_BYTES + k * 32), (kb | k) ? 1 : 0);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc);
                // relu(h + b_enc) of rows 64 half + 16 warp + g (+8), hidden units 8j + 2tq (+1) -> block of the row's warp
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int row = 64 * half + 16 * warp + g + 8 * (q >> 1), k = 8 * j + 2 * tq + (q & 1);
                        const float rh = fmaxf(acc[4 * j + q] + benc[j][q & 1], 0.f);
                        if (DBG && p.dbg_hidden && t == 0) p.dbg_hidden[(int64_t)(e0 + row) * 128 + k] = rh;
                        *reinterpret_cast<float*>(other + (row >> 5) * RO_KBLK_BYTES + k * 128 +
                                                  ((((row & 31) >> 2) ^ (k & 7)) << 4) + (row & 3) * 4) = rh;
                    }
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");      // every relu(h) row is staged
            uint8_t* blk = other + warp * RO_KBLK_BYTES;        // [128 hidden units][32 rows]: rows 32 warp .. 32 warp + 31
            float out[8];
            {
                float hp[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
                const uint8_t* a_lo = blk + (2 * tq) * 128 + ((g ^ (2 * tq)) << 4);          // hidden unit 8kb + 2t, rows 4g..4g+3
                const uint8_t* a_hi = blk + (2 * tq + 1) * 128 + ((g ^ (2 * tq + 1)) << 4);  // hidden unit 8kb + 2t + 1
#pragma unroll
                for (int kb = 0; kb < 16; ++kb) {
                    const float4 lo = *reinterpret_cast<const float4*>(a_lo + kb * 1024);
                    const float4 hi = *reinterpret_cast<const float4*>(a_hi + kb * 1024);
                    ro_mma_tf32(hp[0], __float_as_uint(lo.x), __float_as_uint(lo.y), __float_as_uint(hi.x), __float_as_uint(hi.y), hb[kb][0], hb[kb][1]);
                    ro_mma_tf32(hp[1], __float_as_uint(lo.z), __float_as_uint(lo.w), __float_as_uint(hi.z), __float_as_uint(hi.w), hb[kb][0], hb[kb][1]);
                }
                __syncwarp();        // all fragment loads done: the head of the block becomes the [32 rows][10] redistribution scratch
                float* scr = reinterpret_cast<float*>(blk);
#pragma unroll
                for (int mb = 0; mb < 2; ++mb) {
                    *reinterpret_cast<float2*>(scr + (4 * g + 2 * mb) * 10 + 2 * tq) = make_float2(hp[mb][0], hp[mb][1]);
                    *reinterpret_cast<float2*>(scr + (4 * g + 2 * mb + 1) * 10 + 2 * tq) = make_float2(hp[mb][2], hp[mb][3]);
                }
                __syncwarp();
#pragma unroll
                for (int a2 = 0; a2 < 4; ++a2) {
                    const float2 o2 = *reinterpret_cast<const float2*>(scr + lane * 10 + 2 * a2);
                    out[2 * a2] = o2.x + bh_row[2 * a2];
                    out[2 * a2 + 1] = o2.y + bh_row[2 * a2 + 1];
                }
            }
            if (DBG && p.dbg_out && t == 0)
#pragma unroll
                for (int a = 0; a < 8; ++a) p.dbg_out[(int64_t)e * 8 + a] = out[a];
            // sample_logits (frameworks/cleanrl.py:25-47) by inverse CDF -- the arithmetic of k_policy_mlp_sample, with the
            // action count fixed at compile time (breakout: 4 logits, value in column 4)
            constexpr int NA = RO_HEADS - 1;
            float mx = out[0];
#pragma unroll
            for (int k = 1; k < NA; ++k) mx = fmaxf(mx, out[k]);
            float sum = 0.f;
#pragma unroll
            for (int k = 0; k < NA; ++k) sum += expf(out[k] - mx);
            const float lse = mx + logf(sum);
            const uint32_t rnd = pb_mix32(p.seed * 0x9E3779B97F4A7C15ull + (offset0 + (uint64_t)t) * 0xD1B54A32D192ED03ull +
                                          (uint64_t)e * 0x2545F4914F6CDD1Dull);
            const float u = (float)(rnd >> 8) * (1.0f / 16777216.0f);
            const float value = out[NA];
            float cdf = 0.f, lp = 0.f;
            int act = -1;
#pragma unroll
            for (int k = 0; k < NA; ++k) {
                const float nl = out[k] - lse, pk = expf(nl);
                cdf += pk;
                if (act < 0 && u < cdf) { act = k; lp = nl; }
            }
            if (act < 0) {   // rounding left cdf a hair below u: last action with non-negligible probability
#pragma unroll
                for (int k = NA - 1; k >= 0; --k)
                    if (act < 0 && out[k] - lse > -80.f) { act = k; lp = out[k] - lse; }
                if (act < 0) { act = NA - 1; lp = out[NA - 1] - lse; }
            }
            const int64_t row = (int64_t)t * p.n + e;
            p.values[row] = value;
            p.logprobs[row] = lp;
            p.actions[row] = act;

            // ---- vectoriser send: reset-or-step (vector.py:147-151), EpisodeStats (postprocess.py:22-54)
            int reward = 0;
            bool terminal = false;
            float score = 0.f;
            const bool reset_row = done;
            if (done) {
                px = 68; lives = 5; in_play = 0; wait = 0; vx = 0; vy = 0; bx = 79; by = 188; tick = 0;
                bricks = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0x00ffffffu);
            } else {
                bk_physics(px, lives, in_play, wait, vx, vy, bx, by, tick, bricks, ctr, act, seed_e, p.st.max_ticks, reward,
                           terminal, score);
            }
            done = terminal;
            if (reset_row) {
                ep_ret = 0.0; ep_len = 0;
            } else {
                ep_ret += (double)reward; ep_len += 1;
                if (terminal) {
                    p.acc.row_return[e] = ep_ret; p.acc.row_length[e] = ep_len; p.acc.row_score[e] = score;
                }
            }
            const bool fin = !reset_row && terminal;
            const unsigned fm = __ballot_sync(0xffffffffu, fin);
            if (fm) {      // warp-aggregated statistics, as episode_update()
                double sr = fin ? ep_ret : 0.0, sl = fin ? (double)ep_len : 0.0, ss = fin ? (double)score : 0.0;
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) {
                    sr += __shfl_xor_sync(0xffffffffu, sr, off);
                    sl += __shfl_xor_sync(0xffffffffu, sl, off);
                    ss += __shfl_xor_sync(0xffffffffu, ss, off);
                }
                if (lane == 0) {
                    const unsigned gw = (unsigned)(blockIdx.x * 4 + warp);
                    double* slot = p.acc.stats + 4 * ((gw * 2654435761u) >> 24);
                    atomicAdd(slot + 0, (double)__popc(fm));
                    atomicAdd(slot + 1, sr);
                    atomicAdd(slot + 2, sl);
                    atomicAdd(slot + 3, ss);
                }
            }
            // ---- outputs of this step: rollout row t+1, or the vecenv's own buffers for the step that closes the rollout
            if (t + 1 < H) {
                p.rewards[row + p.n] = (float)reward;
                p.dones[row + p.n] = terminal ? 1.f : 0.f;
            } else {
                p.out_rewards[e] = (float)reward;
                p.out_dones[e] = terminal ? 1.f : 0.f;
                p.out_terminals[e] = terminal ? 1 : 0;
            }
            const int s1 = (t + 1) & 1;
            asm volatile("bar.sync 1, 128;" ::: "memory");     // every env warp is done with its relu(h) block in that tile
            ro_write_obs(smem + RO_SMEM_X + s1 * RO_TILE_BYTES, r, px, bx, by, vx, vy, lives, in_play, bricks);
            fence_proxy_async_smem();
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&tile_full[s1])) : "memory");
        }
        // ---- state back to HBM
        p.st.s0[e] = (uint32_t)px | ((uint32_t)lives << 8) | ((uint32_t)in_play << 11) | ((uint32_t)wait << 12) |
                     ((uint32_t)(vx + 3) << 17) | ((uint32_t)(vy + 2) << 20);
        p.st.s1[e] = (uint32_t)bx | ((uint32_t)by << 8) | ((uint32_t)tick << 16);
        p.st.bricks[e] = bricks;
        p.st.ctr[e] = ctr;
        p.done[e] = done ? 1 : 0;
        p.acc.ep_return[e] = ep_ret;
        p.acc.ep_length[e] = ep_len;
    }
}

__global__ void k_counter_add(uint64_t* c, uint64_t v) { *c += v; }
float* g_ro_dbg_hidden = nullptr;
float* g_ro_dbg_out = nullptr;

typedef CUresult (*RoEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int ro_make_map(RoEncodeTiledFn fn, CUtensorMap* map, const float* base, int64_t rows, int64_t row_stride_floats) {
    const cuuint64_t dims[2] = {128, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)row_stride_floats * 4};
    const cuuint32_t box[2] = {32, (cuuint32_t)RO_ENVS};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PB_REQUIRE(r == CUDA_SUCCESS, PB_ERR_CUDA, "cuTensorMapEncodeTiled failed: %d", (int)r);
    return PB_OK;
}

int breakout_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    BreakoutState* st = (BreakoutState*)env->kind;
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 16 == 0 && ((uintptr_t)out->obs & 15) == 0, PB_ERR_INVALID,
               "breakout: obs pointer/stride must be 16-byte aligned");
    BkOut o{(float*)out->obs, out->obs_stride / 4, out->rewards, out->terminals, out->truncations, out->masks,
            out->dones_f32,
            env->write_const};
    const int blocks = (int)pb_ceil_div(n, (128 / 32) * EPW);
    if (mode == 0) k_breakout<0><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, o, pb_episode_acc(env));
    else k_breakout<1><<<blocks, 128, 0, s>>>(*st, n, actions, env->d_done, o, pb_episode_acc(env));
    PB_LAUNCH_CHECK();
    return PB_OK;
}

int breakout_reset(pb_env* env, uint64_t seed, const pb_env_out* out, cudaStream_t s) {
    BreakoutState* st = (BreakoutState*)env->kind;
    st->seed = seed + (uint64_t)env->cfg.env_index_offset;
    return breakout_launch(env, 0, nullptr, out, s);
}

int breakout_step(pb_env* env, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    return breakout_launch(env, 1, actions, out, s);
}

void breakout_destroy(pb_env* env) {
    BreakoutState* st = (BreakoutState*)env->kind;
    if (!st) return;
    cudaFree(st->s0); cudaFree(st->s1); cudaFree(st->bricks); cudaFree(st->ctr);
    delete st;
    env->kind = nullptr;
}

const pb_env_vtable BREAKOUT_VT = {breakout_reset, breakout_step, breakout_destroy};

}  // namespace

int pb_breakout_create(pb_env* env) {
    BreakoutState* st = new BreakoutState();
    env->kind = st;
    env->vt = &BREAKOUT_VT;
    st->max_ticks = env->cfg.iparam[0] > 0 ? env->cfg.iparam[0] : 4096;
    PB_REQUIRE(st->max_ticks <= 65535, PB_ERR_INVALID, "breakout: max_ticks must be <= 65535");
    const size_t n = (size_t)env->cfg.num_envs;
    PB_CUDA(cudaMalloc(&st->s0, n * 4));
    PB_CUDA(cudaMalloc(&st->s1, n * 4));
    PB_CUDA(cudaMalloc(&st->bricks, n * 16));
    PB_CUDA(cudaMalloc(&st->ctr, n * 4));
    PB_CUDA(cudaMemset(st->s0, 0, n * 4));
    PB_CUDA(cudaMemset(st->s1, 0, n * 4));
    PB_CUDA(cudaMemset(st->bricks, 0, n * 16));
    PB_CUDA(cudaMemset(st->ctr, 0, n * 4));
    env->info.obs_dtype = PB_DTYPE_F32;
    env->info.obs_ndim = 1;
    env->info.obs_shape[0] = 128;
    env->info.obs_bytes = 512;
    env->info.num_actions = 4;
    env->info.obs_low = -1.f;
    env->info.obs_high = 1.f;
    return PB_OK;
}

extern "C" int pb_rollout_breakout_mlp(pb_env* env, int32_t horizon, float* obs, float* rewards, float* dones, float* values,
                                       float* logprobs, int64_t* actions, const pb_env_out* carry, const float* w_enc,
                                       const float* b_enc, const float* w_heads, const float* b_heads, int32_t n_act,
                                       uint64_t seed, uint64_t* counter_dev, void* stream) {
    PB_REQUIRE(env && env->cfg.kind == PB_ENV_BREAKOUT, PB_ERR_INVALID, "pb_rollout_breakout_mlp: not a breakout handle");
    PB_REQUIRE(env->was_reset, PB_ERR_STATE, "pb_rollout_breakout_mlp: reset() first");
    const int n = env->cfg.num_envs;
    PB_REQUIRE(n % RO_ENVS == 0, PB_ERR_UNSUPPORTED, "pb_rollout_breakout_mlp: num_envs must be a multiple of %d", RO_ENVS);
    PB_REQUIRE(horizon >= 1 && (int64_t)horizon * n <= 0x7FFFFFFF, PB_ERR_INVALID, "pb_rollout_breakout_mlp: bad horizon");
    PB_REQUIRE(obs && rewards && dones && values && logprobs && actions && carry && carry->obs && carry->rewards &&
                   carry->terminals && carry->dones_f32 && w_enc && b_enc && w_heads && b_heads && counter_dev,
               PB_ERR_INVALID, "pb_rollout_breakout_mlp: null pointer (the carry buffers need dones_f32)");
    PB_REQUIRE(n_act == RO_HEADS - 1, PB_ERR_INVALID, "pb_rollout_breakout_mlp: breakout has %d actions", RO_HEADS - 1);
    PB_REQUIRE(carry->obs_stride == 512 && ((uintptr_t)obs & 15) == 0 && ((uintptr_t)carry->obs & 15) == 0 &&
                   ((uintptr_t)w_enc & 15) == 0,
               PB_ERR_INVALID, "pb_rollout_breakout_mlp: 16-byte aligned, densely packed observation rows required");
    PB_CUDA(cudaSetDevice(env->cfg.device));
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    PB_REQUIRE(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) == cudaSuccess && fn &&
                   qr == cudaDriverEntryPointSuccess,
               PB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    alignas(64) CUtensorMap map_obs, map_carry, map_w;
    int rc = ro_make_map((RoEncodeTiledFn)fn, &map_obs, obs, (int64_t)horizon * n, 128);
    if (rc == PB_OK) rc = ro_make_map((RoEncodeTiledFn)fn, &map_carry, (const float*)carry->obs, n, 128);
    if (rc == PB_OK) rc = ro_make_map((RoEncodeTiledFn)fn, &map_w, w_enc, 128, 128);
    if (rc != PB_OK) return rc;
    BreakoutState* st = (BreakoutState*)env->kind;
    cudaStream_t s = (cudaStream_t)stream;
    RolloutParams p;
    p.st = *st; p.acc = pb_episode_acc(env); p.done = env->d_done; p.n = n; p.horizon = horizon; p.n_act = n_act;
    p.rewards = rewards; p.dones = dones; p.values = values; p.logprobs = logprobs; p.actions = actions;
    p.carry_rewards = carry->rewards; p.carry_dones = carry->dones_f32;
    p.out_rewards = carry->rewards; p.out_terminals = carry->terminals; p.out_dones = carry->dones_f32;
    p.seed = seed; p.counter = counter_dev; p.dbg_hidden = g_ro_dbg_hidden; p.dbg_out = g_ro_dbg_out;
    PB_CUDA(cudaMemcpyToSymbolAsync(c_ro_wh, w_heads, sizeof(float) * 8 * 128, 0, cudaMemcpyDeviceToDevice, s));
    PB_CUDA(cudaMemcpyToSymbolAsync(c_ro_benc, b_enc, sizeof(float) * 128, 0, cudaMemcpyDeviceToDevice, s));
    PB_CUDA(cudaMemcpyToSymbolAsync(c_ro_bh, b_heads, sizeof(float) * 8, 0, cudaMemcpyDeviceToDevice, s));
    static bool attr_set = false;
    if (!attr_set) {
        PB_CUDA(cudaFuncSetAttribute(k_breakout_rollout<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RO_SMEM_TOTAL));
        PB_CUDA(cudaFuncSetAttribute(k_breakout_rollout<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RO_SMEM_TOTAL));
        attr_set = true;
    }
    if (p.dbg_hidden || p.dbg_out) k_breakout_rollout<true><<<n / RO_ENVS, RO_THREADS, RO_SMEM_TOTAL, s>>>(map_obs, map_carry, map_w, p);
    else k_breakout_rollout<false><<<n / RO_ENVS, RO_THREADS, RO_SMEM_TOTAL, s>>>(map_obs, map_carry, map_w, p);
    PB_LAUNCH_CHECK();
    k_counter_add<<<1, 1, 0, s>>>(counter_dev, (uint64_t)horizon);
    PB_LAUNCH_CHECK();
    env->write_const = false;
    env->cur_obs = carry->obs;
    env->cur_obs_stride = carry->obs_stride;
    return PB_OK;
}

// validation hook: device buffers ([N][128], [N][8]) that receive relu(h) and the head outputs of step 0 of the next rollouts
extern "C" int pb_rollout_debug_buffers(float* hidden, float* out) {
    g_ro_dbg_hidden = hidden;
    g_ro_dbg_out = out;
    return PB_OK;
}
