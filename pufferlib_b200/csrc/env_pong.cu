// env_pong.cu -- N Pong instances with (4,84,84) uint8 frame-stack observations (oracle/SPEC.md §Pong), sm_90a.
//
// Dynamics are the builder's spec (the reference's pong is ALE behind third-party wrappers: SURVEY.md §0); the
// observation layout (4,84,84) uint8 NCHW, oldest frame first, is the reference's (atari/environment.py:37-39,
// environments/test/mock_environments.py:211) and so are the vectoriser / EpisodeStats conventions
// (vector.py:147-151, emulation.py:187-192, postprocess.py:22-54).  Bit-exact against oracle/csrc/envs.c.
//
// The 28,224-byte observation row is moved by the TMA engine, never by the LSU: per env one cp.async.bulk pulls
// the three surviving frames of row t-1 (21,168 B) into a shared-memory stage while the CTA renders the new 84x84
// frame into the same stage (zero fill + 52 pixel stores), then ONE cp.async.bulk pushes the whole 28,224 B row to
// row t.  A ring of 4 stages per CTA keeps 4 envs in flight; 2 CTAs per SM.  Per-env state is 12 B of SoA.
#include "env_common.cuh"
#include "tma.cuh"

namespace {

constexpr int PG_STAGES = 4;
constexpr uint32_t FRAME = 84 * 84;        // 7056 = 441 * 16
constexpr uint32_t ROW = 4 * FRAME;        // 28224
constexpr uint32_t STAGE_BYTES = 28672;    // ROW rounded up to 1 KiB
constexpr int PG_THREADS = 128;

struct PongState {
    uint32_t* s0;   // ly(8) | ry(8)<<8 | (bx+2)(8)<<16 | (by)(8)<<24
    uint32_t* s1;   // (vx+2)(3) | (vy+2)(3)<<3 | score_l(4)<<6 | score_r(4)<<10 | tick(16)<<16
    uint32_t* ctr;
    uint64_t seed;
    int max_score, max_ticks;
};

struct PgOut {
    unsigned char* obs;
    int64_t stride;
    float* rewards;
    uint8_t* terminals;
    uint8_t* truncations;
    uint8_t* masks;
    float* dones_f32;
    bool write_const;
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

// MODE 0: async_reset;  MODE 1: vectoriser send
template <int MODE>
__global__ void __launch_bounds__(PG_THREADS) k_pong(PongState st, int n, const int64_t* __restrict__ actions,
                                                    uint8_t* done, const unsigned char* __restrict__ prev,
                                                    int64_t prev_stride, PgOut out, EpisodeAcc acc) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bars[PG_STAGES];
    const int tid = threadIdx.x;
    const int64_t step = gridDim.x;
    uint32_t phase[PG_STAGES] = {0, 0, 0, 0};

    auto needs_load = [&](int64_t e) -> bool { return MODE == 1 && done[e] == 0; };
    auto issue_load = [&](int s, int64_t e) {  // thread 0 only
        if (needs_load(e)) {
            mbar_expect_tx(&bars[s], 3 * FRAME);
            tma_load_1d(smem + (size_t)s * STAGE_BYTES, prev + e * prev_stride + FRAME, 3 * FRAME, &bars[s]);
        }
    };

    if (tid == 0) {
        for (int s = 0; s < PG_STAGES; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
        int64_t e = blockIdx.x;
        for (int s = 0; s < PG_STAGES && e < n; ++s, e += step) issue_load(s, e);
    }
    __syncthreads();

    int it = 0;
    for (int64_t e = blockIdx.x; e < n; e += step, ++it) {
        const int s = it % PG_STAGES;
        unsigned char* buf = smem + (size_t)s * STAGE_BYTES;
        unsigned char* frame = buf + 3 * FRAME;
        // refill the stage that was stored one iteration ago: by now its bulk store has long read shared memory, so
        // this wait does not stall, and the load gets PG_STAGES - 1 iterations of lead time
        if (tid == 0 && it > 0) {
            const int64_t e_next = e + step * (PG_STAGES - 1);
            if (e_next < n) {
                tma_wait_read<0>();
                issue_load((it - 1) % PG_STAGES, e_next);
            }
        }
        // ---- integer physics, computed redundantly by every thread (same inputs: broadcast loads)
        const uint64_t seed_e = st.seed + (uint64_t)e;
        PongEnv p;
        float reward = 0.f;
        bool terminal = false;
        const bool loaded = needs_load(e);     // false -> this row is a reset row
        if (!loaded) {
            p.ctr = (MODE == 1) ? st.ctr[e] : 0u;
            p.ly = 36; p.ry = 36; p.score_l = 0; p.score_r = 0; p.tick = 0;
            pong_serve(p, seed_e);
        } else {
            const uint32_t a0 = st.s0[e], a1 = st.s1[e];
            p.ly = a0 & 0xff; p.ry = (a0 >> 8) & 0xff; p.bx = (int)((a0 >> 16) & 0xff) - 2; p.by = (a0 >> 24) & 0xff;
            p.vx = (int)(a1 & 7) - 2; p.vy = (int)((a1 >> 3) & 7) - 2;
            p.score_l = (a1 >> 6) & 15; p.score_r = (a1 >> 10) & 15; p.tick = a1 >> 16;
            p.ctr = st.ctr[e];
            int a = (int)actions[e];
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
        }
        // ---- render the new frame into the stage: zero fill, then opponent paddle, agent paddle, ball
        for (int k = tid; k < (int)(FRAME / 16); k += PG_THREADS) reinterpret_cast<uint4*>(frame)[k] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        if (tid < 24) frame[(p.ly + (tid >> 1)) * 84 + 4 + (tid & 1)] = 128;
        else if (tid < 48) frame[(p.ry + ((tid - 24) >> 1)) * 84 + 78 + (tid & 1)] = 192;
        __syncthreads();   // ball is drawn last (it may overlap a paddle pixel)
        if (tid < 4) {
            const int x = p.bx + (tid & 1), y = p.by + (tid >> 1);
            if (x >= 0 && x < 84 && y >= 0 && y < 84) frame[y * 84 + x] = 255;
        }
        fence_proxy_async_smem();
        __syncthreads();
        // ---- thread 0: bookkeeping + the bulk stores
        if (tid == 0) {
            st.s0[e] = (uint32_t)p.ly | ((uint32_t)p.ry << 8) | ((uint32_t)(p.bx + 2) << 16) | ((uint32_t)p.by << 24);
            st.s1[e] = (uint32_t)(p.vx + 2) | ((uint32_t)(p.vy + 2) << 3) | ((uint32_t)p.score_l << 6) |
                       ((uint32_t)p.score_r << 10) | ((uint32_t)p.tick << 16);
            st.ctr[e] = p.ctr;
            done[e] = terminal ? 1 : 0;
            out.rewards[e] = reward;
            out.terminals[e] = terminal ? 1 : 0;
            if (out.write_const) out.truncations[e] = 0;
            if (out.write_const) out.masks[e] = 1;
            if (out.dones_f32) out.dones_f32[e] = terminal ? 1.f : 0.f;
            // EpisodeStats (postprocess.py:22-54), scalar form
            if (!loaded) { acc.ep_return[e] = 0.0; acc.ep_length[e] = 0; }
            else {
                const double ret = acc.ep_return[e] + (double)reward;
                const int len = acc.ep_length[e] + 1;
                acc.ep_return[e] = ret; acc.ep_length[e] = len;
                if (terminal) {
                    const float score = (float)(p.score_r - p.score_l);
                    acc.row_return[e] = ret; acc.row_length[e] = len; acc.row_score[e] = score;
                    double* slot = acc.stats + 4 * (blockIdx.x & (PB_STAT_SLOTS - 1));
                    atomicAdd(slot + 0, 1.0); atomicAdd(slot + 1, ret);
                    atomicAdd(slot + 2, (double)len); atomicAdd(slot + 3, (double)score);
                }
            }
            unsigned char* row = out.obs + e * out.stride;
            if (loaded) {
                mbar_wait(&bars[s], phase[s]);     // the three old frames have landed
                tma_store_1d(row, buf, ROW);
            } else {
                for (int k = 0; k < 4; ++k) tma_store_1d(row + (size_t)k * FRAME, frame, FRAME);
            }
            tma_commit();
        }
        if (loaded) phase[s] ^= 1;
        // no trailing barrier: the next iteration uses another stage; this stage is refilled by thread 0 at the top of
        // the next iteration (after wait_read) and rendered into PG_STAGES iterations later, behind block barriers
    }
    if (tid == 0) tma_wait_all<0>();
}

int pong_launch(pb_env* env, int mode, const int64_t* actions, const pb_env_out* out, cudaStream_t s) {
    PongState* st = (PongState*)env->kind;
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 16 == 0 && ((uintptr_t)out->obs & 15) == 0, PB_ERR_INVALID,
               "pong: obs pointer/stride must be 16-byte aligned");
    PgOut o{(unsigned char*)out->obs, out->obs_stride, out->rewards, out->terminals, out->truncations, out->masks,
            out->dones_f32,
            env->write_const};
    int grid = PB_NUM_SMS * 2;
    if (grid > n) grid = n;
    const size_t smem = (size_t)PG_STAGES * STAGE_BYTES;
    if (mode == 0) {
        PB_CUDA(cudaFuncSetAttribute(k_pong<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_pong<0><<<grid, PG_THREADS, smem, s>>>(*st, n, actions, env->d_done, nullptr, 0, o, pb_episode_acc(env));
    } else {
        PB_CUDA(cudaFuncSetAttribute(k_pong<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_pong<1><<<grid, PG_THREADS, smem, s>>>(*st, n, actions, env->d_done, (const unsigned char*)env->cur_obs,
                                                 env->cur_obs_stride, o, pb_episode_acc(env));
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
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
    env->info.obs_bytes = ROW;
    env->info.num_actions = 6;
    env->info.obs_low = 0.f;
    env->info.obs_high = 255.f;
    return PB_OK;
}
