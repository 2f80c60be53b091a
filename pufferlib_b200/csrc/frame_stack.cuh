// frame_stack.cuh -- the TMA ring that writes (4,84,84) uint8 frame-stack observation rows, shared by the pixel env
// kinds (pong: env_pong.cu, breakout_pixels: env_breakout_pixels.cu).  The game is a template parameter; the ring, its
// mbarrier phases, the store / refill order, the reward / flag rows and EpisodeStats are this one body.
//
// The 28,224-byte observation row is moved by the TMA engine, never by the LSU: per env one cp.async.bulk pulls the
// three surviving frames of row t-1 (21,168 B) into a shared-memory stage while the CTA renders the new 84x84 frame
// into the same stage, then ONE cp.async.bulk pushes the whole 28,224 B row to row t.  A reset row is one rendered
// frame stored to all 4 slots.  A ring of FS_STAGES stages per CTA keeps 4 envs in flight; 2 CTAs per SM.
//
// A game G provides
//   G::State                                           per-env SoA state in HBM (passed by value to the kernel)
//   G::Env                                             one env's unpacked state (every thread holds a copy)
//   G::reset(st, e, seed_e, keep_ctr, p)               reset state (keep_ctr: keep the draw counter, the send path)
//   G::step(st, e, action, seed_e, p, reward, terminal, score)   load state and run one step of the dynamics
//   G::render(p, frame, tid)                           all FS_THREADS threads draw the 84x84 frame into shared memory
//   G::store(st, e, p)                                 thread 0 writes the state back
// Every thread runs reset / step redundantly on the same inputs (broadcast loads), so no barrier is needed before render.
#pragma once
#include "env_common.cuh"
#include "tma.cuh"

constexpr int FS_STAGES = 4;
constexpr uint32_t FS_FRAME = 84 * 84;      // 7056 = 441 * 16
constexpr uint32_t FS_ROW = 4 * FS_FRAME;   // 28224
constexpr uint32_t FS_STAGE_BYTES = 28672;  // FS_ROW rounded up to 1 KiB
constexpr int FS_THREADS = 128;
constexpr size_t FS_SMEM = (size_t)FS_STAGES * FS_STAGE_BYTES;

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

#ifdef __CUDACC__
// MODE 0: async_reset;  MODE 1: vectoriser send.  The body of a __launch_bounds__(FS_THREADS) kernel with FS_SMEM bytes of
// dynamic shared memory.
template <int MODE, class G>
__device__ __forceinline__ void frame_stack_run(const typename G::State& st, int n, const int64_t* __restrict__ actions,
                                                uint8_t* done, const unsigned char* __restrict__ prev, int64_t prev_stride,
                                                const FsOut& out, const EpisodeAcc& acc) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bars[FS_STAGES];
    const int tid = threadIdx.x;
    const int64_t step = gridDim.x;
    uint32_t phase[FS_STAGES] = {0, 0, 0, 0};

    auto needs_load = [&](int64_t e) -> bool { return MODE == 1 && done[e] == 0; };
    auto issue_load = [&](int s, int64_t e) {  // thread 0 only
        if (needs_load(e)) {
            mbar_expect_tx(&bars[s], 3 * FS_FRAME);
            tma_load_1d(smem + (size_t)s * FS_STAGE_BYTES, prev + e * prev_stride + FS_FRAME, 3 * FS_FRAME, &bars[s]);
        }
    };

    if (tid == 0) {
        for (int s = 0; s < FS_STAGES; ++s) mbar_init(&bars[s], 1);
        mbar_fence_init();
        int64_t e = blockIdx.x;
        for (int s = 0; s < FS_STAGES && e < n; ++s, e += step) issue_load(s, e);
    }
    __syncthreads();

    int it = 0;
    for (int64_t e = blockIdx.x; e < n; e += step, ++it) {
        const int s = it % FS_STAGES;
        unsigned char* buf = smem + (size_t)s * FS_STAGE_BYTES;
        unsigned char* frame = buf + 3 * FS_FRAME;
        // refill the stage that was stored one iteration ago: by now its bulk store has long read shared memory, so
        // this wait does not stall, and the load gets FS_STAGES - 1 iterations of lead time
        if (tid == 0 && it > 0) {
            const int64_t e_next = e + step * (FS_STAGES - 1);
            if (e_next < n) {
                tma_wait_read<0>();
                issue_load((it - 1) % FS_STAGES, e_next);
            }
        }
        // ---- integer dynamics, computed redundantly by every thread (same inputs: broadcast loads)
        const uint64_t seed_e = st.seed + (uint64_t)e;
        typename G::Env p;
        float reward = 0.f, score = 0.f;
        bool terminal = false;
        const bool loaded = needs_load(e);     // false -> this row is a reset row
        if (!loaded) G::reset(st, e, seed_e, MODE == 1, p);
        else G::step(st, e, actions[e], seed_e, p, reward, terminal, score);
        // ---- render the new frame into the stage
        G::render(p, frame, tid);
        fence_proxy_async_smem();
        __syncthreads();
        // ---- thread 0: bookkeeping + the bulk stores
        if (tid == 0) {
            G::store(st, e, p);
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
                    acc.row_return[e] = ret; acc.row_length[e] = len; acc.row_score[e] = score;
                    double* slot = acc.stats + 4 * (blockIdx.x & (PB_STAT_SLOTS - 1));
                    atomicAdd(slot + 0, 1.0); atomicAdd(slot + 1, ret);
                    atomicAdd(slot + 2, (double)len); atomicAdd(slot + 3, (double)score);
                }
            }
            unsigned char* row = out.obs + e * out.stride;
            if (loaded) {
                mbar_wait(&bars[s], phase[s]);     // the three old frames have landed
                tma_store_1d(row, buf, FS_ROW);
            } else {
                for (int k = 0; k < 4; ++k) tma_store_1d(row + (size_t)k * FS_FRAME, frame, FS_FRAME);
            }
            tma_commit();
        }
        if (loaded) phase[s] ^= 1;
        // no trailing barrier: the next iteration uses another stage; this stage is refilled by thread 0 at the top of
        // the next iteration (after wait_read) and rendered into FS_STAGES iterations later, behind block barriers
    }
    if (tid == 0) tma_wait_all<0>();
}

// The obs pointer / stride check and the launch: 2 CTAs per SM, at most one per env.  `k0` / `k1` are the game's MODE 0 / 1
// kernels (__global__ wrappers of frame_stack_run).
template <class State, class K0, class K1>
int fs_launch(pb_env* env, int mode, const State& st, const int64_t* actions, const pb_env_out* out, cudaStream_t s,
              K0* k0, K1* k1, const char* who) {
    const int n = env->cfg.num_envs;
    PB_REQUIRE(out->obs_stride % 16 == 0 && ((uintptr_t)out->obs & 15) == 0, PB_ERR_INVALID,
               "%s: obs pointer/stride must be 16-byte aligned", who);
    const FsOut o = fs_out(env, out);
    int grid = PB_NUM_SMS * 2;
    if (grid > n) grid = n;
    if (mode == 0) {
        PB_CUDA(cudaFuncSetAttribute(k0, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FS_SMEM));
        k0<<<grid, FS_THREADS, FS_SMEM, s>>>(st, n, actions, env->d_done, nullptr, 0, o, pb_episode_acc(env));
    } else {
        PB_CUDA(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FS_SMEM));
        k1<<<grid, FS_THREADS, FS_SMEM, s>>>(st, n, actions, env->d_done, (const unsigned char*)env->cur_obs,
                                             env->cur_obs_stride, o, pb_episode_acc(env));
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}
#endif
