// image.cu -- image-observation row movers staged through shared memory by the TMA engine (sm_90a).
//
//   pb_image_pack            frame-stack pack: obs_out[e] = [prev_obs[e][1..S-1], new_frame[e]]  (or S copies of the
//                            new frame where reset_mask[e]).  Replaces the LazyFrames -> ndarray materialisation
//                            inside `self.obs[:] = ob` (reference pufferlib/emulation.py:161-162) for the
//                            (4,84,84) uint8 stack built by atari/environment.py:37-39.
//   pb_minibatch_gather_tma  `b_obs = obs[b_idxs_obs]` (reference clean_pufferl.py:477) for rows >= 4 KiB.
//
// One warp per CTA; ONE elected thread drives a ring of STAGES shared-memory buffers: cp.async.bulk global->shared
// (mbarrier complete_tx) then cp.async.bulk shared->global (bulk_group); no register staging, no LSU traffic.
// 132 SMs x 2 resident CTAs x STAGES x <=28 KiB in flight covers the HBM latency-bandwidth product many times over.
#include "pb_common.cuh"
#include "tma.cuh"

namespace {

constexpr int STAGES = 4;
constexpr uint32_t MAX_CHUNK = 28672;  // bytes per stage buffer (>= one 84x84x4 row = 28224); 4 x 28 KiB = 112 KiB

struct RowMap {        // output row o -> source row, for the minibatch gather
    int64_t N, H, n_mb, rows, bptt, mb_begin;
};

// Generic pipelined mover: for item i in [first, total) step gridDim: load `chunk_bytes` from src(i), store to dst(i).
template <typename SrcFn, typename DstFn>
__device__ __forceinline__ void move_items(int64_t total, uint32_t chunk_bytes, SrcFn src, DstFn dst,
                                           unsigned char* smem, uint64_t* bars) {
    if (threadIdx.x != 0) return;
    for (int s = 0; s < STAGES; ++s) mbar_init(&bars[s], 1);
    mbar_fence_init();
    int64_t issue = blockIdx.x, drain = blockIdx.x;
    const int64_t step = gridDim.x;
    uint32_t phase[STAGES] = {0, 0, 0, 0};
    int si = 0, sd = 0, inflight = 0;
    // prologue: fill the ring
    while (issue < total && inflight < STAGES) {
        mbar_expect_tx(&bars[si], chunk_bytes);
        tma_load_1d(smem + (size_t)si * MAX_CHUNK, src(issue), chunk_bytes, &bars[si]);
        si = (si + 1) % STAGES; ++inflight; issue += step;
    }
    while (drain < total) {
        mbar_wait(&bars[sd], phase[sd]);
        phase[sd] ^= 1;
        tma_store_1d(dst(drain), smem + (size_t)sd * MAX_CHUNK, chunk_bytes);
        tma_commit();
        drain += step; --inflight;
        if (issue < total) {
            // the buffer about to be refilled is `sd`: its store (the newest group) must have read shared memory
            tma_wait_read<0>();
            mbar_expect_tx(&bars[sd], chunk_bytes);
            tma_load_1d(smem + (size_t)sd * MAX_CHUNK, src(issue), chunk_bytes, &bars[sd]);
            ++inflight; issue += step;
        }
        sd = (sd + 1) % STAGES;
    }
    tma_wait_all<0>();
}

__global__ void __launch_bounds__(32) k_gather_tma(const unsigned char* __restrict__ obs, unsigned char* __restrict__ dst,
                                                  int64_t row_bytes, uint32_t chunk_bytes, int chunks_per_row,
                                                  int64_t n_out_rows, RowMap g) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bars[STAGES];
    const int64_t mb_size = g.rows * g.bptt;
    auto src = [&](int64_t i) -> const void* {
        const int64_t o = i / chunks_per_row, c = i - o * chunks_per_row;
        const int64_t mb = g.mb_begin + o / mb_size, rem = o % mb_size;
        const int64_t r = rem / g.bptt, j = rem - r * g.bptt;
        const int64_t f = (r * g.n_mb + mb) * g.bptt + j;
        const int64_t e = f / g.H, t = f - e * g.H;
        return obs + (t * g.N + e) * row_bytes + c * (int64_t)chunk_bytes;
    };
    auto dstf = [&](int64_t i) -> void* {
        const int64_t o = i / chunks_per_row, c = i - o * chunks_per_row;
        return dst + o * row_bytes + c * (int64_t)chunk_bytes;
    };
    move_items(n_out_rows * chunks_per_row, chunk_bytes, src, dstf, smem, bars);
}

// Frame-stack pack.  Each item is one env: S-1 old frames come from prev_obs slots 1..S-1, the newest from
// new_frames; a reset env gets S copies of the new frame.  Two loads per env land on one mbarrier.
__global__ void __launch_bounds__(32) k_image_pack(const unsigned char* __restrict__ new_frames, int64_t frame_stride,
                                                  const unsigned char* __restrict__ prev, int64_t prev_stride,
                                                  unsigned char* __restrict__ out, int64_t out_stride,
                                                  const uint8_t* __restrict__ reset_mask, int64_t n,
                                                  uint32_t frame_bytes, int stack) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bars[STAGES];
    if (threadIdx.x != 0) return;
    for (int s = 0; s < STAGES; ++s) mbar_init(&bars[s], 1);
    mbar_fence_init();
    const uint32_t old_bytes = frame_bytes * (uint32_t)(stack - 1);
    const uint32_t row_bytes = frame_bytes * (uint32_t)stack;
    uint32_t phase[STAGES] = {0, 0, 0, 0};
    uint8_t was_reset[STAGES];
    int64_t issue = blockIdx.x, drain = blockIdx.x;
    const int64_t step = gridDim.x;
    int si = 0, sd = 0, inflight = 0;
    auto issue_loads = [&](int s, int64_t e) {
        unsigned char* buf = smem + (size_t)s * MAX_CHUNK;
        const bool rs = reset_mask && reset_mask[e];
        was_reset[s] = rs;
        if (rs || stack == 1) {
            mbar_expect_tx(&bars[s], frame_bytes);
            tma_load_1d(buf + old_bytes, new_frames + e * frame_stride, frame_bytes, &bars[s]);
        } else {
            mbar_expect_tx(&bars[s], row_bytes);
            tma_load_1d(buf, prev + e * prev_stride + frame_bytes, old_bytes, &bars[s]);
            tma_load_1d(buf + old_bytes, new_frames + e * frame_stride, frame_bytes, &bars[s]);
        }
    };
    while (issue < n && inflight < STAGES) {
        issue_loads(si, issue);
        si = (si + 1) % STAGES; ++inflight; issue += step;
    }
    while (drain < n) {
        mbar_wait(&bars[sd], phase[sd]);
        phase[sd] ^= 1;
        unsigned char* buf = smem + (size_t)sd * MAX_CHUNK;
        unsigned char* row = out + drain * out_stride;
        if (was_reset[sd] && stack > 1) {
            for (int k = 0; k < stack; ++k) tma_store_1d(row + (size_t)k * frame_bytes, buf + old_bytes, frame_bytes);
        } else {
            tma_store_1d(row, buf, row_bytes);
        }
        tma_commit();
        drain += step; --inflight;
        if (issue < n) {
            tma_wait_read<0>();
            issue_loads(sd, issue);
            ++inflight; issue += step;
        }
        sd = (sd + 1) % STAGES;
    }
    tma_wait_all<0>();
}

int grid_for(int64_t items) {
    int64_t g = (int64_t)PB_NUM_SMS * 2;  // 2 resident CTAs per SM at 112 KiB of shared memory each
    if (g > items) g = items;
    return (int)(g < 1 ? 1 : g);
}

}  // namespace

int pb_minibatch_gather_tma(const void* obs, void* dst, int64_t row_bytes, int64_t N, int64_t H, int64_t n_mb,
                            int64_t rows, int64_t bptt, int64_t mb_begin, int64_t mb_count, cudaStream_t s) {
    // split rows into equal 16-byte-multiple chunks that fit a stage buffer
    int chunks = (int)pb_ceil_div(row_bytes, MAX_CHUNK);
    while (row_bytes % chunks != 0 || (row_bytes / chunks) % 16 != 0) {
        ++chunks;
        PB_REQUIRE(chunks <= row_bytes / 16, PB_ERR_INVALID, "pb_minibatch_gather: row size not chunkable");
    }
    const uint32_t chunk_bytes = (uint32_t)(row_bytes / chunks);
    const int64_t n_out = mb_count * rows * bptt;
    RowMap g{N, H, n_mb, rows, bptt, mb_begin};
    const size_t smem = (size_t)STAGES * MAX_CHUNK;
    PB_CUDA(cudaFuncSetAttribute(k_gather_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_gather_tma<<<grid_for(n_out * chunks), 32, smem, s>>>((const unsigned char*)obs, (unsigned char*)dst, row_bytes,
                                                            chunk_bytes, chunks, n_out, g);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_image_pack(const void* new_frames, int64_t frame_stride, const void* prev_obs, int64_t prev_stride,
                             void* obs_out, int64_t out_stride, const uint8_t* reset_mask, int64_t num_envs,
                             int64_t frame_bytes, int32_t stack, void* stream) {
    PB_REQUIRE(num_envs >= 0 && frame_bytes > 0 && stack >= 1, PB_ERR_INVALID, "pb_image_pack: bad sizes");
    if (num_envs == 0) return PB_OK;
    PB_REQUIRE(new_frames && obs_out && (prev_obs || stack == 1), PB_ERR_INVALID, "pb_image_pack: null pointer");
    PB_REQUIRE(frame_bytes % 16 == 0 && frame_stride % 16 == 0 && prev_stride % 16 == 0 && out_stride % 16 == 0 &&
                   ((uintptr_t)new_frames & 15) == 0 && ((uintptr_t)prev_obs & 15) == 0 && ((uintptr_t)obs_out & 15) == 0,
               PB_ERR_INVALID, "pb_image_pack: frames, strides and pointers must be multiples of 16 bytes");
    PB_REQUIRE(frame_bytes * stack <= MAX_CHUNK, PB_ERR_UNSUPPORTED,
               "pb_image_pack: stacked row of %lld bytes exceeds the %u-byte stage buffer",
               (long long)(frame_bytes * stack), MAX_CHUNK);
    PB_REQUIRE(out_stride >= frame_bytes * stack, PB_ERR_INVALID, "pb_image_pack: out_stride too small");
    const size_t smem = (size_t)STAGES * MAX_CHUNK;
    PB_CUDA(cudaFuncSetAttribute(k_image_pack, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_image_pack<<<grid_for(num_envs), 32, smem, (cudaStream_t)stream>>>(
        (const unsigned char*)new_frames, frame_stride, (const unsigned char*)prev_obs, prev_stride,
        (unsigned char*)obs_out, out_stride, reset_mask, num_envs, (uint32_t)frame_bytes, stack);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
