// mlp_tail.cu -- backward of the policy's "tail" (ReLU -> action/value heads) in one pass over the hidden layer (sm_90a).
//
// The configured policy is models.Default (reference pufferlib/models.py:12-62): Linear(obs->H)+ReLU, then two
// heads H->n_act and H->1.  In train (clean_pufferl.py:193-244) the backward of everything after the encoder GEMM is
// memory-bound work on [M, H] tensors that ATen runs as five launches, each re-reading 268 MB at M = 524288:
//   dHidden = dOut @ W_heads           (skinny GEMM, 8 columns)         dW_heads = dOut^T @ hidden   (skinny GEMM)
//   db_heads = sum_rows dOut           dPre = dHidden * (hidden > 0)    db_enc = sum_rows dPre
// This kernel does all five reading `hidden` ONCE and writing dPre once (2 * 4H + 4R B per row).  The dense H x H
// encoder GEMMs (forward, and dW_enc = dPre^T @ obs) stay on cuBLAS tensor cores.
// R = the padded head rows: 8 for n_act <= 7, 16 for 8 <= n_act <= 15, 32 for 16 <= n_act <= 31
// (models.Default.head_matrix); H = 128, 256, 384 or 512.  One template, k_mlp_tail_bwd<R, TMA>, serves them all.
// A warp owns rows; a lane owns VEC adjacent columns of a slice of SW = 32 VEC columns (512 B coalesced per row at
// VEC = 4), and the grid runs over the slices.  The head weights live in registers (R x VEC per lane); the per-lane
// accumulators (dW: R x VEC, db_enc: VEC, db_heads) are reduced over the block's warps in shared memory and
// written as ONE partial row per block; a second tiny kernel sums the partials in a fixed order (deterministic, no
// atomics).
// Registers at R = 16: the weights and the dW accumulators alone are 128 per thread, so the kernel runs one 256-thread
// CTA per SM (the TMA ring still keeps 72 KB per SM in flight).  Moving W_heads to shared memory would add 16 LDS.128
// per row and warp to the 5 the row needs, about the whole shared-memory bandwidth budget of a row at HBM speed, so the
// weights stay in registers.
#include <type_traits>

#include "pb_common.cuh"
#include "reduce_partials.cuh"
#include "tma.cuh"

namespace {

constexpr int MT_THREADS = 256;
constexpr int MT_WARPS = MT_THREADS / 32;
constexpr int ROWS_PER_BLOCK = 512;
constexpr int TT_STAGES = 4;   // TMA ring: stages of TT_CHUNK rows
constexpr int TT_CHUNK = 32;

// Columns per lane.  At R = 32 four columns would take 4R weights and 4R dW accumulators, 256 registers per lane before
// anything else, so a lane owns two there.
template <int R>
constexpr int TAIL_VEC = R == 32 ? 2 : 4;

// a lane's VEC adjacent columns of one row: one 16- or 8-byte access
template <int VEC>
union Cols {
    std::conditional_t<VEC == 4, float4, float2> v;
    float f[VEC];
};

// db_heads sums of a lane: R <= 16 all R columns of dOut, R = 32 column `lane`
template <int R>
constexpr int TAIL_SUMS = R == 32 ? 1 : R;

// the row's R head gradients from R / 4 float4s (every lane of the warp reads the same bytes: a broadcast), added to
// the db_heads sums.  At R <= 16 every lane adds all R from its registers, which costs less time than a 4-byte load per
// row; at R = 32 that would be 32 more registers and adds, so lane l loads and adds column l alone.
template <int R>
__device__ __forceinline__ void tail_load_dout(const float* src, float (&d)[R], float (&acc_d)[TAIL_SUMS<R>]) {
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        const float4 v = *reinterpret_cast<const float4*>(src + 4 * j);
        d[4 * j] = v.x; d[4 * j + 1] = v.y; d[4 * j + 2] = v.z; d[4 * j + 3] = v.w;
    }
    if constexpr (R == 32) {
        acc_d[0] += src[threadIdx.x & 31];
    } else {
#pragma unroll
        for (int k = 0; k < R; ++k) acc_d[k] += d[k];
    }
}

// one row: the lane's dPre columns g = relu'(h) * sum_k d[k] w[k] (one fmaf chain in k order per column), returned, and
// its accumulators dW_heads += d[k] h, db_enc += g
template <int R, int VEC>
__device__ __forceinline__ Cols<VEC> tail_row(const float (&d)[R], const Cols<VEC>& h, const Cols<VEC> (&w)[R],
                                              Cols<VEC> (&acc_w)[R], Cols<VEC>& acc_b) {
    Cols<VEC> g;
#pragma unroll
    for (int v = 0; v < VEC; ++v) g.f[v] = 0.f;
#pragma unroll
    for (int k = 0; k < R; ++k)
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            g.f[v] = fmaf(d[k], w[k].f[v], g.f[v]);
            acc_w[k].f[v] = fmaf(d[k], h.f[v], acc_w[k].f[v]);
        }
#pragma unroll
    for (int v = 0; v < VEC; ++v) {   // ReLU backward (threshold_backward: the gradient passes where h > 0)
        g.f[v] = h.f[v] > 0.f ? g.f[v] : 0.f;
        acc_b.f[v] += g.f[v];
    }
    return g;
}

// The block's sum of every warp's accumulators into its [R*H | H | R] partial row, in R / 8 passes of 8 dW_heads rows
// through s_red; pass 0 also carries db_enc and (slice 0) db_heads.  Each entry is the sum of the 8 warps in warp order.
template <int R, int VEC, int RSTRIDE>
__device__ __forceinline__ void tail_reduce(const Cols<VEC> (&acc_w)[R], const Cols<VEC>& acc_b,
                                            const float (&acc_d)[TAIL_SUMS<R>], float (*s_red)[RSTRIDE], float* out,
                                            int h, int col0) {
    constexpr int SW = 32 * VEC;
    using V = decltype(Cols<VEC>::v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float acc_o = acc_d[0];   // lane l < R: db_heads column l
#pragma unroll
    for (int k = 1; k < TAIL_SUMS<R>; ++k) acc_o = lane == k ? acc_d[k] : acc_o;
    float* mine = s_red[warp];
#pragma unroll
    for (int pass = 0; pass < R / 8; ++pass) {
        if (pass > 0) __syncthreads();   // the previous pass has been summed
#pragma unroll
        for (int k = 0; k < 8; ++k) *reinterpret_cast<V*>(mine + k * SW + VEC * lane) = acc_w[8 * pass + k].v;
        if (pass == 0) {
            *reinterpret_cast<V*>(mine + 8 * SW + VEC * lane) = acc_b.v;
            if (lane < R) mine[9 * SW + lane] = acc_o;
        }
        __syncthreads();
        const int n = pass == 0 ? (col0 == 0 ? RSTRIDE : 9 * SW) : 8 * SW;
        for (int j = threadIdx.x; j < n; j += MT_THREADS) {
            float s = 0.f;
#pragma unroll
            for (int wq = 0; wq < MT_WARPS; ++wq) s += s_red[wq][j];
            int64_t idx;
            if (j < 8 * SW) idx = (int64_t)(8 * pass + j / SW) * h + col0 + j % SW;     // dW_heads
            else if (j < 9 * SW) idx = (int64_t)R * h + col0 + (j - 8 * SW);          // db_enc
            else idx = (int64_t)R * h + h + (j - 9 * SW);                             // db_heads
            out[idx] = s;
        }
    }
}

// Grid (row blocks of 512, H / SW column slices): a CTA takes columns [col0, col0 + SW) of its rows (row stride h), a
// warp rows row0 + warp, + 8, ..., lane l columns col0 + VEC l ... + VEC - 1.  Every output but db_heads is per hidden
// column, so a slice writes its columns of the block's partial row and slice 0 also db_heads.  TMA (dOut contiguous [M][R]): the rows' slices and dOut rows are pulled into a 4-stage ring of 32
// rows by cp.async.bulk on mbarriers, so ~64 KB per CTA is in flight whatever the register budget, and the warps read
// them from shared memory; otherwise every lane loads its columns of the row and the row's dOut (a broadcast) itself.
template <int R, bool TMA>
__global__ void __launch_bounds__(MT_THREADS) k_mlp_tail_bwd(const float* __restrict__ dout, int64_t dout_stride,
                                                            const float* __restrict__ w_heads,   // [R][h]
                                                            const float* __restrict__ hidden,    // [M][h] post-ReLU
                                                            float* __restrict__ dpre,            // [M][h]
                                                            float* __restrict__ partials, int64_t m, int h) {
    constexpr int VEC = TAIL_VEC<R>, SW = 32 * VEC, RSTRIDE = 9 * SW + R;
    using V = decltype(Cols<VEC>::v);
    __shared__ float s_red[MT_WARPS][RSTRIDE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col0 = SW * (int)blockIdx.y;
    const int64_t row0 = (int64_t)blockIdx.x * ROWS_PER_BLOCK;
    const int64_t row_end = min(row0 + ROWS_PER_BLOCK, m);
    float* dcol = dpre + col0 + VEC * lane;

    // TMA: the ring, and the chunks of the block's rows
    extern __shared__ __align__(128) unsigned char dyn[];
    float* s_h = reinterpret_cast<float*>(dyn);                                          // [STAGES][CHUNK][SW]
    float* s_d = reinterpret_cast<float*>(dyn + (size_t)TT_STAGES * TT_CHUNK * SW * 4);   // [STAGES][CHUNK][R]
    __shared__ uint64_t bars[TT_STAGES];
    const int n_chunks = (int)((row_end - row0 + TT_CHUNK - 1) / TT_CHUNK);
    const bool whole = SW == 128 && h == SW;   // the slice is the whole row (h is a multiple of 128)
    auto issue = [&](int c) {   // warp 0; lane 0 arrives with the byte count before any lane copies
        const int st = c % TT_STAGES;
        const int64_t r = row0 + (int64_t)c * TT_CHUNK;
        const uint32_t rows = (uint32_t)min((int64_t)TT_CHUNK, row_end - r);
        if (lane == 0) {
            mbar_expect_tx(&bars[st], rows * (SW + R) * 4);
            tma_load_1d(s_d + (size_t)st * TT_CHUNK * R, dout + r * R, rows * R * 4, &bars[st]);
            if (whole) tma_load_1d(s_h + (size_t)st * TT_CHUNK * SW, hidden + r * SW, rows * SW * 4, &bars[st]);
        }
        if (!whole) {   // one copy per row of the slice's columns
            __syncwarp();
            if ((uint32_t)lane < rows)
                tma_load_1d(s_h + ((size_t)st * TT_CHUNK + lane) * SW, hidden + (r + lane) * h + col0, SW * 4, &bars[st]);
        }
    };
    if constexpr (TMA) {
        if (threadIdx.x == 0) {
            for (int st = 0; st < TT_STAGES; ++st) mbar_init(&bars[st], 1);
            mbar_fence_init();
        }
        __syncthreads();   // barriers initialised before warp 0 copies and anyone waits on them
        if (warp == 0)
            for (int c = 0; c < TT_STAGES && c < n_chunks; ++c) issue(c);
    }

    Cols<VEC> w[R], acc_w[R], acc_b;
    float acc_d[TAIL_SUMS<R>] = {};
#pragma unroll
    for (int k = 0; k < R; ++k) {
        w[k].v = *reinterpret_cast<const V*>(w_heads + (int64_t)k * h + col0 + VEC * lane);
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc_w[k].f[v] = 0.f;
    }
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc_b.f[v] = 0.f;

    if constexpr (TMA) {
        for (int c = 0; c < n_chunks; ++c) {
            const int st = c % TT_STAGES;
            mbar_wait(&bars[st], (uint32_t)((c / TT_STAGES) & 1));
            const int64_t r0 = row0 + (int64_t)c * TT_CHUNK;
            const int rows = (int)min((int64_t)TT_CHUNK, row_end - r0);
            const float* ch = s_h + (size_t)st * TT_CHUNK * SW;
            const float* cd = s_d + (size_t)st * TT_CHUNK * R;
            float* out = dcol + r0 * h;
#pragma unroll
            for (int i = 0; i < TT_CHUNK / MT_WARPS; ++i) {
                const int rl = warp + i * MT_WARPS;
                if (rl < rows) {
                    float d[R];
                    tail_load_dout<R>(cd + rl * R, d, acc_d);
                    Cols<VEC> hv;
                    hv.v = *reinterpret_cast<const V*>(ch + rl * SW + VEC * lane);
                    __stcs(reinterpret_cast<V*>(out + rl * h), tail_row<R, VEC>(d, hv, w, acc_w, acc_b).v);
                }
            }
            __syncthreads();   // everyone is done reading stage st
            if (warp == 0 && c + TT_STAGES < n_chunks) issue(c + TT_STAGES);
        }
    } else {
        const float* hcol = hidden + col0 + VEC * lane;
        // two rows per iteration at VEC = 4; at VEC = 2 the unrolled loop would take ~60 more registers
#pragma unroll(VEC == 4 ? 2 : 1)
        for (int64_t r = row0 + warp; r < row_end; r += MT_WARPS) {
            float d[R];
            tail_load_dout<R>(dout + r * dout_stride, d, acc_d);
            Cols<VEC> hv;
            hv.v = __ldcs(reinterpret_cast<const V*>(hcol + r * h));
            __stcs(reinterpret_cast<V*>(dcol + r * h), tail_row<R, VEC>(d, hv, w, acc_w, acc_b).v);
        }
    }
    tail_reduce<R, VEC, RSTRIDE>(acc_w, acc_b, acc_d, s_red, partials + (int64_t)blockIdx.x * (R * h + h + R), h, col0);
}

template <int R>
int launch_tail(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden, int64_t m, int h,
                float* dpre, float* workspace, int blocks, cudaStream_t s) {
    constexpr int SW = 32 * TAIL_VEC<R>;
    const dim3 grid((unsigned)blocks, (unsigned)(h / SW));
    if (dout_stride == R) {   // contiguous head gradients: the TMA ring
        const int smem = TT_STAGES * TT_CHUNK * (SW + R) * 4;
        PB_CUDA(cudaFuncSetAttribute(k_mlp_tail_bwd<R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        k_mlp_tail_bwd<R, true><<<grid, MT_THREADS, smem, s>>>(dout, R, w_heads, hidden, dpre, workspace, m, h);
    } else {
        k_mlp_tail_bwd<R, false><<<grid, MT_THREADS, 0, s>>>(dout, dout_stride, w_heads, hidden, dpre, workspace, m, h);
    }
    PB_LAUNCH_CHECK();
    return PB_OK;
}

}  // namespace

extern "C" size_t pb_mlp_tail_workspace_bytes_ex(int64_t m, int32_t hidden, int32_t head_rows) {
    if (m <= 0 || hidden <= 0 || (head_rows != 8 && head_rows != 16 && head_rows != 32)) return 16;
    const int64_t blocks = pb_ceil_div(m, ROWS_PER_BLOCK);
    return (size_t)blocks * (size_t)(head_rows * hidden + hidden + head_rows) * sizeof(float);
}

extern "C" size_t pb_mlp_tail_workspace_bytes(int64_t m, int32_t hidden) {
    return pb_mlp_tail_workspace_bytes_ex(m, hidden, 8);
}

extern "C" int pb_mlp_tail_backward_ex(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden,
                                       int64_t m, int32_t hidden_size, float* dpre, float* grads_out, void* workspace,
                                       size_t workspace_bytes, int32_t head_rows, void* stream) {
    PB_REQUIRE(m >= 1, PB_ERR_INVALID, "pb_mlp_tail_backward: m must be positive");
    PB_REQUIRE(hidden_size >= 128 && hidden_size <= 512 && hidden_size % 128 == 0, PB_ERR_UNSUPPORTED,
               "pb_mlp_tail_backward: hidden size %d (128, 256, 384 and 512 are built)", hidden_size);
    PB_REQUIRE(head_rows == 8 || head_rows == 16 || head_rows == 32, PB_ERR_UNSUPPORTED,
               "pb_mlp_tail_backward: head_rows %d (8, 16 and 32 are built)", head_rows);
    PB_REQUIRE(dout && w_heads && hidden && dpre && grads_out && workspace, PB_ERR_INVALID,
               "pb_mlp_tail_backward: null pointer");
    PB_REQUIRE(dout_stride >= head_rows && dout_stride % 4 == 0 && ((uintptr_t)dout & 15) == 0 &&
                   ((uintptr_t)hidden & 15) == 0 && ((uintptr_t)dpre & 15) == 0 && ((uintptr_t)w_heads & 15) == 0,
               PB_ERR_INVALID, "pb_mlp_tail_backward: dout needs %d padded columns; pointers must be 16-byte aligned",
               head_rows);
    PB_REQUIRE(workspace_bytes >= pb_mlp_tail_workspace_bytes_ex(m, hidden_size, head_rows), PB_ERR_INVALID,
               "pb_mlp_tail_backward: workspace too small");
    const int blocks = (int)pb_ceil_div(m, ROWS_PER_BLOCK);
    const int pstride = head_rows * hidden_size + hidden_size + head_rows;
    cudaStream_t s = (cudaStream_t)stream;
    float* ws = (float*)workspace;
    int rc;
    switch (head_rows) {
    case 8: rc = launch_tail<8>(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, ws, blocks, s); break;
    case 16: rc = launch_tail<16>(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, ws, blocks, s); break;
    default: rc = launch_tail<32>(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, ws, blocks, s); break;
    }
    if (rc != PB_OK) return rc;
    k_reduce_partials<<<(pstride * 32 + 255) / 256, 256, 0, s>>>((const float*)workspace, blocks, pstride, pstride,
                                                                 grads_out);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_mlp_tail_backward(const float* dout, int64_t dout_stride, const float* w_heads, const float* hidden,
                                    int64_t m, int32_t hidden_size, float* dpre, float* grads_out, void* workspace,
                                    size_t workspace_bytes, void* stream) {
    return pb_mlp_tail_backward_ex(dout, dout_stride, w_heads, hidden, m, hidden_size, dpre, grads_out, workspace,
                                   workspace_bytes, 8, stream);
}
