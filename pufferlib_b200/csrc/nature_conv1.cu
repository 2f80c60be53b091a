// nature_conv1.cu -- the first convolution of models.Convolutional (NatureCNN: Conv2d(C, 32, 8, stride=4) + ReLU on
// (C, 84, 84) uint8 frame stacks, C = framestack = 4 or 1, pufferlib/models.py:113-157) read straight from the uint8 rows
// (sm_90a).  Both kernels are templates over C; what follows describes C = 4, and C = 1 is the same with K = 64 (4
// k-pairs), 7 056-byte rows and the weight gradient's warps split as noted there.
//
// The stock path runs `network(x.float() / 255)`: two fp32 copies of every frame stack (4 bytes per pixel) before cuDNN
// reads one, and autograd keeps the scaled copy alive for the weight gradient.  Here the bytes are read once, in place.
// Implicit GEMM per frame stack: M = 400 output pixels (20 x 20), N = 32 output channels, K = 256 with
// k = c*64 + ky*8 + kx, on mma.sync m16n8k8 TF32 tensor-core tiles with fp32 accumulation.  A byte converted to fp32 is an
// exact TF32 value; the 1/255 is folded into the epilogue.
//
// k_conv1_fwd   y = relu(S / 255 + b) with S = conv(x, W), fp32 NCHW [m][32][20][20] (the tensor conv2 reads next).
//               Persistent CTAs of 5 warps; each 28 224-byte row is staged into shared memory by cp.async.bulk on an
//               mbarrier, two stages, so the next row's copy runs under the current row's product.  W (TF32, cvt.rna) is
//               resident in shared memory in B-fragment order; warp w owns m-tiles w, w + 5, ..., w + 20 of the row.
//               The epilogue goes through a per-warp [32][16] tile so that y is written with whole 16-byte stores.
// k_conv1_wgrad dW[co][k] = sum over rows and pixels of dz * x_col / 255 and db = sum dz, with dz = dy * (y > 0)
//               (threshold_backward) formed in registers and never written.  Per row: dz -> shared memory (TF32, cvt.rna),
//               x staged as in the forward; GEMM M = 32 channels, N = 256 k, K = 400 pixels, warp w owning 32 k columns.
//               C = 1 has 64 k columns: warp w owns columns 32 (w & 1) .. +31 over every fourth 8-pixel k-step from
//               w >> 1, and the four warps of a column half are summed in shared memory, in warp order, at the end.
//               Rows are split over a fixed number of CTAs (WG_CTAS, independent of the device) into fp32 partial rows,
//               summed in a fixed order by k_reduce_partials: two launches on the same inputs give the same bits.
//
// k-slot order.  Inside a pair of k-steps for (c, ky, ky + 1), lane t of a fragment quad reads ONE 32-bit word: bytes
// kx = 4(t & 1) .. +3 of input row ky + (t >> 1).  Its bytes 0, 1 are the A elements (slot t, slot t + 4) of the first
// k-step and bytes 2, 3 those of the second, so the matching B fragment (b0, b1 | b0, b1) of output channel co is the four
// adjacent weights W[co][c*64 + (ky + (t >> 1))*8 + 4(t & 1) + 0..3]: one 16-byte shared load per n-tile and k-pair.
#include "pb_common.cuh"
#include "reduce_partials.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace {

constexpr int C1_PLANE = 84 * 84;
template <int C>
constexpr int C1_ROW = C * C1_PLANE;    // bytes of one frame stack
template <int C>
constexpr int C1_K = 64 * C;
constexpr int C1_PIX = 400;             // 20 x 20 output pixels
constexpr int C1_CO = 32;
constexpr int C1_Y = C1_CO * C1_PIX;   // floats of one output row
constexpr int C1_STAGES = 2;
constexpr float C1_INV255 = 1.0f / 255.0f;

constexpr int FW_WARPS = 5;
constexpr int FW_THREADS = FW_WARPS * 32;
constexpr int FW_MT = 25 / FW_WARPS;   // m-tiles (16 pixels) per warp and row
constexpr int FW_OLD = 20;             // output tile row stride (floats): 16 pixels + 4, conflict-free fragment stores

constexpr int WG_THREADS = 256;
constexpr int WG_CTAS = 264;           // row split of the weight gradient: fixed, so the summation order is too
constexpr int WG_DZLD = 404;           // dz row stride (floats): 400 + 4, conflict-free A-fragment loads
template <int C>
constexpr int WG_PSTRIDE = C1_CO * C1_K<C> + C1_CO;   // partial row: dW [32][64 C] | db [32]

template <int C>
struct FwdSmem {
    unsigned char x[C1_STAGES][C1_ROW<C>];
    uint4 w[4 * C][4][32];                    // [k-pair][n-tile][lane]: (b0, b1) of both k-steps, TF32 bits
    float out[FW_WARPS][C1_CO][FW_OLD];
    uint64_t bar[C1_STAGES];
};

template <int C>
struct WgSmem {
    unsigned char x[C1_STAGES][C1_ROW<C>];
    float dz[C1_CO][WG_DZLD];                 // TF32 bits of dz
    uint64_t bar[C1_STAGES];
};

// byte j of w as fp32 (exact): 0x4B0000bj is 2^23 + bj
__device__ __forceinline__ uint32_t byte_f32(uint32_t w, int j) {
    return __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540 | j)) - 8388608.0f);
}

// byte offset of output pixel p's receptive field (row 4 oy, column 4 ox of channel 0) in a frame stack
__device__ __forceinline__ int pix_base(int p) { return (p / 20) * (4 * 84) + (p % 20) * 4; }

// Where row r (the r-th frame stack the kernels process, the r-th row of y and dy) is read from.  Both kernels are
// templates over this, and it is the only thing that differs between the dense and the segment entry points.
struct DenseRows {            // row r at x + r * stride
    const unsigned char* x;
    int64_t stride;
    __device__ __forceinline__ const unsigned char* operator()(int64_t r) const { return x + r * stride; }
};

struct SegmentRows {          // row r = b*T + t, segment b = (e, g) = (b / groups, b % groups): x + e*se + g*sg + t*st
    const unsigned char* x;
    int64_t se, sg, st;
    int32_t steps, groups;
    __device__ __forceinline__ const unsigned char* operator()(int64_t r) const {
        const int64_t b = r / steps, e = b / groups;
        return x + e * se + (b - e * groups) * sg + (r - b * steps) * st;
    }
};

template <int C>
__device__ __forceinline__ void issue_row(unsigned char* dst, uint64_t* bar, const unsigned char* src) {
    mbar_expect_tx(bar, C1_ROW<C>);
    tma_load_1d(dst, src, C1_ROW<C>, bar);
}

template <int C, class Rows>
__global__ void __launch_bounds__(FW_THREADS, 2) k_conv1_fwd(Rows rows, int64_t m, const float* __restrict__ w,
                                                             const float* __restrict__ b, float* __restrict__ y) {
    extern __shared__ __align__(128) unsigned char dyn[];
    FwdSmem<C>& s = *reinterpret_cast<FwdSmem<C>*>(dyn);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int64_t n_rows = (m - blockIdx.x + gridDim.x - 1) / gridDim.x;   // rows blockIdx.x + i * gridDim.x
    if (threadIdx.x == 0) {
        for (int st = 0; st < C1_STAGES; ++st) mbar_init(&s.bar[st], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int i = 0; i < C1_STAGES && i < n_rows; ++i)
            issue_row<C>(s.x[i], &s.bar[i], rows(blockIdx.x + (int64_t)i * gridDim.x));
    // W in B-fragment order (the header comment), rounded to TF32
    for (int e = threadIdx.x; e < 4 * C * 4 * 32; e += FW_THREADS) {
        const int p = e >> 7, nt = (e >> 5) & 3, l = e & 31, lg = l >> 2, lt = l & 3;
        const float4 v = __ldg(reinterpret_cast<const float4*>(
            w + (8 * nt + lg) * C1_K<C> + (p >> 2) * 64 + (2 * (p & 3) + (lt >> 1)) * 8 + 4 * (lt & 1)));
        s.w[p][nt][l] = make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
    }
    float bias[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        bias[nt][0] = __ldg(b + 8 * nt + 2 * t);
        bias[nt][1] = __ldg(b + 8 * nt + 2 * t + 1);
    }
    int pb0[FW_MT], pb1[FW_MT];   // receptive-field offsets of the fragment rows g and g + 8 of each m-tile
#pragma unroll
    for (int i = 0; i < FW_MT; ++i) {
        const int mt = warp + FW_WARPS * i;
        pb0[i] = pix_base(16 * mt + g);
        pb1[i] = pix_base(16 * mt + g + 8);
    }
    const int toff = (t >> 1) * 84 + 4 * (t & 1);
    __syncthreads();   // W staged

    float* so = &s.out[warp][0][0];
    for (int64_t i = 0; i < n_rows; ++i) {
        const int st = (int)(i % C1_STAGES);
        const int64_t row = blockIdx.x + i * gridDim.x;
        mbar_wait(&s.bar[st], (uint32_t)((i / C1_STAGES) & 1));
        const unsigned char* xs = s.x[st];
        float acc[FW_MT][4][4];
#pragma unroll
        for (int a = 0; a < FW_MT; ++a)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[a][nt][e] = 0.f;
#pragma unroll 2
        for (int p = 0; p < 4 * C; ++p) {   // k-steps 2p, 2p + 1: channel p >> 2, kernel rows 2 (p & 3) + 0 / 1
            const int koff = (p >> 2) * C1_PLANE + 2 * (p & 3) * 84 + toff;
            uint4 bf[4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) bf[nt] = s.w[p][nt][lane];
#pragma unroll
            for (int a = 0; a < FW_MT; ++a) {
                const uint32_t w0 = *reinterpret_cast<const uint32_t*>(xs + pb0[a] + koff);
                const uint32_t w1 = *reinterpret_cast<const uint32_t*>(xs + pb1[a] + koff);
                const uint32_t fa[4] = {byte_f32(w0, 0), byte_f32(w1, 0), byte_f32(w0, 1), byte_f32(w1, 1)};
                const uint32_t fb[4] = {byte_f32(w0, 2), byte_f32(w1, 2), byte_f32(w0, 3), byte_f32(w1, 3)};
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    mma_tf32(acc[a][nt], fa, bf[nt].x, bf[nt].y);
                    mma_tf32(acc[a][nt], fb, bf[nt].z, bf[nt].w);
                }
            }
        }
        __syncthreads();   // every warp is done with stage st: refill it with the row after next
        if (threadIdx.x == 0 && i + C1_STAGES < n_rows)
            issue_row<C>(s.x[st], &s.bar[st], rows(row + (int64_t)C1_STAGES * gridDim.x));
        float* yrow = y + row * C1_Y;
#pragma unroll
        for (int a = 0; a < FW_MT; ++a) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int co = 8 * nt + 2 * t;
                so[co * FW_OLD + g] = fmaxf(fmaf(acc[a][nt][0], C1_INV255, bias[nt][0]), 0.f);
                so[(co + 1) * FW_OLD + g] = fmaxf(fmaf(acc[a][nt][1], C1_INV255, bias[nt][1]), 0.f);
                so[co * FW_OLD + g + 8] = fmaxf(fmaf(acc[a][nt][2], C1_INV255, bias[nt][0]), 0.f);
                so[(co + 1) * FW_OLD + g + 8] = fmaxf(fmaf(acc[a][nt][3], C1_INV255, bias[nt][1]), 0.f);
            }
            __syncwarp();
            float* dst = yrow + 16 * (warp + FW_WARPS * a);
#pragma unroll
            for (int q = 0; q < 4; ++q) {   // 32 channels x 4 float4 of the tile's 16 pixels
                const int j = lane + 32 * q, co = j >> 2, c4 = 4 * (j & 3);
                *reinterpret_cast<float4*>(dst + co * C1_PIX + c4) = *reinterpret_cast<const float4*>(so + co * FW_OLD + c4);
            }
            __syncwarp();
        }
    }
}

template <int C, class Rows>
__global__ void __launch_bounds__(WG_THREADS, 2) k_conv1_wgrad(Rows rows, int64_t m, const float* __restrict__ y,
                                                               const float* __restrict__ dy, float* __restrict__ partials) {
    extern __shared__ __align__(128) unsigned char dyn[];
    WgSmem<C>& s = *reinterpret_cast<WgSmem<C>*>(dyn);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int64_t n_rows = (m - blockIdx.x + gridDim.x - 1) / gridDim.x;
    if (threadIdx.x == 0) {
        for (int st = 0; st < C1_STAGES; ++st) mbar_init(&s.bar[st], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int i = 0; i < C1_STAGES && i < n_rows; ++i)
            issue_row<C>(s.x[i], &s.bar[i], rows(blockIdx.x + (int64_t)i * gridDim.x));

    // warp w: channel c = w >> 1, kernel rows 4 (w & 1) .. +3.  n-tile j, column n <-> kernel row 4 (w & 1) + (n >> 1),
    // kx = 4 (n & 1) + j: lane g reads the bytes of all four n-tiles as one word.  C = 1: channel 0, and the k-steps of
    // pixels 8 (w >> 1) + 32 i
    const int xoff = (C == 4 ? warp >> 1 : 0) * C1_PLANE + (4 * (warp & 1) + (g >> 1)) * 84 + 4 * (g & 1);
    const int p_first = C == 4 ? 0 : 8 * (warp >> 1);
    constexpr int P_STEP = C == 4 ? 8 : 32;
    float acc[2][4][4] = {};
    float dbs[4] = {};   // db of channels warp + 8q, this lane's pixels
    for (int64_t i = 0; i < n_rows; ++i) {
        const int st = (int)(i % C1_STAGES);
        const int64_t row = blockIdx.x + i * gridDim.x;
        // dz = dy * (y > 0) for the whole row: warp w takes channels w + 8q, lane l float4 l, l + 32, ... of each
        const float* yr = y + row * C1_Y;
        const float* dr = dy + row * C1_Y;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int co = warp + 8 * q;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = lane + 32 * jj;
                if (j < C1_PIX / 4) {
                    const float4 yv = __ldg(reinterpret_cast<const float4*>(yr + co * C1_PIX) + j);
                    const float4 dv = __ldg(reinterpret_cast<const float4*>(dr + co * C1_PIX) + j);
                    const float z0 = yv.x > 0.f ? dv.x : 0.f, z1 = yv.y > 0.f ? dv.y : 0.f;
                    const float z2 = yv.z > 0.f ? dv.z : 0.f, z3 = yv.w > 0.f ? dv.w : 0.f;
                    dbs[q] += z0; dbs[q] += z1; dbs[q] += z2; dbs[q] += z3;
                    *reinterpret_cast<uint4*>(&s.dz[co][4 * j]) = make_uint4(to_tf32(z0), to_tf32(z1), to_tf32(z2), to_tf32(z3));
                }
            }
        }
        __syncthreads();   // dz staged
        mbar_wait(&s.bar[st], (uint32_t)((i / C1_STAGES) & 1));
        const unsigned char* xs = s.x[st] + xoff;
#pragma unroll (C == 4 ? 2 : 1)
        for (int p0 = p_first; p0 < C1_PIX; p0 += P_STEP) {
            const uint32_t w0 = *reinterpret_cast<const uint32_t*>(xs + pix_base(p0 + t));
            const uint32_t w1 = *reinterpret_cast<const uint32_t*>(xs + pix_base(p0 + t + 4));
            uint32_t fa[2][4];
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                const float* z0 = &s.dz[16 * mi + g][p0 + t];
                const float* z8 = &s.dz[16 * mi + g + 8][p0 + t];
                fa[mi][0] = __float_as_uint(z0[0]);
                fa[mi][1] = __float_as_uint(z8[0]);
                fa[mi][2] = __float_as_uint(z0[4]);
                fa[mi][3] = __float_as_uint(z8[4]);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t b0 = byte_f32(w0, j), b1 = byte_f32(w1, j);
                mma_tf32(acc[0][j], fa[0], b0, b1);
                mma_tf32(acc[1][j], fa[1], b0, b1);
            }
        }
        __syncthreads();   // dz and stage st are free
        if (threadIdx.x == 0 && i + C1_STAGES < n_rows)
            issue_row<C>(s.x[st], &s.bar[st], rows(row + (int64_t)C1_STAGES * gridDim.x));
    }
    // this CTA's partial row: dW / 255 in k order, then db
    float* part = partials + (int64_t)blockIdx.x * WG_PSTRIDE<C>;
    const int kbase = (C == 4 ? warp >> 1 : 0) * 64 + (4 * (warp & 1)) * 8;
    if constexpr (C == 1) {
        // the four pixel quarters of each column half, summed in warp order by warps 0 and 1 (dz is free: the last
        // iteration ended on a barrier)
        float* red = &s.dz[0][0] + warp * 32 * 32 + lane;   // [8 warps][32 values][32 lanes]
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) red[(16 * mi + 4 * j + e) * 32] = acc[mi][j][e];
        __syncthreads();
        if (warp < 2) {
#pragma unroll
            for (int q = 1; q < 4; ++q)
#pragma unroll
                for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int e = 0; e < 4; ++e) acc[mi][j][e] += red[(2 * q * 32 + 16 * mi + 4 * j + e) * 32];
        }
    }
    if (C == 4 || warp < 2) {
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int co = 16 * mi + g + 8 * (e >> 1), n = 2 * t + (e & 1);
                    part[co * C1_K<C> + kbase + (n >> 1) * 8 + 4 * (n & 1) + j] = acc[mi][j][e] * C1_INV255;
                }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        float v = dbs[q];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) part[C1_CO * C1_K<C> + warp + 8 * q] = v;
    }
}

int check_frames(int frames, const char* who) {
    PB_REQUIRE(frames == 1 || frames == 4, PB_ERR_INVALID, "%s: frames must be 1 or 4, got %d", who, frames);
    return PB_OK;
}

int check_rows(int frames, const void* x, int64_t row_stride, int64_t m, const char* who) {
    const int row = frames * C1_PLANE;
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "%s: m must not be negative", who);
    PB_REQUIRE(x && ((uintptr_t)x & 15) == 0, PB_ERR_INVALID, "%s: x must be a 16-byte aligned device pointer", who);
    PB_REQUIRE(row_stride >= row && row_stride % 16 == 0, PB_ERR_INVALID,
               "%s: row_stride %lld must be >= %d and a multiple of 16", who, (long long)row_stride, row);
    return PB_OK;
}

// The segment entry points' checks: batch segments of `steps` rows, every stride (bytes) a whole aligned row or more
int check_segments(int frames, const void* x, int64_t batch, int32_t steps, int32_t groups, int64_t se, int64_t sg,
                   int64_t st, const char* who) {
    const int row = frames * C1_PLANE;
    PB_REQUIRE(batch >= 0 && steps >= 1, PB_ERR_INVALID, "%s: need batch >= 0 and steps >= 1", who);
    PB_REQUIRE(groups >= 1 && batch % groups == 0, PB_ERR_INVALID, "%s: need groups >= 1 dividing batch (got %d, %lld)",
               who, groups, (long long)batch);
    PB_REQUIRE(x && ((uintptr_t)x & 15) == 0, PB_ERR_INVALID, "%s: x must be a 16-byte aligned device pointer", who);
    for (const int64_t stride : {se, sg, st})
        PB_REQUIRE(stride >= row && stride % 16 == 0, PB_ERR_INVALID,
                   "%s: stride %lld must be >= %d and a multiple of 16", who, (long long)stride, row);
    return PB_OK;
}

template <int C, class Rows>
int forward(const char* who, Rows rows, int64_t m, const float* w, const float* b, float* y, void* stream) {
    PB_REQUIRE(w && b && y && ((uintptr_t)w & 15) == 0 && ((uintptr_t)b & 3) == 0 && ((uintptr_t)y & 15) == 0,
               PB_ERR_INVALID, "%s: w and y must be 16-byte aligned, b 4-byte aligned", who);
    if (m == 0) return PB_OK;
    const int smem = (int)sizeof(FwdSmem<C>);
    PB_CUDA(cudaFuncSetAttribute(k_conv1_fwd<C, Rows>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int grid = (int)(m < 2 * (int64_t)PB_NUM_SMS ? m : 2 * (int64_t)PB_NUM_SMS);
    k_conv1_fwd<C><<<grid, FW_THREADS, smem, (cudaStream_t)stream>>>(rows, m, w, b, y);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

template <int C, class Rows>
int wgrad(const char* who, Rows rows, int64_t m, const float* y, const float* dy, float* dw, float* db, void* workspace,
          size_t workspace_bytes, void* stream) {
    PB_REQUIRE(y && dy && dw && db && workspace && ((uintptr_t)y & 15) == 0 && ((uintptr_t)dy & 15) == 0 &&
                   ((uintptr_t)dw & 3) == 0 && ((uintptr_t)db & 3) == 0 && ((uintptr_t)workspace & 15) == 0,
               PB_ERR_INVALID, "%s: y, dy and workspace must be 16-byte aligned, dw and db 4-byte aligned", who);
    PB_REQUIRE(workspace_bytes >= pb_conv1_u8_wgrad_workspace_bytes(m), PB_ERR_INVALID, "%s: workspace too small", who);
    if (m == 0) return PB_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const int smem = (int)sizeof(WgSmem<C>);
    PB_CUDA(cudaFuncSetAttribute(k_conv1_wgrad<C, Rows>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int ctas = (int)(m < WG_CTAS ? m : WG_CTAS);
    float* part = (float*)workspace;
    k_conv1_wgrad<C><<<ctas, WG_THREADS, smem, s>>>(rows, m, y, dy, part);
    PB_LAUNCH_CHECK();
    k_reduce_partials<<<(C1_CO * C1_K<C> * 32 + 255) / 256, 256, 0, s>>>(part, ctas, WG_PSTRIDE<C>, C1_CO * C1_K<C>, dw);
    PB_LAUNCH_CHECK();
    k_reduce_partials<<<(C1_CO * 32 + 255) / 256, 256, 0, s>>>(part + C1_CO * C1_K<C>, ctas, WG_PSTRIDE<C>, C1_CO, db);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

// The entry points' bodies: the checks of an S-frame row (frames = S), then the C = frames instance.  Every refusal
// returns before anything is launched.
int dense_forward(const char* who, int frames, const uint8_t* x, int64_t row_stride, int64_t m, const float* w,
                  const float* b, float* y, void* stream) {
    int rc = check_frames(frames, who);
    if (rc == PB_OK) rc = check_rows(frames, x, row_stride, m, who);
    if (rc != PB_OK) return rc;
    const DenseRows rows{x, row_stride};
    return frames == 1 ? forward<1>(who, rows, m, w, b, y, stream) : forward<4>(who, rows, m, w, b, y, stream);
}

int segment_forward(const char* who, int frames, const uint8_t* x, int64_t batch, int32_t steps, int32_t groups,
                    int64_t se, int64_t sg, int64_t st, const float* w, const float* b, float* y, void* stream) {
    int rc = check_frames(frames, who);
    if (rc == PB_OK) rc = check_segments(frames, x, batch, steps, groups, se, sg, st, who);
    if (rc != PB_OK) return rc;
    const SegmentRows rows{x, se, sg, st, steps, groups};
    return frames == 1 ? forward<1>(who, rows, batch * steps, w, b, y, stream)
                       : forward<4>(who, rows, batch * steps, w, b, y, stream);
}

int dense_wgrad(const char* who, int frames, const uint8_t* x, int64_t row_stride, int64_t m, const float* y,
                const float* dy, float* dw, float* db, void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_frames(frames, who);
    if (rc == PB_OK) rc = check_rows(frames, x, row_stride, m, who);
    if (rc != PB_OK) return rc;
    const DenseRows rows{x, row_stride};
    return frames == 1 ? wgrad<1>(who, rows, m, y, dy, dw, db, workspace, workspace_bytes, stream)
                       : wgrad<4>(who, rows, m, y, dy, dw, db, workspace, workspace_bytes, stream);
}

int segment_wgrad(const char* who, int frames, const uint8_t* x, int64_t batch, int32_t steps, int32_t groups,
                  int64_t se, int64_t sg, int64_t st, const float* y, const float* dy, float* dw, float* db,
                  void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_frames(frames, who);
    if (rc == PB_OK) rc = check_segments(frames, x, batch, steps, groups, se, sg, st, who);
    if (rc != PB_OK) return rc;
    const SegmentRows rows{x, se, sg, st, steps, groups};
    return frames == 1 ? wgrad<1>(who, rows, batch * steps, y, dy, dw, db, workspace, workspace_bytes, stream)
                       : wgrad<4>(who, rows, batch * steps, y, dy, dw, db, workspace, workspace_bytes, stream);
}

}  // namespace

extern "C" int pb_conv1_u8_forward(const uint8_t* x, int64_t row_stride, int64_t m, const float* w, const float* b, float* y,
                                   void* stream) {
    return dense_forward("pb_conv1_u8_forward", 4, x, row_stride, m, w, b, y, stream);
}

extern "C" int pb_conv1_u8_forward_rows(const uint8_t* x, int64_t batch, int32_t steps, int32_t groups, int64_t stride_e,
                                        int64_t stride_g, int64_t stride_t, const float* w, const float* b, float* y,
                                        void* stream) {
    return segment_forward("pb_conv1_u8_forward_rows", 4, x, batch, steps, groups, stride_e, stride_g, stride_t, w, b, y,
                           stream);
}

extern "C" size_t pb_conv1_u8_wgrad_workspace_bytes(int64_t m) {   // both C: a C = 1 partial row is the shorter one
    const int64_t ctas = m < WG_CTAS ? m : WG_CTAS;
    return ctas <= 0 ? 16 : (size_t)ctas * WG_PSTRIDE<4> * sizeof(float);
}

extern "C" int pb_conv1_u8_wgrad(const uint8_t* x, int64_t row_stride, int64_t m, const float* y, const float* dy, float* dw,
                                 float* db, void* workspace, size_t workspace_bytes, void* stream) {
    return dense_wgrad("pb_conv1_u8_wgrad", 4, x, row_stride, m, y, dy, dw, db, workspace, workspace_bytes, stream);
}

extern "C" int pb_conv1_u8_wgrad_rows(const uint8_t* x, int64_t batch, int32_t steps, int32_t groups, int64_t stride_e,
                                      int64_t stride_g, int64_t stride_t, const float* y, const float* dy, float* dw,
                                      float* db, void* workspace, size_t workspace_bytes, void* stream) {
    return segment_wgrad("pb_conv1_u8_wgrad_rows", 4, x, batch, steps, groups, stride_e, stride_g, stride_t, y, dy, dw, db,
                         workspace, workspace_bytes, stream);
}

extern "C" int pb_conv1_u8_forward_ex(int32_t frames, const uint8_t* x, int64_t row_stride, int64_t m, const float* w,
                                      const float* b, float* y, void* stream) {
    return dense_forward("pb_conv1_u8_forward_ex", frames, x, row_stride, m, w, b, y, stream);
}

extern "C" int pb_conv1_u8_forward_rows_ex(int32_t frames, const uint8_t* x, int64_t batch, int32_t steps, int32_t groups,
                                           int64_t stride_e, int64_t stride_g, int64_t stride_t, const float* w,
                                           const float* b, float* y, void* stream) {
    return segment_forward("pb_conv1_u8_forward_rows_ex", frames, x, batch, steps, groups, stride_e, stride_g, stride_t, w,
                           b, y, stream);
}

extern "C" int pb_conv1_u8_wgrad_ex(int32_t frames, const uint8_t* x, int64_t row_stride, int64_t m, const float* y,
                                    const float* dy, float* dw, float* db, void* workspace, size_t workspace_bytes,
                                    void* stream) {
    return dense_wgrad("pb_conv1_u8_wgrad_ex", frames, x, row_stride, m, y, dy, dw, db, workspace, workspace_bytes, stream);
}

extern "C" int pb_conv1_u8_wgrad_rows_ex(int32_t frames, const uint8_t* x, int64_t batch, int32_t steps, int32_t groups,
                                         int64_t stride_e, int64_t stride_g, int64_t stride_t, const float* y,
                                         const float* dy, float* dw, float* db, void* workspace, size_t workspace_bytes,
                                         void* stream) {
    return segment_wgrad("pb_conv1_u8_wgrad_rows_ex", frames, x, batch, steps, groups, stride_e, stride_g, stride_t, y, dy,
                         dw, db, workspace, workspace_bytes, stream);
}
