// nature_trunk.cu -- conv2 and conv3 of models.Convolutional (NatureCNN, pufferlib/models.py:113-157): Conv2d(32, 64, 4,
// stride=2) + ReLU on y1 [32][20][20] and Conv2d(64, 64, 3, stride=1) + ReLU on y2 [64][9][9], fp32 NCHW rows, on TF32
// mma.sync m16n8k8 tensor-core tiles with fp32 accumulation (sm_90a).  Every kernel is one template over the layer shape
// (Layer<C_in, H_in, kernel, stride>, C_out = 64), instantiated for both layers.
//
// GEMM k order.  The reduction index of the forward is tap-major, k' = tap * C_in + c with
// tap = ky * KS + kx, so that a k-step of 8 is 8 consecutive input channels at one tap; the weights are read from the
// stock [64][C_in][KS][KS] layout and dW is written back in it.  Every operand is rounded to TF32 with cvt.rna: x and dz
// once, in shared memory, W when it is laid out in B-fragment order.
//
// Shared memory decides the tiling.  W as TF32 is 128 KiB (conv2) / 144 KiB (conv3) and stays resident per CTA in
// B-fragment order (one 16-byte load per k-step pair, n-tile and lane), so the forward and the input gradient run one
// persistent CTA per SM.  A y1 row (50 KiB) does not fit beside W2 twice, so conv2's forward streams each row in two
// channel halves (25 KiB) through a two-stage cp.async.bulk ring: the copy of the next half runs under the product of
// the current one.  conv3's row (20.25 KiB) is one stage.
//
// k_trunk_fwd<L>   y = relu(conv(x, W) + b).  M = output pixels of one row (81 / 49, in 16-pixel m-tiles), N = 64,
//                  K = 512 / 576.  Warp w owns 2 m-tiles x 4 n-tiles.  Epilogue through a shared [64][P] row, written
//                  with 16-byte stores (a row of y is 20 736 / 12 544 bytes, a multiple of 16).
// k_trunk_dgrad<L> dx = conv_transpose(dz, W), dz = dy * (y > 0) (threshold_backward) formed in registers while the row
//                  is staged into shared memory as TF32, zero-padded to an 11 x 11 plane per channel; dz is never
//                  written.  Stride 2 (conv2) is split into its S^2 = 4 sub-pixel stride classes (py, px): input pixel
//                  (2a + py, 2b + px) takes the taps ky = py + 2 jy, kx = px + 2 jx from dz[a - jy][b - jx], a dense
//                  GEMM per class (M = 100 pixels, N = 32, K = 64 x 4) with no scatter and no atomics, so every dx
//                  element is written once by one thread.  Stride 1 (conv3) is the one class with 9 taps.
// k_trunk_wgrad<L> dW[co][k] = sum over rows and pixels of dz * im2col(x), db = sum dz.  Per row: dz staged as in the
//                  input gradient (TF32), x staged by cp.async.bulk (two stages, rounded in place); GEMM M = 64 channels,
//                  N = K columns in the stock k order (warp w owns 32 channels x K / 64 columns), reduction over the row's pixels padded to a multiple of 8
//                  with zero dz.  Rows are split over WG_CTAS CTAs (a constant, not the device's SM count) into fp32
//                  partial rows, summed in a fixed order by k_reduce_partials: deterministic.
#include "pb_common.cuh"
#include "reduce_partials.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace {

constexpr int CO = 64;
constexpr int STAGES = 2;
constexpr int WG_CTAS = 132;       // row split of the weight gradient: fixed, so the summation order is too
constexpr int WG_WARPS = 16;     // 8 column slices x 2 channel halves

template <int CIN_, int H_, int KS_, int S_, int FWD_CHUNKS_, int DG_MT_>
struct Layer {
    static constexpr int CIN = CIN_, H = H_, KS = KS_, S = S_;
    static constexpr int HO = (H - KS) / S + 1;        // 9 / 7
    static constexpr int HH = H * H, P = HO * HO;      // input plane, output pixels
    static constexpr int TAPS = KS * KS, K = CIN * TAPS;
    static constexpr int XROW = CIN * HH;              // floats of one input row
    static constexpr int YROW = CO * P;                // floats of one output row
    // forward
    static constexpr int FWD_CHUNKS = FWD_CHUNKS_, CPC = CIN / FWD_CHUNKS, XCH = CPC * HH;
    static constexpr int FWD_MTILES = (P + 15) / 16, FWD_WARPS = FWD_MTILES / 2 * 2;   // 2 m-tiles x 4 n-tiles a warp
    // input gradient: stride classes, dz plane padded by PAD on each side
    static constexpr int CLS = S * S, JT = KS / S, TAPC = JT * JT, HC = H / S, PC = HC * HC;
    static constexpr int PAD = JT - 1, DZW = HO + 2 * PAD, DZP = DZW * DZW;
    static constexpr int DG_KP = CO * TAPC / 16, DG_NTILES = CIN / 8;
    static constexpr int DG_MT = DG_MT_, DG_MG = ((PC + 15) / 16 + DG_MT - 1) / DG_MT, DG_NG = DG_NTILES / 4;
    static constexpr int DG_WARPS = CLS * DG_MG * DG_NG;
    // weight gradient
    static constexpr int PPAD = (P + 7) / 8 * 8, PLD = PPAD + ((36 - PPAD % 32) % 32);   // PLD = 4 mod 32
    static constexpr int WG_NT = K / 8 / (WG_WARPS / 2);
    static constexpr int PSTRIDE = CO * K + CO;        // partial row: dW [64][K] | db [64]
    static_assert(KS % S == 0 && H % S == 0 && HC <= HO + PAD && DZW >= HO + PAD + 1, "stride classes");
    static_assert(CPC % 16 == 0 && FWD_MTILES % 2 == 0 && DG_NTILES % 4 == 0 && K % (4 * WG_WARPS) == 0, "tiling");
    static_assert((XCH * 4) % 16 == 0 && (YROW * 4) % 16 == 0 && (XROW * 4) % 16 == 0, "16-byte rows");
};
using Conv2 = Layer<32, 20, 4, 2, 2, 4>;   // M = 81, K = 512
using Conv3 = Layer<64, 9, 3, 1, 1, 2>;    // M = 49, K = 576

template <class L> struct FwdSmem {
    uint4 w[L::K / 16][8][32];                  // [k-step pair][n-tile][lane]: (b0, b1) of both k-steps, TF32 bits
    float x[STAGES][L::XCH];
    float out[L::YROW];
    uint64_t bar[STAGES];
};
template <class L> struct DgSmem {
    uint4 w[L::CLS][L::DG_KP][L::DG_NTILES][32];
    float dz[CO * L::DZP];                      // TF32 bits, zero border
    float dx[L::XROW];
};
template <class L> struct WgSmem {
    float x[STAGES][L::XROW];
    float dz[CO * L::PLD];                      // TF32 bits, zero for pixels >= P
    int pix[L::PPAD];                           // offset of output pixel p's receptive field in an input row
    float db[CO];                               // this CTA's db, in row order
    uint64_t bar[STAGES];
};

__device__ __forceinline__ void prefetch_l2(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// round n floats of shared memory to TF32 in place (all threads), then order those generic writes before later
// cp.async.bulk writes to the same bytes
__device__ __forceinline__ void round_tf32_smem(float* p, int n) {
    for (int i = threadIdx.x; i < n / 4; i += blockDim.x) {
        float4 v = reinterpret_cast<float4*>(p)[i];
        reinterpret_cast<uint4*>(p)[i] = make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
    }
    fence_proxy_async_smem();
}

__device__ __forceinline__ void copy_out(float* dst, const float* src, int n) {
    for (int i = threadIdx.x; i < n / 4; i += blockDim.x)
        reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(src)[i];
}

// dz = dy * (y > 0) of one row into shared memory as TF32 at dz[co * ld + off(p)], warp w taking channels w + NW q;
// with db, the row's fp32 dz sum of each channel (lane sums, then a fixed shuffle tree) is added to db[co]
template <class L, int NW, class Off>
__device__ __forceinline__ void stage_dz(float* dzs, int ld, const float* yr, const float* dr, Off off, float* db) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll 1
    for (int co = warp; co < CO; co += NW) {
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < (L::P + 31) / 32; ++j) {
            const int p = lane + 32 * j;
            if (p < L::P) {
                const float z = __ldg(yr + co * L::P + p) > 0.f ? __ldg(dr + co * L::P + p) : 0.f;
                sum += z;
                dzs[co * ld + off(p)] = __uint_as_float(to_tf32(z));
            }
        }
        if (db) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            if (lane == 0) db[co] += sum;
        }
    }
}

// ---- forward ----------------------------------------------------------------------------------------------------------
template <class L>
__device__ __forceinline__ void issue_chunk(FwdSmem<L>& s, int st, const float* x, int64_t unit) {
    mbar_expect_tx(&s.bar[st], L::XCH * 4);
    tma_load_1d(s.x[st], x + unit * L::XCH, L::XCH * 4, &s.bar[st]);   // chunks of a row are consecutive
}

template <class L>
__global__ void __launch_bounds__(L::FWD_WARPS * 32, 1) k_trunk_fwd(const float* __restrict__ x, int64_t m,
                                                                    const float* __restrict__ w,
                                                                    const float* __restrict__ b, float* __restrict__ y) {
    extern __shared__ __align__(128) unsigned char dyn[];
    FwdSmem<L>& s = *reinterpret_cast<FwdSmem<L>*>(dyn);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int mg = warp >> 1, ng = warp & 1;
    const int64_t n_rows = (m - blockIdx.x + gridDim.x - 1) / gridDim.x;   // rows blockIdx.x + i * gridDim.x
    const int64_t n_units = n_rows * L::FWD_CHUNKS;
    auto unit_of = [&](int64_t u) { return (blockIdx.x + (u / L::FWD_CHUNKS) * gridDim.x) * L::FWD_CHUNKS + u % L::FWD_CHUNKS; };
    if (threadIdx.x == 0) {
        for (int st = 0; st < STAGES; ++st) mbar_init(&s.bar[st], 1);
        mbar_fence_init();
        for (int u = 0; u < STAGES && u < n_units; ++u) issue_chunk(s, u, x, unit_of(u));
    }
    // W in B-fragment order: k' = 16 kp + lt + 4 e (e = 0..3), n = co
    for (int e = threadIdx.x; e < L::K / 16 * 8 * 32; e += blockDim.x) {
        const int kp = e >> 8, nt = (e >> 5) & 7, l = e & 31, co = 8 * nt + (l >> 2);
        uint32_t v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int kk = 16 * kp + (l & 3) + 4 * q, tap = kk / L::CIN, c = kk % L::CIN;
            v[q] = to_tf32(__ldg(w + co * L::K + c * L::TAPS + tap));
        }
        s.w[kp][nt][l] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    float bias[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        bias[nt][0] = __ldg(b + 8 * (4 * ng + nt) + 2 * t);
        bias[nt][1] = __ldg(b + 8 * (4 * ng + nt) + 2 * t + 1);
    }
    int ro[2][2];   // receptive-field offsets of fragment rows g, g + 8 of each m-tile, plus channel t
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            int p = 16 * (2 * mg + i) + g + 8 * r;
            p = p < L::P ? p : L::P - 1;   // padding rows: computed, never stored
            ro[i][r] = L::S * (p / L::HO) * L::H + L::S * (p % L::HO) + t * L::HH;
        }
    __syncthreads();   // W staged, barriers initialised

    float acc[2][4][4] = {};
    for (int64_t u = 0; u < n_units; ++u) {
        const int st = (int)(u % STAGES), h = (int)(u % L::FWD_CHUNKS);
        mbar_wait(&s.bar[st], (uint32_t)((u / STAGES) & 1));
        round_tf32_smem(s.x[st], L::XCH);
        __syncthreads();
        const float* xs = s.x[st];
#pragma unroll
        for (int tap = 0; tap < L::TAPS; ++tap) {
            const int toff = (tap / L::KS) * L::H + tap % L::KS;
#pragma unroll
            for (int j = 0; j < L::CPC / 16; ++j) {
                const int kp = tap * (L::CIN / 16) + h * (L::CPC / 16) + j;
                uint4 bf[4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) bf[nt] = s.w[kp][4 * ng + nt][lane];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const float* a0 = xs + ro[i][0] + toff + 16 * j * L::HH;
                    const float* a1 = xs + ro[i][1] + toff + 16 * j * L::HH;
                    const uint32_t fa[4] = {__float_as_uint(a0[0]), __float_as_uint(a1[0]),
                                            __float_as_uint(a0[4 * L::HH]), __float_as_uint(a1[4 * L::HH])};
                    const uint32_t fb[4] = {__float_as_uint(a0[8 * L::HH]), __float_as_uint(a1[8 * L::HH]),
                                            __float_as_uint(a0[12 * L::HH]), __float_as_uint(a1[12 * L::HH])};
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        mma_tf32(acc[i][nt], fa, bf[nt].x, bf[nt].y);
                        mma_tf32(acc[i][nt], fb, bf[nt].z, bf[nt].w);
                    }
                }
            }
        }
        __syncthreads();   // every warp is done with stage st: refill it
        if (threadIdx.x == 0 && u + STAGES < n_units) issue_chunk(s, st, x, unit_of(u + STAGES));
        if (h == L::FWD_CHUNKS - 1) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int p = 16 * (2 * mg + i) + g + 8 * (e >> 1), co = 8 * (4 * ng + nt) + 2 * t + (e & 1);
                        if (p < L::P) s.out[co * L::P + p] = fmaxf(acc[i][nt][e] + bias[nt][e & 1], 0.f);
                        acc[i][nt][e] = 0.f;
                    }
            __syncthreads();
            copy_out(y + (unit_of(u) / L::FWD_CHUNKS) * L::YROW, s.out, L::YROW);
        }
    }
}

// ---- input gradient ---------------------------------------------------------------------------------------------------
template <class L>
__global__ void __launch_bounds__(L::DG_WARPS * 32, 1) k_trunk_dgrad(const float* __restrict__ y,
                                                                     const float* __restrict__ dy, int64_t m,
                                                                     const float* __restrict__ w, float* __restrict__ dx) {
    constexpr int MT = L::DG_MT;
    extern __shared__ __align__(128) unsigned char dyn[];
    DgSmem<L>& s = *reinterpret_cast<DgSmem<L>*>(dyn);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int cls = warp / (L::DG_MG * L::DG_NG), mg = (warp / L::DG_NG) % L::DG_MG, ng = warp % L::DG_NG;
    const int py = cls / L::S, px = cls % L::S;
    const int64_t n_rows = (m - blockIdx.x + gridDim.x - 1) / gridDim.x;
    // W in B-fragment order per class: k' = 16 kp + lt + 4 e = tapc * 64 + co, n = c
    for (int e = threadIdx.x; e < L::CLS * L::DG_KP * L::DG_NTILES * 32; e += blockDim.x) {
        const int l = e & 31, nt = (e >> 5) % L::DG_NTILES, kp = (e >> 5) / L::DG_NTILES % L::DG_KP;
        const int cl = (e >> 5) / L::DG_NTILES / L::DG_KP, c = 8 * nt + (l >> 2);
        uint32_t v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int kk = 16 * kp + (l & 3) + 4 * q, tapc = kk / CO, co = kk % CO;
            const int ky = cl / L::S + L::S * (tapc / L::JT), kx = cl % L::S + L::S * (tapc % L::JT);
            v[q] = to_tf32(__ldg(w + co * L::K + c * L::TAPS + ky * L::KS + kx));
        }
        s.w[cl][kp][nt][l] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    for (int i = threadIdx.x; i < CO * L::DZP; i += blockDim.x) s.dz[i] = 0.f;
    int ro[MT][2];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            int p = 16 * (MT * mg + i) + g + 8 * r;
            p = p < L::PC ? p : L::PC - 1;
            ro[i][r] = (p / L::HC + L::PAD) * L::DZW + p % L::HC + L::PAD + t * L::DZP;
        }
    __syncthreads();

    auto dz_off = [](int p) { return (p / L::HO + L::PAD) * L::DZW + p % L::HO + L::PAD; };
    for (int64_t i = 0; i < n_rows; ++i) {
        const int64_t row = blockIdx.x + i * gridDim.x;
        if (threadIdx.x == 0 && row + gridDim.x < m) {
            prefetch_l2(y + (row + gridDim.x) * L::YROW, L::YROW * 4);
            prefetch_l2(dy + (row + gridDim.x) * L::YROW, L::YROW * 4);
        }
        stage_dz<L, L::DG_WARPS>(s.dz, L::DZP, y + row * L::YROW, dy + row * L::YROW, dz_off, nullptr);
        __syncthreads();
        float acc[MT][4][4] = {};
#pragma unroll
        for (int tc = 0; tc < L::TAPC; ++tc) {
            const int shift = (tc / L::JT) * L::DZW + tc % L::JT;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                uint4 bf[4];
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) bf[nt] = s.w[cls][4 * tc + j][4 * ng + nt][lane];
#pragma unroll
                for (int a = 0; a < MT; ++a) {
                    const float* a0 = s.dz + ro[a][0] - shift + 16 * j * L::DZP;
                    const float* a1 = s.dz + ro[a][1] - shift + 16 * j * L::DZP;
                    const uint32_t fa[4] = {__float_as_uint(a0[0]), __float_as_uint(a1[0]),
                                            __float_as_uint(a0[4 * L::DZP]), __float_as_uint(a1[4 * L::DZP])};
                    const uint32_t fb[4] = {__float_as_uint(a0[8 * L::DZP]), __float_as_uint(a1[8 * L::DZP]),
                                            __float_as_uint(a0[12 * L::DZP]), __float_as_uint(a1[12 * L::DZP])};
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        mma_tf32(acc[a][nt], fa, bf[nt].x, bf[nt].y);
                        mma_tf32(acc[a][nt], fb, bf[nt].z, bf[nt].w);
                    }
                }
            }
        }
#pragma unroll
        for (int a = 0; a < MT; ++a)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int p = 16 * (MT * mg + a) + g + 8 * (e >> 1), c = 8 * (4 * ng + nt) + 2 * t + (e & 1);
                    if (p < L::PC)
                        s.dx[c * L::HH + (L::S * (p / L::HC) + py) * L::H + L::S * (p % L::HC) + px] = acc[a][nt][e];
                }
        __syncthreads();   // dz free, dx complete
        copy_out(dx + row * L::XROW, s.dx, L::XROW);
    }
}

// ---- weight gradient --------------------------------------------------------------------------------------------------
template <class L>
__device__ __forceinline__ void issue_row(WgSmem<L>& s, int st, const float* x, int64_t row) {
    mbar_expect_tx(&s.bar[st], L::XROW * 4);
    tma_load_1d(s.x[st], x + row * L::XROW, L::XROW * 4, &s.bar[st]);
}

template <class L>
__global__ void __launch_bounds__(WG_WARPS * 32, 1) k_trunk_wgrad(const float* __restrict__ x,
                                                                  const float* __restrict__ y,
                                                                  const float* __restrict__ dy, int64_t m,
                                                                  float* __restrict__ partials) {
    constexpr int NT = L::WG_NT;
    extern __shared__ __align__(128) unsigned char dyn[];
    WgSmem<L>& s = *reinterpret_cast<WgSmem<L>*>(dyn);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int64_t n_rows = (m - blockIdx.x + gridDim.x - 1) / gridDim.x;
    if (threadIdx.x == 0) {
        for (int st = 0; st < STAGES; ++st) mbar_init(&s.bar[st], 1);
        mbar_fence_init();
        for (int i = 0; i < STAGES && i < n_rows; ++i) issue_row(s, i, x, blockIdx.x + (int64_t)i * gridDim.x);
    }
    for (int i = threadIdx.x; i < CO * L::PLD; i += blockDim.x) s.dz[i] = 0.f;
    for (int i = threadIdx.x; i < CO; i += blockDim.x) s.db[i] = 0.f;
    for (int p = threadIdx.x; p < L::PPAD; p += blockDim.x)
        s.pix[p] = p < L::P ? L::S * (p / L::HO) * L::H + L::S * (p % L::HO) : 0;   // pixels >= P: dz is 0 there
    const int mh = warp & 1, ns = warp >> 1;   // channels 32 mh .. +31, columns 8 NT ns .. +8 NT - 1
    // column k = 8 (ns NT + j) + g in the stock order k = c * TAPS + tap: offset of (c, ky, kx) in an input row
    auto col = [&](int j) {
        const int kk = 8 * (ns * NT + j) + g, tap = kk % L::TAPS, c = kk / L::TAPS;
        return c * L::HH + (tap / L::KS) * L::H + tap % L::KS;
    };
    __syncthreads();

    float acc[2][NT][4] = {};
    auto dz_off = [](int p) { return p; };
    for (int64_t i = 0; i < n_rows; ++i) {
        const int st = (int)(i % STAGES);
        const int64_t row = blockIdx.x + i * gridDim.x;
        if (threadIdx.x == 0 && row + gridDim.x < m) {
            prefetch_l2(y + (row + gridDim.x) * L::YROW, L::YROW * 4);
            prefetch_l2(dy + (row + gridDim.x) * L::YROW, L::YROW * 4);
        }
        stage_dz<L, WG_WARPS>(s.dz, L::PLD, y + row * L::YROW, dy + row * L::YROW, dz_off, s.db);
        mbar_wait(&s.bar[st], (uint32_t)((i / STAGES) & 1));
        round_tf32_smem(s.x[st], L::XROW);
        __syncthreads();   // dz and x staged
        const float* xs = s.x[st];
#pragma unroll 2
        for (int ks = 0; ks < L::PPAD / 8; ++ks) {
            const int p0 = s.pix[8 * ks + t], p1 = s.pix[8 * ks + t + 4];
            uint32_t fa[2][4];
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                const float* z0 = s.dz + (32 * mh + 16 * mi + g) * L::PLD + 8 * ks + t;
                const float* z8 = z0 + 8 * L::PLD;
                fa[mi][0] = __float_as_uint(z0[0]);
                fa[mi][1] = __float_as_uint(z8[0]);
                fa[mi][2] = __float_as_uint(z0[4]);
                fa[mi][3] = __float_as_uint(z8[4]);
            }
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const float* xc = xs + col(j);
                const uint32_t b0 = __float_as_uint(xc[p0]), b1 = __float_as_uint(xc[p1]);
#pragma unroll
                for (int mi = 0; mi < 2; ++mi) mma_tf32(acc[mi][j], fa[mi], b0, b1);
            }
        }
        __syncthreads();   // dz and stage st are free
        if (threadIdx.x == 0 && i + STAGES < n_rows) issue_row(s, st, x, row + (int64_t)STAGES * gridDim.x);
    }
    // this CTA's partial row: dW in the stock [64][CIN][KS][KS] order, then db
    float* part = partials + (int64_t)blockIdx.x * L::PSTRIDE;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int co = 32 * mh + 16 * mi + g + 8 * (e >> 1), kk = 8 * (ns * NT + j) + 2 * t + (e & 1);
                part[co * L::K + kk] = acc[mi][j][e];
            }
    for (int i = threadIdx.x; i < CO; i += blockDim.x) part[CO * L::K + i] = s.db[i];   // after the loop's last barrier
}

// ---- host -------------------------------------------------------------------------------------------------------------
bool aligned16(const void* p) { return p && ((uintptr_t)p & 15) == 0; }
bool aligned4(const void* p) { return p && ((uintptr_t)p & 3) == 0; }

template <class L>
int forward(const float* x, int64_t m, const float* w, const float* b, float* y, cudaStream_t st) {
    const int smem = (int)sizeof(FwdSmem<L>);
    PB_CUDA(cudaFuncSetAttribute(k_trunk_fwd<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int grid = (int)(m < (int64_t)PB_NUM_SMS ? m : (int64_t)PB_NUM_SMS);
    k_trunk_fwd<L><<<grid, L::FWD_WARPS * 32, smem, st>>>(x, m, w, b, y);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

template <class L>
int dgrad(const float* y, const float* dy, const float* w, int64_t m, float* dx, cudaStream_t st) {
    const int smem = (int)sizeof(DgSmem<L>);
    PB_CUDA(cudaFuncSetAttribute(k_trunk_dgrad<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int grid = (int)(m < (int64_t)PB_NUM_SMS ? m : (int64_t)PB_NUM_SMS);
    k_trunk_dgrad<L><<<grid, L::DG_WARPS * 32, smem, st>>>(y, dy, m, w, dx);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

template <class L>
size_t wgrad_bytes(int64_t m) {
    const int64_t ctas = m < WG_CTAS ? m : WG_CTAS;
    return ctas <= 0 ? 16 : (size_t)ctas * L::PSTRIDE * sizeof(float);
}

template <class L>
int wgrad(const float* x, const float* y, const float* dy, int64_t m, float* dw, float* db, float* part, cudaStream_t st) {
    const int smem = (int)sizeof(WgSmem<L>);
    PB_CUDA(cudaFuncSetAttribute(k_trunk_wgrad<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int ctas = (int)(m < WG_CTAS ? m : WG_CTAS);
    k_trunk_wgrad<L><<<ctas, WG_WARPS * 32, smem, st>>>(x, y, dy, m, part);
    PB_LAUNCH_CHECK();
    k_reduce_partials<<<(CO * L::K * 32 + 255) / 256, 256, 0, st>>>(part, ctas, L::PSTRIDE, CO * L::K, dw);
    PB_LAUNCH_CHECK();
    k_reduce_partials<<<(CO * 32 + 255) / 256, 256, 0, st>>>(part + CO * L::K, ctas, L::PSTRIDE, CO, db);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

}  // namespace

extern "C" int pb_nature_conv_forward(int32_t layer, const float* x, int64_t m, const float* w, const float* b, float* y,
                                      void* stream) {
    PB_REQUIRE(layer == 2 || layer == 3, PB_ERR_INVALID, "pb_nature_conv_forward: layer must be 2 or 3, not %d", layer);
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "pb_nature_conv_forward: m must not be negative");
    PB_REQUIRE(aligned16(x) && aligned16(w) && aligned4(b) && aligned16(y), PB_ERR_INVALID,
               "pb_nature_conv_forward: x, w and y must be 16-byte aligned, b 4-byte aligned");
    if (m == 0) return PB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    return layer == 2 ? forward<Conv2>(x, m, w, b, y, st) : forward<Conv3>(x, m, w, b, y, st);
}

extern "C" int pb_nature_conv_dgrad(int32_t layer, const float* y, const float* dy, const float* w, int64_t m, float* dx,
                                    void* stream) {
    PB_REQUIRE(layer == 2 || layer == 3, PB_ERR_INVALID, "pb_nature_conv_dgrad: layer must be 2 or 3, not %d", layer);
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "pb_nature_conv_dgrad: m must not be negative");
    PB_REQUIRE(aligned16(y) && aligned16(dy) && aligned16(w) && aligned16(dx), PB_ERR_INVALID,
               "pb_nature_conv_dgrad: y, dy, w and dx must be 16-byte aligned");
    if (m == 0) return PB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    return layer == 2 ? dgrad<Conv2>(y, dy, w, m, dx, st) : dgrad<Conv3>(y, dy, w, m, dx, st);
}

extern "C" size_t pb_nature_conv_wgrad_workspace_bytes(int32_t layer, int64_t m) {
    return layer == 2 ? wgrad_bytes<Conv2>(m) : layer == 3 ? wgrad_bytes<Conv3>(m) : 0;
}

extern "C" int pb_nature_conv_wgrad(int32_t layer, const float* x, const float* y, const float* dy, int64_t m, float* dw,
                                    float* db, void* workspace, size_t workspace_bytes, void* stream) {
    PB_REQUIRE(layer == 2 || layer == 3, PB_ERR_INVALID, "pb_nature_conv_wgrad: layer must be 2 or 3, not %d", layer);
    PB_REQUIRE(m >= 0, PB_ERR_INVALID, "pb_nature_conv_wgrad: m must not be negative");
    PB_REQUIRE(aligned16(x) && aligned16(y) && aligned16(dy) && aligned4(dw) && aligned4(db) && aligned16(workspace),
               PB_ERR_INVALID, "pb_nature_conv_wgrad: x, y, dy and workspace must be 16-byte aligned, dw and db 4-byte aligned");
    PB_REQUIRE(workspace_bytes >= pb_nature_conv_wgrad_workspace_bytes(layer, m), PB_ERR_INVALID,
               "pb_nature_conv_wgrad: workspace too small");
    if (m == 0) return PB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    float* part = (float*)workspace;
    return layer == 2 ? wgrad<Conv2>(x, y, dy, m, dw, db, part, st) : wgrad<Conv3>(x, y, dy, m, dw, db, part, st);
}
