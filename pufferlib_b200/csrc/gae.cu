// gae.cu -- GAE as a single-pass affine suffix scan with decoupled look-back (sm_90a).
//
// Replaces reference clean_pufferl.py:163-169 (sort_training_data + 3 numpy gathers) and
// reference c_gae.pyx:11-32 (compute_gae).  Recurrence over the sorted batch f = e*H + t, B = N*H:
//     A[B-1] = 0;   A[f] = a_f + b_f * A[f+1]
//     nnt = 1 - d[f+1];  a_f = r[f+1] + (gamma*v[f+1])*nnt - v[f];  b_f = (gamma*lambda)*nnt
// Affine maps compose associatively, (a,b)o(a',b') = (a + b a', b b'), so the chain is a suffix scan.
//
// Data layout: inputs are the arrival-order rollout tensors x[t*N + e] (time-major); the sorted order is never
// materialised.  A tile is a contiguous f-range: E whole envs (E a power of two, all H steps) or, for N == 1 /
// very long horizons, a flat chunk.  PERSISTENT blocks (one wave, no tail) claim tiles by atomic ticket in suffix
// order and double-buffer them: the loader walks a tile with e fastest -- every warp request is runs of E
// consecutive floats of one time row (full 32 B sectors for E >= 8) -- and lands the data transposed in shared
// memory with cp.async (LDGSTS, no register staging; row pitch H|1 is conflict-free for the f-order reads), so the
// loads of tile k+1 are in flight while tile k is scanned.  Each warp scans its 32-element rounds with shuffles,
// (P,Q) partials stay in registers, tiles chain through a 16-byte status word each (aggregate / inclusive) with a
// warp-wide look-back window that stops as soon as the accumulated slope is exactly 0 (any done flag, or
// (gamma*lambda)^k underflow).  Outputs are written in sorted order, 128 B per warp store.
// HBM traffic = 12 B read + 4 (or 8 with returns) B written per agent-step.
#include <stdlib.h>

#include "pb_common.cuh"

namespace {

constexpr int GAE_THREADS = 128;
constexpr int GAE_WARPS = GAE_THREADS / 32;

struct __align__(16) GaeStatus {
    float P, Q, X;
    uint32_t flag;  // 0 = empty, 1 = aggregate (P,Q) valid, 2 = inclusive X valid
};

struct GaeHeader {
    uint32_t ticket, exited, pad0, pad1;
};

struct GaeParams {
    const float* r;
    const float* v;
    const float* d;
    float* adv;
    float* ret;
    float* adv_tm;     // optional: advantages in arrival (time-major) order [H][N] as well (fast path only)
    int64_t N, H, B;
    float gamma, gl;
    int E, logE;       // envs per tile (power of two) or 0 in flat mode
    int L;             // tile length in elements (E*H or flat chunk)
    int pitch;         // shared row pitch (E-mode) ; flat mode: unused
    uint32_t magicH;   // ceil(2^32 / H) for f_local / H (E-mode)
    int numTiles;
    GaeHeader* hdr;
    GaeStatus* status;
};

// A tile's status is ONE aligned 16-byte word {P, Q, X, flag}: it is published with a single 128-bit store and read
// with a single 128-bit load (both L2-coherent, one transaction), so value and flag can never be observed torn and no
// __threadfence is needed around the hand-off (the scheme CUB's decoupled look-back uses for <= 16-byte payloads).
__device__ __forceinline__ void status_store(GaeStatus* s, float P, float Q, float X, uint32_t flag) {
    asm volatile("st.relaxed.gpu.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(s), "r"(__float_as_uint(P)),
                 "r"(__float_as_uint(Q)), "r"(__float_as_uint(X)), "r"(flag)
                 : "memory");
}
__device__ __forceinline__ uint32_t status_load(const GaeStatus* s, float& P, float& Q, float& X) {
    uint32_t a, b, c, f;
    asm volatile("ld.relaxed.gpu.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(f) : "l"(s)
                 : "memory");
    P = __uint_as_float(a); Q = __uint_as_float(b); X = __uint_as_float(c);
    return f;
}

__device__ __forceinline__ void compose(float& a, float& b, float a2, float b2) {
    // (a,b) o (a2,b2): first apply the later map (a2,b2), then this one
    a = fmaf(b, a2, a);
    b = b * b2;
}

__device__ __forceinline__ float tile_lookback(GaeStatus* st, int tile, int numTiles, float tP, float tQ, int lane) {
    if (tile == numTiles - 1) {
        if (lane == 0) status_store(&st[tile], tP, tQ, tP, 2u);   // A beyond the batch is 0: inclusive = aggregate
        return 0.f;
    }
    if (lane == 0) status_store(&st[tile], tP, tQ, 0.f, 1u);
    float accP = 0.f, accQ = 1.f;    // composition of the successor tiles already walked
    int base = tile + 1;
    bool finished = false;
    while (!finished) {
        const int j = base + lane;
        uint32_t fl = 2u;
        float jP = 0.f, jQ = 0.f;    // beyond the last tile: inclusive value 0
        if (j < numTiles) {
            float P, Q, X;
            uint32_t polls = 0;
            do {
                fl = status_load(&st[j], P, Q, X);
                if (++polls == (1u << 27)) __trap();   // seconds of polling: abort rather than hang the GPU
            } while (fl == 0u);
            if (fl == 2u) { jP = X; jQ = 0.f; }
            else { jP = P; jQ = Q; }
        }
        // an inclusive tile or an exactly-zero slope ends the chain: A = P regardless of what follows
        const unsigned stop = __ballot_sync(0xffffffffu, fl == 2u || jQ == 0.f);
        const int last = stop ? (__ffs(stop) - 1) : 31;
        float x = (lane <= last) ? jP : 0.f, y = (lane <= last) ? jQ : 1.f;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const float x2 = __shfl_down_sync(0xffffffffu, x, off);
            const float y2 = __shfl_down_sync(0xffffffffu, y, off);
            if (lane + off < 32) compose(x, y, x2, y2);
        }
        x = __shfl_sync(0xffffffffu, x, 0);
        y = __shfl_sync(0xffffffffu, y, 0);
        compose(accP, accQ, x, y);
        finished = stop != 0u;
        base += 32;
    }
    const float carry = accP;        // accQ == 0 here: value of A at the first element after this tile
    if (lane == 0) status_store(&st[tile], tP, tQ, fmaf(tQ, carry, tP), 2u);
    return carry;
}

__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct TileGeom {
    int64_t f0, e0;
    int Lt, Et;
};

__device__ __forceinline__ TileGeom tile_geom(const GaeParams& p, int tile) {
    TileGeom g;
    if (p.E > 0) {
        g.e0 = (int64_t)tile * p.E;
        g.Et = (int)min((int64_t)p.E, p.N - g.e0);
        g.f0 = g.e0 * p.H;
        g.Lt = g.Et * (int)p.H;
    } else {
        g.e0 = 0; g.Et = 0;
        g.f0 = (int64_t)tile * p.L;
        g.Lt = (int)min((int64_t)p.L, p.B - g.f0);
    }
    return g;
}

// Asynchronously load one tile (transposing) + its halo element into a shared-memory buffer.
__device__ __forceinline__ void load_tile(const GaeParams& p, const TileGeom& g, float* sR, float* sV, float* sD,
                                          float* halo) {
    const int tid = threadIdx.x;
    if (p.E > 0) {
        const int total = p.E * (int)p.H, mask = p.E - 1;
        for (int idx = tid; idx < total; idx += GAE_THREADS) {
            const int el = idx & mask, t = idx >> p.logE;
            if (el < g.Et) {
                const int64_t a = (int64_t)t * p.N + g.e0 + el;
                const int sp = el * p.pitch + t;
                cp_async4(sR + sp, p.r + a);
                cp_async4(sV + sp, p.v + a);
                cp_async4(sD + sp, p.d + a);
            }
        }
    } else if (p.N == 1) {
        for (int idx = tid; idx < g.Lt; idx += GAE_THREADS) {
            cp_async4(sR + idx, p.r + g.f0 + idx);
            cp_async4(sV + idx, p.v + g.f0 + idx);
            cp_async4(sD + idx, p.d + g.f0 + idx);
        }
    } else {  // long-horizon fallback: strided gathers
        for (int idx = tid; idx < g.Lt; idx += GAE_THREADS) {
            const int64_t f = g.f0 + idx, e = f / p.H, t = f - e * p.H;
            const int64_t a = t * p.N + e;
            cp_async4(sR + idx, p.r + a);
            cp_async4(sV + idx, p.v + a);
            cp_async4(sD + idx, p.d + a);
        }
    }
    if (tid == 0) {  // halo: the element after the tile (the chain crosses env and tile boundaries)
        const int64_t fn = g.f0 + g.Lt;
        if (fn < p.B) {
            const int64_t e = fn / p.H, t = fn - e * p.H;
            const int64_t a = t * p.N + e;
            cp_async4(halo + 0, p.r + a);
            cp_async4(halo + 1, p.v + a);
            cp_async4(halo + 2, p.d + a);
        } else {
            halo[0] = 0.f; halo[1] = 0.f; halo[2] = 1.f;
        }
    }
    cp_async_commit();
}

template <int RW>
__global__ void __launch_bounds__(GAE_THREADS) k_gae(GaeParams p) {
    extern __shared__ float smem[];
    __shared__ int s_ticket[2];
    __shared__ float s_halo[2][4];
    __shared__ float s_wP[GAE_WARPS], s_wQ[GAE_WARPS];
    __shared__ float s_carry;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool emode = p.E > 0;
    const int stride_arr = emode ? p.E * p.pitch : p.L;
    const int buf_floats = 3 * stride_arr;
    const int dp = p.pitch - (int)p.H;            // shared index = i + (i / H) * dp   (E-mode)

    // ---- prologue: claim the first tile and start its loads
    if (tid == 0) s_ticket[0] = (int)atomicAdd(&p.hdr->ticket, 1u);
    __syncthreads();
    int ticket = s_ticket[0];
    int cur = 0;
    if (ticket < p.numTiles) {
        const TileGeom g0 = tile_geom(p, p.numTiles - 1 - ticket);   // suffix order: last tile first
        float* b0 = smem;
        load_tile(p, g0, b0, b0 + stride_arr, b0 + 2 * stride_arr, s_halo[0]);
    }

    while (ticket < p.numTiles) {
        const int tile = p.numTiles - 1 - ticket;
        const TileGeom g = tile_geom(p, tile);
        float* sR = smem + cur * buf_floats;
        float* sV = sR + stride_arr;
        float* sD = sR + 2 * stride_arr;
        const float* halo = s_halo[cur];

        // ---- claim the next tile and put its loads in flight behind this tile's
        if (tid == 0) s_ticket[cur ^ 1] = (int)atomicAdd(&p.hdr->ticket, 1u);
        __syncthreads();
        const int next_ticket = s_ticket[cur ^ 1];
        if (next_ticket < p.numTiles) {
            const TileGeom gn = tile_geom(p, p.numTiles - 1 - next_ticket);
            float* bn = smem + (cur ^ 1) * buf_floats;
            load_tile(p, gn, bn, bn + stride_arr, bn + 2 * stride_arr, s_halo[cur ^ 1]);
            cp_async_wait<1>();      // everything but the newest group (the next tile) has landed
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();

        const int64_t f0 = g.f0;
        const int Lt = g.Lt;
        // ---- per-element maps into registers
        const int R = (Lt + 31) >> 5;                    // rounds of 32 in this tile
        const int Rw = (R + GAE_WARPS - 1) / GAE_WARPS;  // rounds per warp (<= RW)
        const int r_begin = warp * Rw;
        float a[RW], b[RW];
#pragma unroll
        for (int k = 0; k < RW; ++k) {
            const int i = ((r_begin + k) << 5) + lane;
            a[k] = 0.f;
            b[k] = 1.f;  // identity for padding lanes
            if (k < Rw && i < Lt) {
                int sp0 = i, sp1 = i + 1;
                if (emode) {
                    sp0 = i + (int)__umulhi((uint32_t)i, p.magicH) * dp;
                    sp1 = i + 1 + (int)__umulhi((uint32_t)(i + 1), p.magicH) * dp;
                }
                float r1, v1, d1;
                if (i + 1 < Lt) {
                    r1 = sR[sp1]; v1 = sV[sp1]; d1 = sD[sp1];
                } else {
                    r1 = halo[0]; v1 = halo[1]; d1 = halo[2];
                }
                const float v0 = sV[sp0];
                const float nnt = __fsub_rn(1.0f, d1);
                // c_gae.pyx:28-29 association, no FMA contraction inside an element
                a[k] = __fsub_rn(__fadd_rn(r1, __fmul_rn(__fmul_rn(p.gamma, v1), nnt)), v0);
                b[k] = __fmul_rn(p.gl, nnt);
                if (f0 + i == p.B - 1) {  // A[B-1] = 0
                    a[k] = 0.f;
                    b[k] = 0.f;
                }
            }
        }

        // ---- warp-level suffix scan, rounds from last to first; (a,b) become tile-local partials (P,Q) w.r.t.
        //      the value entering this warp's range from the right
        float cP = 0.f, cQ = 1.f;
#pragma unroll
        for (int k = RW - 1; k >= 0; --k) {
            if (k < Rw) {
                float x = a[k], y = b[k];
#pragma unroll
                for (int off = 1; off < 32; off <<= 1) {
                    const float x2 = __shfl_down_sync(0xffffffffu, x, off);
                    const float y2 = __shfl_down_sync(0xffffffffu, y, off);
                    if (lane + off < 32) compose(x, y, x2, y2);
                }
                compose(x, y, cP, cQ);
                a[k] = x;
                b[k] = y;
                cP = __shfl_sync(0xffffffffu, x, 0);
                cQ = __shfl_sync(0xffffffffu, y, 0);
            }
        }
        if (lane == 0) {
            s_wP[warp] = cP;
            s_wQ[warp] = cQ;
        }
        __syncthreads();

        // ---- tile aggregate + decoupled look-back (warp 0)
        if (warp == 0) {
            float tP = 0.f, tQ = 1.f;  // composition of all warps, in order 0..W-1
#pragma unroll
            for (int w = GAE_WARPS - 1; w >= 0; --w) {
                float x = s_wP[w], y = s_wQ[w];
                compose(x, y, tP, tQ);
                tP = x;
                tQ = y;
            }
            const float carry = tile_lookback(p.status, tile, p.numTiles, tP, tQ, lane);
            if (lane == 0) s_carry = carry;
        }
        __syncthreads();

        // ---- carry entering this warp's range = later warps' aggregates applied to the tile carry
        float cin = s_carry;
        for (int w = GAE_WARPS - 1; w > warp; --w) cin = fmaf(s_wQ[w], cin, s_wP[w]);

        // ---- outputs in sorted order (coalesced 128 B per warp store)
#pragma unroll
        for (int k = 0; k < RW; ++k) {
            const int i = ((r_begin + k) << 5) + lane;
            if (k < Rw && i < Lt) {
                const float A = fmaf(b[k], cin, a[k]);
                __stcs(p.adv + f0 + i, A);
                if (p.ret) {
                    const int sp0 = emode ? i + (int)__umulhi((uint32_t)i, p.magicH) * dp : i;
                    __stcs(p.ret + f0 + i, A + sV[sp0]);
                }
            }
        }
        __syncthreads();   // this buffer (and s_wP/s_wQ/s_carry) may be refilled from here on
        ticket = next_ticket;
        cur ^= 1;
    }

    // ---- self-cleaning workspace: the last block to leave zeroes the header and every status word
    if (tid == 0) {
        __threadfence();
        const uint32_t prev = atomicAdd(&p.hdr->exited, 1u);
        s_ticket[0] = (prev == gridDim.x - 1u) ? 1 : 0;
    }
    __syncthreads();
    if (s_ticket[0]) {
        for (int j = tid; j < p.numTiles; j += GAE_THREADS) {
            p.status[j].P = 0.f; p.status[j].Q = 0.f; p.status[j].X = 0.f; p.status[j].flag = 0u;
        }
        if (tid == 0) { p.hdr->ticket = 0u; p.hdr->exited = 0u; }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Fast path (N > 1, N % 4 == 0, H in {128, 256, 512}): tile = 32 whole envs, 256 threads.
//   * loads: every time row of the tile is one 128-byte run (32 envs), copied global->shared with 16-byte cp.async
//     (LDGSTS.128): 12*KC async copies per thread, no register staging, no transposition -- shared layout is [t][32];
//   * pass 1: thread (env = lane, chunk) composes its 16 consecutive steps SERIALLY in registers (2 FMAs per element
//     instead of a 5-step shuffle scan); a warp's 32 lanes read 32 consecutive floats: conflict-free;
//   * pass 2 (one warp): chunk carries inside each env, a 5-step shuffle suffix over the 32 env aggregates, then the
//     decoupled look-back; pass 3: apply carries, 64 B of output per thread-chunk.
// ~40 thread-instructions per element instead of ~180 for the generic kernel.
constexpr int FE = 32;            // envs per tile
constexpr int FC = 16;            // steps per chunk
constexpr int FAST_THREADS = 256; // 32 envs x 8 chunk slots

__device__ __forceinline__ void cp_async16(float* dst_smem, const float* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src)
                 : "memory");
}

template <int KC>   // chunks per thread: H = 128 * KC
__global__ void __launch_bounds__(FAST_THREADS) k_gae_fast(GaeParams p) {
    constexpr int H = 128 * KC;
    constexpr int CE = H / FC;                 // chunks per env
    constexpr int ARR = H * FE;                // floats per array
    extern __shared__ __align__(16) float smem[];   // {r, v, d} x [H][32]
    __shared__ int s_ticket[2];
    __shared__ float s_halo[4];
    __shared__ float2 s_cagg[CE][FE];          // chunk aggregates, then chunk carry maps (w.r.t. the env's right end)
    __shared__ float2 s_eagg[FE];              // env carry maps w.r.t. the tile's right end
    __shared__ float s_carry;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float* sR = smem;
    float* sV = smem + ARR;
    float* sD = smem + 2 * ARR;

    if (tid == 0) s_ticket[0] = (int)atomicAdd(&p.hdr->ticket, 1u);
    __syncthreads();
    int ticket = s_ticket[0];

    while (ticket < p.numTiles) {
        const int tile = p.numTiles - 1 - ticket;          // suffix order: last tile first
        const int64_t e0 = (int64_t)tile * FE;
        const int Et = (int)min((int64_t)FE, p.N - e0);     // multiple of 4 (N % 4 == 0)

        // ---- async loads: row t of the tile = floats [t*N + e0, +Et)
        {
            const int quad = tid & 7, t0 = tid >> 3;         // 8 float4 per row, 32 rows per sweep
            if (4 * quad < Et) {
                const int64_t g0 = (int64_t)t0 * p.N + e0 + 4 * quad;
                const int64_t gstep = 32 * p.N;
                const float* pr = p.r + g0;
                const float* pv = p.v + g0;
                const float* pd = p.d + g0;
                int sp = t0 * FE + 4 * quad;
#pragma unroll
                for (int k = 0; k < H / 32; ++k) {
                    cp_async16(sR + sp, pr);
                    cp_async16(sV + sp, pv);
                    cp_async16(sD + sp, pd);
                    pr += gstep; pv += gstep; pd += gstep;
                    sp += 32 * FE;
                }
            }
            if (tid == 0) {
                const int64_t en = e0 + Et;                  // first env after the tile; its t = 0 row entry
                if (en < p.N) {
                    cp_async4(&s_halo[0], p.r + en);
                    cp_async4(&s_halo[1], p.v + en);
                    cp_async4(&s_halo[2], p.d + en);
                } else {
                    s_halo[0] = 0.f; s_halo[1] = 0.f; s_halo[2] = 1.f;
                }
                // claim the next tile now; the value is only read at the end of this iteration (latency hidden)
                s_ticket[1] = (int)atomicAdd(&p.hdr->ticket, 1u);
            }
            cp_async_commit();
            cp_async_wait<0>();
        }
        __syncthreads();

        // ---- pass 1: per-chunk serial composition (suffix order), element maps kept in registers
        float a[KC][FC], b[KC][FC];
#pragma unroll
        for (int kc = 0; kc < KC; ++kc) {
            const int c = warp + kc * (FAST_THREADS / 32);      // chunk index; env = lane
            float P = 0.f, Q = 1.f;
            if (lane < Et) {
                const int base = c * FC * FE + lane;
                // the element after the chunk: next step of the env, next env's first step, or the tile halo
                float rn, vn, dn;
                if (c < CE - 1) { rn = sR[base + FC * FE]; vn = sV[base + FC * FE]; dn = sD[base + FC * FE]; }
                else if (lane + 1 < Et) { rn = sR[lane + 1]; vn = sV[lane + 1]; dn = sD[lane + 1]; }
                else { rn = s_halo[0]; vn = s_halo[1]; dn = s_halo[2]; }
                const bool last_of_batch = (e0 + lane == p.N - 1) && (c == CE - 1);
#pragma unroll
                for (int j = FC - 1; j >= 0; --j) {
                    const float r0 = sR[base + j * FE], v0 = sV[base + j * FE], d0 = sD[base + j * FE];
                    const float nnt = __fsub_rn(1.0f, dn);
                    // c_gae.pyx:28-29 association, no FMA contraction inside an element
                    float aj = __fsub_rn(__fadd_rn(rn, __fmul_rn(__fmul_rn(p.gamma, vn), nnt)), v0);
                    float bj = __fmul_rn(p.gl, nnt);
                    if (last_of_batch && j == FC - 1) { aj = 0.f; bj = 0.f; }   // A[B-1] = 0
                    a[kc][j] = aj;
                    b[kc][j] = bj;
                    P = fmaf(bj, P, aj);     // (aj,bj) o (P,Q)
                    Q = bj * Q;
                    rn = r0; vn = v0; dn = d0;
                }
            } else {
#pragma unroll
                for (int j = 0; j < FC; ++j) { a[kc][j] = 0.f; b[kc][j] = 1.f; }
            }
            s_cagg[c][lane] = make_float2(P, Q);
        }
        __syncthreads();

        // ---- pass 2 (warp 0): chunk carries inside each env, env carries inside the tile, then the look-back
        if (warp == 0) {
            float cP = 0.f, cQ = 1.f;                    // composition of the chunks to the right, w.r.t. the env end
#pragma unroll
            for (int c = CE - 1; c >= 0; --c) {
                const float2 g = s_cagg[c][lane];
                s_cagg[c][lane] = make_float2(cP, cQ);   // carry map entering chunk c from the right
                const float nP = fmaf(g.y, cP, g.x), nQ = g.y * cQ;
                cP = nP; cQ = nQ;
            }
            // inclusive suffix over the 32 env aggregates (missing envs are the identity)
            float x = cP, y = cQ;
#pragma unroll
            for (int off = 1; off < FE; off <<= 1) {
                const float x2 = __shfl_down_sync(0xffffffffu, x, off);
                const float y2 = __shfl_down_sync(0xffffffffu, y, off);
                if (lane + off < FE) compose(x, y, x2, y2);
            }
            const float tP = __shfl_sync(0xffffffffu, x, 0), tQ = __shfl_sync(0xffffffffu, y, 0);
            // exclusive: map from the tile's right end to env `lane`'s right end
            float exP = __shfl_down_sync(0xffffffffu, x, 1), exQ = __shfl_down_sync(0xffffffffu, y, 1);
            if (lane == FE - 1) { exP = 0.f; exQ = 1.f; }
            s_eagg[lane] = make_float2(exP, exQ);
            const float carry = tile_lookback(p.status, tile, p.numTiles, tP, tQ, lane);
            if (lane == 0) s_carry = carry;
        }
        __syncthreads();

        // ---- pass 3: apply carries, write outputs in sorted order (64 B per thread-chunk, full sectors)
        const float C = s_carry;
        if (lane < Et) {
            const float2 em = s_eagg[lane];
            const float a_env_end = fmaf(em.y, C, em.x);                // A just after this env
#pragma unroll
            for (int kc = 0; kc < KC; ++kc) {
                const int c = warp + kc * (FAST_THREADS / 32);
                const float2 cm = s_cagg[c][lane];
                float A = fmaf(cm.y, a_env_end, cm.x);                  // A just after this chunk
                const int64_t f = (e0 + lane) * (int64_t)H + c * FC;
                float outA[FC];
#pragma unroll
                for (int j = FC - 1; j >= 0; --j) {
                    A = fmaf(b[kc][j], A, a[kc][j]);
                    outA[j] = A;
                }
                if (p.adv) {
                    float4* pa = reinterpret_cast<float4*>(p.adv + f);
#pragma unroll
                    for (int j4 = 0; j4 < FC / 4; ++j4)
                        __stcs(pa + j4, make_float4(outA[4 * j4], outA[4 * j4 + 1], outA[4 * j4 + 2], outA[4 * j4 + 3]));
                }
                if (p.adv_tm) {   // stage in the (now idle) reward tile, same [t][32] layout: conflict-free, lanes = envs
#pragma unroll
                    for (int j = 0; j < FC; ++j) sR[(c * FC + j) * FE + lane] = outA[j];
                }
                if (p.ret) {
                    const int base = c * FC * FE + lane;
                    float4* pr = reinterpret_cast<float4*>(p.ret + f);
#pragma unroll
                    for (int j4 = 0; j4 < FC / 4; ++j4)
                        __stcs(pr + j4, make_float4(outA[4 * j4] + sV[base + (4 * j4) * FE],
                                                    outA[4 * j4 + 1] + sV[base + (4 * j4 + 1) * FE],
                                                    outA[4 * j4 + 2] + sV[base + (4 * j4 + 2) * FE],
                                                    outA[4 * j4 + 3] + sV[base + (4 * j4 + 3) * FE]));
                }
            }
        }
        if (p.adv_tm) {   // arrival-order rows: one fully coalesced 128-byte store per time step of the tile
            __syncthreads();
            if (lane < Et) {
                float* dst = p.adv_tm + e0 + lane;
#pragma unroll 4
                for (int t = warp; t < H; t += FAST_THREADS / 32) __stcs(dst + (int64_t)t * p.N, sR[t * FE + lane]);
            }
        }
        __syncthreads();          // the tile buffers, s_cagg / s_eagg / s_carry are free again
        ticket = s_ticket[1];
        __syncthreads();          // everyone has read s_ticket[1] before thread 0 overwrites it next iteration
    }

    if (tid == 0) {
        __threadfence();
        const uint32_t prev = atomicAdd(&p.hdr->exited, 1u);
        s_ticket[0] = (prev == gridDim.x - 1u) ? 1 : 0;
    }
    __syncthreads();
    if (s_ticket[0]) {
        for (int j = tid; j < p.numTiles; j += FAST_THREADS) {
            p.status[j].P = 0.f; p.status[j].Q = 0.f; p.status[j].X = 0.f; p.status[j].flag = 0u;
        }
        if (tid == 0) { p.hdr->ticket = 0u; p.hdr->exited = 0u; }
    }
}


// ---------------------------------------------------------------------------------------------------------------
// Tile kernel v2 (same shapes as k_gae_fast: N % 4 == 0, H in {128, 256, 512}; same arithmetic, bit-identical results).
// What changes is how the bytes move:
//   * DOUBLE-BUFFERED tiles: the cp.async loads of the next tile (claimed by ticket at the top of the iteration) are in
//     flight while this tile is scanned and written out, so DRAM does not idle during the scan (NBUF = 2 where 2 tiles
//     fit in shared memory: 96 KB at H = 128 -> 2 CTAs / SM, 192 KB at H = 256 -> 1 CTA / SM);
//   * COALESCED OUTPUTS: pass 3 stages its results in the tile arrays that are dead after pass 1 -- sorted order
//     ([env][t], 16-byte chunks XOR-swizzled by env & 7: conflict-free for the lane = env writes and for the row reads)
//     or arrival order ([t][32]) -- and the block then writes whole 512-byte env rows / 128-byte time rows, instead of
//     32 scattered 16-byte pieces per store instruction;
//   * one warp per 16-step chunk of all 32 envs (THREADS = 32 * min(H / 16, 16)): H = 256 runs 16 warps.
template <int KC, int NBUF, int THREADS>
__global__ void __launch_bounds__(THREADS) k_gae_tile(GaeParams p) {
    constexpr int NW = THREADS / 32;
    constexpr int H = FC * NW * KC;
    constexpr int CE = H / FC;                 // chunks per env
    constexpr int ARR = H * FE;                // floats per array
    extern __shared__ __align__(16) float smem[];   // NBUF x {r, v, d} x [H][32]
    __shared__ int s_ticket[2];
    __shared__ float s_halo[2][4];
    __shared__ float2 s_cagg[CE][FE];
    __shared__ float2 s_eagg[FE];
    __shared__ float s_carry;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    auto issue_loads = [&](int tile, int b) {
        float* sR = smem + (size_t)b * 3 * ARR;
        float* sV = sR + ARR;
        float* sD = sR + 2 * ARR;
        const int64_t e0 = (int64_t)tile * FE;
        const int Et = (int)min((int64_t)FE, p.N - e0);
        const int quad = tid & 7, t0 = tid >> 3;         // 8 float4 per row, THREADS / 8 rows per sweep
        if (4 * quad < Et) {
            const int64_t g0 = (int64_t)t0 * p.N + e0 + 4 * quad;
            const int64_t gstep = (int64_t)(THREADS / 8) * p.N;
            const float* pr = p.r + g0;
            const float* pv = p.v + g0;
            const float* pd = p.d + g0;
            int sp = t0 * FE + 4 * quad;
#pragma unroll
            for (int k = 0; k < H / (THREADS / 8); ++k) {
                cp_async16(sR + sp, pr);
                cp_async16(sV + sp, pv);
                cp_async16(sD + sp, pd);
                pr += gstep; pv += gstep; pd += gstep;
                sp += (THREADS / 8) * FE;
            }
        }
        if (tid == 0) {
            const int64_t en = e0 + Et;                  // first env after the tile; its t = 0 row entry
            if (en < p.N) {
                cp_async4(&s_halo[b][0], p.r + en);
                cp_async4(&s_halo[b][1], p.v + en);
                cp_async4(&s_halo[b][2], p.d + en);
            } else {
                s_halo[b][0] = 0.f; s_halo[b][1] = 0.f; s_halo[b][2] = 1.f;
            }
        }
        cp_async_commit();
    };

    if (tid == 0) s_ticket[0] = (int)atomicAdd(&p.hdr->ticket, 1u);
    __syncthreads();
    int ticket = s_ticket[0];
    int cur = 0;
    if (ticket < p.numTiles) issue_loads(p.numTiles - 1 - ticket, 0);

    while (ticket < p.numTiles) {
        const int tile = p.numTiles - 1 - ticket;          // suffix order: last tile first
        const int64_t e0 = (int64_t)tile * FE;
        const int Et = (int)min((int64_t)FE, p.N - e0);     // multiple of 4 (N % 4 == 0)
        float* sR = smem + (size_t)cur * 3 * ARR;
        float* sV = sR + ARR;
        float* sD = sR + 2 * ARR;
        const float* halo = s_halo[cur];

        // ---- claim the next tile and (NBUF == 2) start its loads before touching this one
        if (tid == 0) s_ticket[1] = (int)atomicAdd(&p.hdr->ticket, 1u);
        __syncthreads();
        const int next_ticket = s_ticket[1];
        const bool prefetch = NBUF == 2 && next_ticket < p.numTiles;
        if (prefetch) {
            issue_loads(p.numTiles - 1 - next_ticket, cur ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();

        // ---- pass 1: per-chunk serial composition (suffix order), element maps kept in registers
        float a[KC][FC], b[KC][FC];
#pragma unroll
        for (int kc = 0; kc < KC; ++kc) {
            const int c = warp + kc * NW;                       // chunk index; env = lane
            float P = 0.f, Q = 1.f;
            if (lane < Et) {
                const int base = c * FC * FE + lane;
                float rn, vn, dn;
                if (c < CE - 1) { rn = sR[base + FC * FE]; vn = sV[base + FC * FE]; dn = sD[base + FC * FE]; }
                else if (lane + 1 < Et) { rn = sR[lane + 1]; vn = sV[lane + 1]; dn = sD[lane + 1]; }
                else { rn = halo[0]; vn = halo[1]; dn = halo[2]; }
                const bool last_of_batch = (e0 + lane == p.N - 1) && (c == CE - 1);
#pragma unroll
                for (int j = FC - 1; j >= 0; --j) {
                    const float r0 = sR[base + j * FE], v0 = sV[base + j * FE], d0 = sD[base + j * FE];
                    const float nnt = __fsub_rn(1.0f, dn);
                    float aj = __fsub_rn(__fadd_rn(rn, __fmul_rn(__fmul_rn(p.gamma, vn), nnt)), v0);
                    float bj = __fmul_rn(p.gl, nnt);
                    if (last_of_batch && j == FC - 1) { aj = 0.f; bj = 0.f; }   // A[B-1] = 0
                    a[kc][j] = aj;
                    b[kc][j] = bj;
                    P = fmaf(bj, P, aj);
                    Q = bj * Q;
                    rn = r0; vn = v0; dn = d0;
                }
            } else {
#pragma unroll
                for (int j = 0; j < FC; ++j) { a[kc][j] = 0.f; b[kc][j] = 1.f; }
            }
            s_cagg[c][lane] = make_float2(P, Q);
        }
        __syncthreads();

        // ---- pass 2 (warp 0): chunk carries inside each env, env carries inside the tile, then the look-back
        if (warp == 0) {
            float cP = 0.f, cQ = 1.f;
#pragma unroll
            for (int c = CE - 1; c >= 0; --c) {
                const float2 g = s_cagg[c][lane];
                s_cagg[c][lane] = make_float2(cP, cQ);
                const float nP = fmaf(g.y, cP, g.x), nQ = g.y * cQ;
                cP = nP; cQ = nQ;
            }
            float x = cP, y = cQ;
#pragma unroll
            for (int off = 1; off < FE; off <<= 1) {
                const float x2 = __shfl_down_sync(0xffffffffu, x, off);
                const float y2 = __shfl_down_sync(0xffffffffu, y, off);
                if (lane + off < FE) compose(x, y, x2, y2);
            }
            const float tP = __shfl_sync(0xffffffffu, x, 0), tQ = __shfl_sync(0xffffffffu, y, 0);
            float exP = __shfl_down_sync(0xffffffffu, x, 1), exQ = __shfl_down_sync(0xffffffffu, y, 1);
            if (lane == FE - 1) { exP = 0.f; exQ = 1.f; }
            s_eagg[lane] = make_float2(exP, exQ);
            const float carry = tile_lookback(p.status, tile, p.numTiles, tP, tQ, lane);
            if (lane == 0) s_carry = carry;
        }
        __syncthreads();

        // ---- pass 3: apply carries; results staged in the dead tile arrays:
        //      sR <- advantages, sorted layout [env][t] (16-byte chunk q of env row at position q ^ (env & 7))
        //      sD <- returns in the same layout, or (time-major output) advantages as [t][32]
        const float C = s_carry;
        if (lane < Et) {
            const float2 em = s_eagg[lane];
            const float a_env_end = fmaf(em.y, C, em.x);
#pragma unroll
            for (int kc = 0; kc < KC; ++kc) {
                const int c = warp + kc * NW;
                const float2 cm = s_cagg[c][lane];
                float A = fmaf(cm.y, a_env_end, cm.x);
                float outA[FC];
#pragma unroll
                for (int j = FC - 1; j >= 0; --j) {
                    A = fmaf(b[kc][j], A, a[kc][j]);
                    outA[j] = A;
                }
                const int base = c * FC * FE + lane;
                float vv[FC];
                if (p.ret) {
#pragma unroll
                    for (int j = 0; j < FC; ++j) vv[j] = sV[base + j * FE];
                }
                if (p.adv) {
#pragma unroll
                    for (int j4 = 0; j4 < FC / 4; ++j4) {
                        const int q = c * (FC / 4) + j4;
                        *reinterpret_cast<float4*>(sR + lane * H + ((q ^ (lane & 7)) << 2)) =
                            make_float4(outA[4 * j4], outA[4 * j4 + 1], outA[4 * j4 + 2], outA[4 * j4 + 3]);
                    }
                }
                if (p.ret) {
#pragma unroll
                    for (int j4 = 0; j4 < FC / 4; ++j4) {
                        const int q = c * (FC / 4) + j4;
                        *reinterpret_cast<float4*>(sD + lane * H + ((q ^ (lane & 7)) << 2)) =
                            make_float4(outA[4 * j4] + vv[4 * j4], outA[4 * j4 + 1] + vv[4 * j4 + 1],
                                        outA[4 * j4 + 2] + vv[4 * j4 + 2], outA[4 * j4 + 3] + vv[4 * j4 + 3]);
                    }
                } else if (p.adv_tm) {
#pragma unroll
                    for (int j = 0; j < FC; ++j) sD[(c * FC + j) * FE + lane] = outA[j];
                }
            }
        }
        __syncthreads();
        // NOTE: pass 1 of this tile has finished for every warp (barriers above), so overwriting sR / sD was safe; sV
        // is only read.  Now the coalesced stores: one warp per env row (sorted) / per time row (arrival order).
        {
            const int64_t f0 = e0 * (int64_t)H;
            for (int env = warp; env < Et; env += NW) {
#pragma unroll
                for (int q0 = 0; q0 < H / 4; q0 += 32) {
                    const int q = q0 + lane;
                    const int sp = env * H + ((q ^ (env & 7)) << 2);
                    if (p.adv) __stcs(reinterpret_cast<float4*>(p.adv + f0 + (int64_t)env * H) + q, *reinterpret_cast<const float4*>(sR + sp));
                    if (p.ret) __stcs(reinterpret_cast<float4*>(p.ret + f0 + (int64_t)env * H) + q, *reinterpret_cast<const float4*>(sD + sp));
                }
            }
            if (p.adv_tm && !p.ret && lane < Et) {
                float* dst = p.adv_tm + e0 + lane;
#pragma unroll 4
                for (int t = warp; t < H; t += NW) __stcs(dst + (int64_t)t * p.N, sD[t * FE + lane]);
            }
        }
        __syncthreads();          // this buffer, s_cagg / s_eagg / s_carry are free again
        ticket = next_ticket;
        if (NBUF == 2) cur ^= 1;
        else if (ticket < p.numTiles) issue_loads(p.numTiles - 1 - ticket, 0);
    }

    if (tid == 0) {
        __threadfence();
        const uint32_t prev = atomicAdd(&p.hdr->exited, 1u);
        s_ticket[0] = (prev == gridDim.x - 1u) ? 1 : 0;
    }
    __syncthreads();
    if (s_ticket[0]) {
        for (int j = tid; j < p.numTiles; j += THREADS) {
            p.status[j].P = 0.f; p.status[j].Q = 0.f; p.status[j].X = 0.f; p.status[j].flag = 0u;
        }
        if (tid == 0) { p.hdr->ticket = 0u; p.hdr->exited = 0u; }
    }
}

// 0: by horizon -- 2 at H <= 128, 3 above (H100 80GB HBM3 at 700 W, bench.py: C2 H = 128 23.7 us double- vs 25.0 us
// single-buffered; C3 H = 256 162 us single- vs 177 us double-buffered); 2 / 3: k_gae_tile double- / single-buffered;
// 1: k_gae_fast
int g_gae_variant = 0;

struct GaePlan {
    int fastKC;   // > 0: k_gae_fast<fastKC, nbuf>
    int nbuf;
    int E, logE, L, pitch, numTiles, RW;
    uint32_t magicH;
    size_t smem;
};

GaePlan gae_plan(int64_t N, int64_t H) {
    GaePlan g{};
    const int64_t B = N * H;
    const int Ltarget = 2048, Lmax = 4096;
    if (N > 1 && N % 4 == 0 && (H == 128 || H == 256 || H == 512)) {
        g.fastKC = (int)(H / 128);
        g.nbuf = 1;
        g.E = FE; g.logE = 5; g.L = FE * (int)H; g.pitch = FE; g.magicH = 0;
        g.numTiles = (int)pb_ceil_div(N, FE);
        g.smem = (size_t)3 * FE * H * sizeof(float);
        g.RW = 16;
        return g;
    }
    if (N > 1 && H * 8 <= Lmax) {
        int E = 8;
        while ((int64_t)E * 2 * H <= Ltarget) E *= 2;   // largest power of two with E*H <= Ltarget, at least 8
        while (E > 8 && E / 2 >= N) E /= 2;             // do not over-allocate for tiny N
        g.E = E;
        g.logE = 0;
        while ((1 << g.logE) < E) ++g.logE;
        g.L = E * (int)H;
        g.pitch = (int)(H | 1);
        g.magicH = (uint32_t)(((1ull << 32) + (uint64_t)H - 1) / (uint64_t)H);
        g.numTiles = (int)pb_ceil_div(N, E);
        g.smem = (size_t)2 * 3 * E * g.pitch * sizeof(float);   // double-buffered
    } else {
        g.E = 0;
        g.L = (int)(B < Ltarget ? (B > 0 ? B : 1) : Ltarget);
        g.pitch = 0;
        g.magicH = 0;
        g.numTiles = (int)pb_ceil_div(B, g.L);
        g.smem = (size_t)2 * 3 * g.L * sizeof(float);
    }
    const int R = (g.L + 31) / 32;
    const int Rw = (R + GAE_WARPS - 1) / GAE_WARPS;
    g.RW = Rw <= 16 ? 16 : 32;
    return g;
}

}  // namespace

extern "C" size_t pb_gae_workspace_bytes(int64_t num_envs, int64_t horizon) {
    if (num_envs <= 0 || horizon <= 0) return sizeof(GaeHeader);
    GaePlan g = gae_plan(num_envs, horizon);
    return sizeof(GaeHeader) + (size_t)g.numTiles * sizeof(GaeStatus);
}

extern "C" int pb_gae(const float* rewards, const float* values, const float* dones, float* advantages,
                      float* returns_sorted, int64_t num_envs, int64_t horizon, float gamma, float gae_lambda,
                      void* workspace, size_t workspace_bytes, void* stream) {
    PB_REQUIRE(advantages || num_envs == 0 || horizon == 0, PB_ERR_INVALID, "pb_gae: null pointer");
    return pb_gae_tm(rewards, values, dones, advantages, returns_sorted, nullptr, num_envs, horizon, gamma, gae_lambda,
                     workspace, workspace_bytes, stream);
}

extern "C" int pb_gae_time_major_supported(int64_t num_envs, int64_t horizon) {
    return (num_envs > 0 && horizon > 0 && gae_plan(num_envs, horizon).fastKC > 0) ? 1 : 0;
}

extern "C" int pb_gae_tm(const float* rewards, const float* values, const float* dones, float* advantages,
                         float* returns_sorted, float* advantages_time_major, int64_t num_envs, int64_t horizon,
                         float gamma, float gae_lambda, void* workspace, size_t workspace_bytes, void* stream) {
    PB_REQUIRE(num_envs >= 0 && horizon >= 0, PB_ERR_INVALID, "pb_gae: negative size");
    if (num_envs == 0 || horizon == 0) return PB_OK;
    PB_REQUIRE(rewards && values && dones && (advantages || advantages_time_major), PB_ERR_INVALID, "pb_gae: null pointer");
    PB_REQUIRE(!advantages_time_major || gae_plan(num_envs, horizon).fastKC > 0, PB_ERR_UNSUPPORTED,
               "pb_gae_tm: the time-major output needs the tile kernel (horizon in {128, 256, 512}, num_envs %% 4 == 0)");
    PB_REQUIRE(advantages || gae_plan(num_envs, horizon).fastKC > 0, PB_ERR_INVALID, "pb_gae: null advantages");
    PB_REQUIRE(num_envs * horizon < (1ll << 40), PB_ERR_INVALID, "pb_gae: batch too large");
    GaePlan g = gae_plan(num_envs, horizon);
    const size_t need = sizeof(GaeHeader) + (size_t)g.numTiles * sizeof(GaeStatus);
    PB_REQUIRE(workspace && workspace_bytes >= need, PB_ERR_INVALID,
               "pb_gae: workspace too small (%zu < %zu)", workspace_bytes, need);
    GaeParams p{};
    p.r = rewards; p.v = values; p.d = dones; p.adv = advantages; p.ret = returns_sorted; p.adv_tm = advantages_time_major;
    p.N = num_envs; p.H = horizon; p.B = num_envs * horizon;
    p.gamma = gamma;
    p.gl = gamma * gae_lambda;  // float product, as `gamma * gae_lambda` in c_gae.pyx:29
    p.E = g.E; p.logE = g.logE; p.L = g.L; p.pitch = g.pitch; p.magicH = g.magicH; p.numTiles = g.numTiles;
    p.hdr = (GaeHeader*)workspace;
    p.status = (GaeStatus*)((char*)workspace + sizeof(GaeHeader));
    cudaStream_t s = (cudaStream_t)stream;
    // persistent grid: every resident slot of the chip, never more blocks than tiles (one wave, no tail)
    int per_sm = 0;
    if (g.fastKC > 0) {
        PB_REQUIRE((!advantages || ((uintptr_t)advantages & 15) == 0) && (!returns_sorted || ((uintptr_t)returns_sorted & 15) == 0),
                   PB_ERR_INVALID, "pb_gae: advantages / returns must be 16-byte aligned");
        PB_REQUIRE(((uintptr_t)rewards & 15) == 0 && ((uintptr_t)values & 15) == 0 && ((uintptr_t)dones & 15) == 0,
                   PB_ERR_INVALID, "pb_gae: rewards / values / dones must be 16-byte aligned");
#define PB_GAE_FAST(KC)                                                                                               \
    {                                                                                                                 \
        PB_CUDA(cudaFuncSetAttribute(k_gae_fast<KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));     \
        PB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gae_fast<KC>, FAST_THREADS, g.smem));       \
        PB_REQUIRE(per_sm >= 1, PB_ERR_CUDA, "pb_gae: kernel does not fit on an SM (smem %zu)", g.smem);              \
        int grid = per_sm * PB_NUM_SMS;                                                                               \
        if (grid > g.numTiles) grid = g.numTiles;                                                                     \
        k_gae_fast<KC><<<grid, FAST_THREADS, g.smem, s>>>(p);                                                         \
    }
#define PB_GAE_TILE(KC, NBUF, THREADS)                                                                                \
    {                                                                                                                 \
        const size_t smem2 = (size_t)NBUF * g.smem;                                                                   \
        PB_CUDA(cudaFuncSetAttribute(k_gae_tile<KC, NBUF, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize,      \
                                     (int)smem2));                                                                    \
        PB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gae_tile<KC, NBUF, THREADS>, THREADS, smem2)); \
        PB_REQUIRE(per_sm >= 1, PB_ERR_CUDA, "pb_gae: kernel does not fit on an SM (smem %zu)", smem2);               \
        int grid = per_sm * PB_NUM_SMS;                                                                               \
        if (grid > g.numTiles) grid = g.numTiles;                                                                     \
        k_gae_tile<KC, NBUF, THREADS><<<grid, THREADS, smem2, s>>>(p);                                                \
    }
        const bool v2_ok = !(returns_sorted && advantages_time_major);   // v2 stages two outputs: adv + (ret | adv_tm)
        const int variant = g_gae_variant ? g_gae_variant : (g.fastKC == 1 ? 2 : 3);   // double-buffered tiles for H = 128, single-buffered above
        if (variant == 2 && v2_ok) {
            if (g.fastKC == 1) PB_GAE_TILE(1, 2, 256) else if (g.fastKC == 2) PB_GAE_TILE(1, 2, 512) else PB_GAE_TILE(2, 1, 512)
        } else if (variant == 3 && v2_ok) {   // single-buffered tiles (more CTAs per SM), coalesced outputs
            if (g.fastKC == 1) PB_GAE_TILE(1, 1, 256) else if (g.fastKC == 2) PB_GAE_TILE(2, 1, 256) else PB_GAE_TILE(2, 1, 512)
        } else {
            if (g.fastKC == 1) PB_GAE_FAST(1) else if (g.fastKC == 2) PB_GAE_FAST(2) else PB_GAE_FAST(4)
        }
#undef PB_GAE_TILE
#undef PB_GAE_FAST
        PB_LAUNCH_CHECK();
        return PB_OK;
    }
    if (g.RW == 16) {
        PB_CUDA(cudaFuncSetAttribute(k_gae<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));
        PB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gae<16>, GAE_THREADS, g.smem));
    } else {
        PB_CUDA(cudaFuncSetAttribute(k_gae<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));
        PB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_gae<32>, GAE_THREADS, g.smem));
    }
    PB_REQUIRE(per_sm >= 1, PB_ERR_CUDA, "pb_gae: kernel does not fit on an SM (smem %zu)", g.smem);
    int grid = per_sm * PB_NUM_SMS;
    if (grid > g.numTiles) grid = g.numTiles;
    if (g.RW == 16) k_gae<16><<<grid, GAE_THREADS, g.smem, s>>>(p);
    else k_gae<32><<<grid, GAE_THREADS, g.smem, s>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

// 0 (default): chosen by horizon; 2: k_gae_tile (double-buffered tiles, coalesced outputs); 3: k_gae_tile single-buffered;
// 1: the round-1 k_gae_fast.  For A/B measurements.
extern "C" int pb_gae_set_variant(int32_t variant) {
    PB_REQUIRE(variant >= 0 && variant <= 3, PB_ERR_INVALID, "pb_gae_set_variant: 0 .. 3");
    g_gae_variant = variant;
    return PB_OK;
}
