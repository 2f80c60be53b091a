// mt19937.cuh -- MT19937 pieces shared by the env kinds that restate a process-global Mersenne Twister stream:
// CPython's `random` (squared: init_by_array seeding) and numpy's legacy `np.random` (memory, password, bandit:
// init_genrand seeding).  Both generators twist and temper identically; only the seeding differs.
#pragma once
#include <stdint.h>

constexpr int MT_N = 624, MT_M = 397;

__host__ __device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
    y ^= y >> 11;
    y ^= (y << 7) & 0x9D2C5680u;
    y ^= (y << 15) & 0xEFC60000u;
    y ^= y >> 18;
    return y;
}
__host__ __device__ __forceinline__ uint32_t mt_mix(uint32_t u, uint32_t v) {
    const uint32_t y = (u & 0x80000000u) | (v & 0x7FFFFFFFu);
    return (y >> 1) ^ ((y & 1u) ? 0x9908B0DFu : 0u);
}

// numpy RandomState.seed(int) / mt19937_seed: init_genrand(s).  The next output twists first.
__host__ __device__ inline void mt_seed_genrand(uint32_t* mt, uint32_t s) {
    mt[0] = s;
    for (int k = 1; k < MT_N; ++k) mt[k] = 1812433253u * (mt[k - 1] ^ (mt[k - 1] >> 30)) + (uint32_t)k;
}

// CPython random.seed(int): init_by_array(32-bit little-endian words of |seed|).  The next output twists first.
__host__ __device__ inline void mt_seed_by_array(uint32_t* mt, uint64_t s) {
    uint32_t key[2] = {(uint32_t)s, (uint32_t)(s >> 32)};
    const int klen = key[1] ? 2 : 1;
    mt_seed_genrand(mt, 19650218u);
    int a = 1, b = 0;
    for (int k = (MT_N > klen ? MT_N : klen); k; --k) {
        mt[a] = (mt[a] ^ ((mt[a - 1] ^ (mt[a - 1] >> 30)) * 1664525u)) + key[b] + (uint32_t)b;
        ++a; ++b;
        if (a >= MT_N) { mt[0] = mt[MT_N - 1]; a = 1; }
        if (b >= klen) b = 0;
    }
    for (int k = MT_N - 1; k; --k) {
        mt[a] = (mt[a] ^ ((mt[a - 1] ^ (mt[a - 1] >> 30)) * 1566083941u)) - (uint32_t)a;
        ++a;
        if (a >= MT_N) { mt[0] = mt[MT_N - 1]; a = 1; }
    }
    mt[0] = 0x80000000u;
}

// One thread's twist of a whole state (in place, serial order).
__host__ __device__ inline void mt_twist(uint32_t* mt) {
    for (int k = 0; k < MT_N; ++k) mt[k] = mt[(k + MT_M) % MT_N] ^ mt_mix(mt[k], mt[(k + 1) % MT_N]);
}

// Next output of a thread-local generator (`idx` = position in the state, MT_N after seeding).
__host__ __device__ __forceinline__ uint32_t mt_next(uint32_t* mt, int& idx) {
    if (idx >= MT_N) {
        mt_twist(mt);
        idx = 0;
    }
    return mt_temper(mt[idx++]);
}

#ifdef __CUDACC__
// Block-parallel twist of a shared-memory state by THREADS threads: 3 independent spans + the wrap-around element.
template <int THREADS>
__device__ void mt_twist_block(uint32_t* mt) {
    constexpr int PER = (MT_N - MT_M + THREADS - 1) / THREADS;
    const int tid = threadIdx.x;
    uint32_t v[PER];
    int cnt = 0;
    for (int k = tid; k < MT_N - MT_M; k += THREADS) v[cnt++] = mt[k + MT_M] ^ mt_mix(mt[k], mt[k + 1]);
    __syncthreads();
    cnt = 0;
    for (int k = tid; k < MT_N - MT_M; k += THREADS) mt[k] = v[cnt++];
    __syncthreads();
    cnt = 0;
    for (int k = MT_N - MT_M + tid; k < 2 * (MT_N - MT_M); k += THREADS)
        v[cnt++] = mt[k - (MT_N - MT_M)] ^ mt_mix(mt[k], mt[k + 1]);
    __syncthreads();
    cnt = 0;
    for (int k = MT_N - MT_M + tid; k < 2 * (MT_N - MT_M); k += THREADS) mt[k] = v[cnt++];
    __syncthreads();
    cnt = 0;
    for (int k = 2 * (MT_N - MT_M) + tid; k < MT_N - 1; k += THREADS)
        v[cnt++] = mt[k - (MT_N - MT_M)] ^ mt_mix(mt[k], mt[k + 1]);
    __syncthreads();
    cnt = 0;
    for (int k = 2 * (MT_N - MT_M) + tid; k < MT_N - 1; k += THREADS) mt[k] = v[cnt++];
    __syncthreads();
    if (tid == 0) mt[MT_N - 1] = mt[MT_M - 1] ^ mt_mix(mt[MT_N - 1], mt[0]);
    __syncthreads();
}

// Exclusive prefix sum of one int per thread over a block of THREADS threads; *total = the block's sum.
template <int THREADS>
__device__ int block_exclusive_scan(int v, int* total, int* s_warp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, off);
        if (lane >= off) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int base = 0, tot = 0;
    for (int w = 0; w < THREADS / 32; ++w) {
        if (w < warp) base += s_warp[w];
        tot += s_warp[w];
    }
    __syncthreads();
    *total = tot;
    return base + x - v;
}

// Rank, in env order, the envs whose `done` flag is set (d_rank[e] = rank or -1); returns the count R.
template <int THREADS>
__device__ int rank_resets(const uint8_t* done, int n, int32_t* d_rank, int* s_warp) {
    int R = 0;
    for (int base = 0; base < n; base += THREADS) {
        const int e = base + threadIdx.x;
        const int flag = (e < n && done[e]) ? 1 : 0;
        int tot;
        const int off = block_exclusive_scan<THREADS>(flag, &tot, s_warp);
        if (e < n) d_rank[e] = flag ? R + off : -1;
        R += tot;
    }
    return R;
}
#endif
