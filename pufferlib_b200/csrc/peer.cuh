// peer.cuh -- device side of the NVLink peer-memory all-reduce (see peer.cu); included by the optimizer kernel.
#pragma once
#include <string.h>

#include "pb_common.cuh"

constexpr int PB_PEER_HEADER_BYTES = 1024;   // 8 flag lines of 128 B

// Host check shared by every entry point that takes the optional fp64 payload: both or neither of kl_in / kl_out, 8-byte
// aligned; with them the communicator has >= 2 ranks and the slot has room for the 4 payload floats after round4(n) gradient
// floats.
static inline int pb_peer_check_payload(const char* who, const pb_peer_comm* comm, int64_t n, const double* kl_in,
                                        const double* kl_out) {
    PB_REQUIRE((kl_in == nullptr) == (kl_out == nullptr), PB_ERR_INVALID, "%s: give both kl_in and kl_out, or neither", who);
    PB_REQUIRE((uintptr_t)kl_in % 8 == 0 && (uintptr_t)kl_out % 8 == 0, PB_ERR_INVALID, "%s: misaligned kl_in or kl_out", who);
    if (kl_in) {
        PB_REQUIRE(comm && comm->world >= 2, PB_ERR_INVALID, "%s: a KL payload needs a communicator of 2 or more ranks", who);
        PB_REQUIRE(((n + 3) & ~(int64_t)3) + 4 <= comm->capacity, PB_ERR_INVALID,
                   "%s: no room for the KL payload (round4(%lld) + 4 floats > capacity %lld)", who, (long long)n,
                   (long long)comm->capacity);
    }
    return PB_OK;
}

#ifdef __CUDACC__
__device__ __forceinline__ void pb_st_release_sys_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t pb_ld_acquire_sys_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float pb_ld_relaxed_sys_f32(const float* p) {   // peer data: never from a stale L1 line
    float v;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ float4 pb_ld_relaxed_sys_f32x4(const float* p) {
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}

// The optional fp64 payload of an exchange (the KL row sum of pb_clip_adam_peer_ex / _parts_ex): 4 reserved floats of the
// slot right after the gradient, at round4(n), as 32-bit words (lo, hi, 0, 0) -- word stores, so a slot of any alignment
// holds it.  Written by one thread before its CTA's flag store, read by one thread after the CTA's flag waits.
__device__ __forceinline__ int64_t pb_peer_payload_offset(int64_t n) { return (n + 3) & ~(int64_t)3; }
__device__ __forceinline__ void pb_peer_payload_put(float* slot_payload, double v) {
    uint32_t* w = reinterpret_cast<uint32_t*>(slot_payload);
    w[0] = (uint32_t)__double2loint(v);
    w[1] = (uint32_t)__double2hiint(v);
    w[2] = 0u;
    w[3] = 0u;
}
// sum over ranks of the payloads in slot offset `off`, in rank order from 0.0: the same bits on every rank
__device__ __forceinline__ double pb_peer_payload_sum(const pb_peer_comm& c, int64_t off) {
    double s = 0.0;
    for (int r = 0; r < c.world; ++r) {
        const float* p = reinterpret_cast<const float*>(c.base[r]) + off;
        s += __hiloint2double(__float_as_int(pb_ld_relaxed_sys_f32(p + 1)), __float_as_int(pb_ld_relaxed_sys_f32(p)));
    }
    return s;
}

// One CTA (any size that is a multiple of 32): flat[0..n) <- sum over ranks, in rank order (bit-identical everywhere).
// kl_in (nullable, then kl_out too): this rank's payload; *kl_out <- the ranks' payloads summed in rank order.
__device__ __forceinline__ void pb_peer_allreduce_sum(const pb_peer_comm& c, float* flat, int64_t n, const double* kl_in = nullptr,
                                                      double* kl_out = nullptr) {
    if (c.world <= 1) return;
    __shared__ uint64_t s_epoch;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) s_epoch = *c.epoch + 1;
    __syncthreads();
    const uint64_t e = s_epoch;
    const int64_t slot_off = PB_PEER_HEADER_BYTES / 4 + (int64_t)(e & 1) * c.capacity;
    float* mine = reinterpret_cast<float*>(c.base[c.rank]) + slot_off;
    // 128-bit accesses where the layout allows (capacity % 4 == 0 keeps both slots 16-byte aligned): at 68 KB per rank the
    // exchange is latency-bound, so every thread should have all its peer loads in flight at once
    const bool vec = (c.capacity & 3) == 0 && (reinterpret_cast<uintptr_t>(flat) & 15) == 0;
    const int64_t n4 = vec ? n >> 2 : 0;
    for (int64_t i = tid; i < n4; i += nt) reinterpret_cast<float4*>(mine)[i] = reinterpret_cast<const float4*>(flat)[i];
    for (int64_t i = 4 * n4 + tid; i < n; i += nt) mine[i] = flat[i];
    if (kl_in && tid == 0) pb_peer_payload_put(mine + pb_peer_payload_offset(n), *kl_in);
    __threadfence_system();
    __syncthreads();
    if (tid < c.world) {   // raise my flag in every rank's buffer (mine included)
        uint64_t* flag = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(c.base[tid]) + 128 * c.rank);
        pb_st_release_sys_u64(flag, e);
        // ... and wait for rank `tid`'s flag in my buffer
        const uint64_t* theirs = reinterpret_cast<const uint64_t*>(reinterpret_cast<const char*>(c.base[c.rank]) + 128 * tid);
        const long long t0 = clock64();
        while (pb_ld_acquire_sys_u64(theirs) < e) {
            if (clock64() - t0 > 20000000000ll) __trap();   // ~10 s: a peer died; do not hang the box
            __nanosleep(64);
        }
    }
    __syncthreads();
    for (int64_t i = tid; i < n4; i += nt) {
        float4 v[PB_PEER_MAX_RANKS];
#pragma unroll
        for (int r = 0; r < PB_PEER_MAX_RANKS; ++r)
            if (r < c.world) v[r] = pb_ld_relaxed_sys_f32x4(reinterpret_cast<const float*>(c.base[r]) + slot_off + 4 * i);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < PB_PEER_MAX_RANKS; ++r)      // rank order: the same bits on every rank
            if (r < c.world) { s.x += v[r].x; s.y += v[r].y; s.z += v[r].z; s.w += v[r].w; }
        reinterpret_cast<float4*>(flat)[i] = s;
    }
    for (int64_t i = 4 * n4 + tid; i < n; i += nt) {
        float s = 0.f;
        for (int r = 0; r < c.world; ++r) s += pb_ld_relaxed_sys_f32(reinterpret_cast<const float*>(c.base[r]) + slot_off + i);
        flat[i] = s;
    }
    if (kl_in && tid == 0) *kl_out = pb_peer_payload_sum(c, slot_off + pb_peer_payload_offset(n));
    __syncthreads();
    if (tid == 0) *c.epoch = e;
}

constexpr int PB_PEER_SLICES = 16;           // flags of source rank r, slice b at byte 128 r + 8 b of the header

// Multi-CTA form: CTA b (of PB_PEER_SLICES) sums slice b over all ranks.  Slices are independent (own flag per rank and
// slice), so there is no grid-wide barrier; the epoch counter is NOT advanced here (every CTA reads it at its start): the
// kernel that follows in the stream does it (pb_clip_adam_parts).  sumsq[b] = sum of squares of the summed slice.
// kl_in / kl_out: the payload, as in pb_peer_allreduce_sum, owned by the CTA of the last slice (the payload follows the
// gradient's tail) and carried by that CTA's own flags.
__device__ __forceinline__ void pb_peer_allreduce_slice(const pb_peer_comm& c, float* flat, int64_t n, double* sumsq,
                                                        const double* kl_in = nullptr, double* kl_out = nullptr) {
    __shared__ uint64_t s_epoch;
    __shared__ double s_sq[32];
    const int tid = threadIdx.x, nt = blockDim.x, b = blockIdx.x;
    if (tid == 0) s_epoch = *c.epoch + 1;
    __syncthreads();
    const uint64_t e = s_epoch;
    const int64_t chunk = ((n + PB_PEER_SLICES - 1) / PB_PEER_SLICES + 3) & ~(int64_t)3;
    // a short buffer leaves the trailing slices empty: lo = hi = n (an unclamped lo > n would put hi4 below hi when n % 4 != 0,
    // and this CTA would then sum the last n % 4 elements a second time)
    const int64_t lo = (int64_t)b * chunk < n ? (int64_t)b * chunk : n, hi = lo + chunk < n ? lo + chunk : n;
    const int64_t slot_off = PB_PEER_HEADER_BYTES / 4 + (int64_t)(e & 1) * c.capacity;
    float* mine = reinterpret_cast<float*>(c.base[c.rank]) + slot_off;
    // 128-bit accesses where the layout allows (slices start at multiples of 4 floats): one peer load per thread and rank,
    // all in flight at once -- the exchange is a handful of NVLink round trips, not bandwidth
    const bool vec = (c.capacity & 3) == 0 && (reinterpret_cast<uintptr_t>(flat) & 15) == 0;
    const int64_t hi4 = vec ? lo + ((hi - lo) & ~(int64_t)3) : lo;          // [lo, hi4) in float4 steps, [hi4, hi) scalar
    for (int64_t i = lo + 4 * tid; i < hi4; i += 4 * nt)
        *reinterpret_cast<float4*>(mine + i) = *reinterpret_cast<const float4*>(flat + i);
    for (int64_t i = hi4 + tid; i < hi; i += nt) mine[i] = flat[i];
    const bool payload = kl_in && b == PB_PEER_SLICES - 1;
    if (payload && tid == 0) pb_peer_payload_put(mine + pb_peer_payload_offset(n), *kl_in);
    __syncthreads();
    if (tid < c.world) {
        __threadfence_system();      // (cumulative: the CTA barrier ordered every thread's slot writes before this thread)
        uint64_t* flag = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(c.base[tid]) + 128 * c.rank + 8 * b);
        pb_st_release_sys_u64(flag, e);
        const uint64_t* theirs = reinterpret_cast<const uint64_t*>(reinterpret_cast<const char*>(c.base[c.rank]) + 128 * tid + 8 * b);
        const long long t0 = clock64();
        while (pb_ld_acquire_sys_u64(theirs) < e) {
            if (clock64() - t0 > 20000000000ll) __trap();
        }
    }
    __syncthreads();
    if (payload && tid == 0) *kl_out = pb_peer_payload_sum(c, slot_off + pb_peer_payload_offset(n));
    double sq = 0.0;
    for (int64_t i = lo + 4 * tid; i < hi4; i += 4 * nt) {
        float4 v[PB_PEER_MAX_RANKS];
#pragma unroll
        for (int r = 0; r < PB_PEER_MAX_RANKS; ++r)
            if (r < c.world) v[r] = pb_ld_relaxed_sys_f32x4(reinterpret_cast<const float*>(c.base[r]) + slot_off + i);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < PB_PEER_MAX_RANKS; ++r)      // rank order: the same bits on every rank
            if (r < c.world) { s.x += v[r].x; s.y += v[r].y; s.z += v[r].z; s.w += v[r].w; }
        *reinterpret_cast<float4*>(flat + i) = s;
        sq += ((double)s.x * (double)s.x + (double)s.y * (double)s.y) + ((double)s.z * (double)s.z + (double)s.w * (double)s.w);
    }
    for (int64_t i = hi4 + tid; i < hi; i += nt) {
        float s = 0.f;
        for (int r = 0; r < c.world; ++r) s += pb_ld_relaxed_sys_f32(reinterpret_cast<const float*>(c.base[r]) + slot_off + i);
        flat[i] = s;
        sq += (double)s * (double)s;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
    if ((tid & 31) == 0) s_sq[tid >> 5] = sq;
    __syncthreads();
    if (tid == 0) {
        double tot = 0.0;
        for (int w = 0; w < (nt + 31) / 32; ++w) tot += s_sq[w];
        sumsq[b] = tot;
    }
}
#endif
