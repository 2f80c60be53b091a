// peer.cu -- gradient all-reduce over NVLink peer memory, fused into the optimizer step (sm_90a, one node).
//
// The reference has no distributed path (SURVEY §8e); ours shards envs over the GPUs of one box and sums ONE flat
// fp32 gradient buffer per optimizer step (17 157 floats = 68.6 KB for models.Default).  At that size an NCCL call is
// pure launch / host latency (16 calls per step outside the CUDA graph),
// so the exchange is done by the optimizer kernel itself: every rank owns a cudaMalloc'ed buffer mapped into all peers
// (cudaIpc*), copies its gradients into it, raises a flag in every peer's buffer, waits for the peers' flags, and sums
// all ranks' buffers in rank order with direct NVLink loads -- identical bits on every rank, no host involvement, so
// the whole update stays ONE CUDA graph for any world size.
//
// Buffer layout (same on every rank):  [0, 1024) flags: uint64 arrival epoch of source rank r at byte 128 r
//                                      [1024, ...) two gradient slots (epoch parity) of `capacity` floats
// Epoch protocol: e = ++local epoch; slot = e & 1.  A rank can only be one epoch ahead of the slowest peer (it needs
// every peer's flag e to finish epoch e, and a peer raises flag e+1 only after it has finished reading epoch e), so two
// slots suffice.  Waits are bounded (trap instead of a hang).
#include "pb_common.cuh"
#include "peer.cuh"

extern "C" int pb_peer_alloc(size_t bytes, void** ptr_out, void* handle64_out) {
    PB_REQUIRE(bytes >= 1 && ptr_out && handle64_out, PB_ERR_INVALID, "pb_peer_alloc: bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    void* p = nullptr;
    PB_CUDA(cudaMalloc(&p, bytes));
    PB_CUDA(cudaMemset(p, 0, bytes));
    PB_CUDA(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    PB_CUDA(cudaIpcGetMemHandle(&h, p));
    memcpy(handle64_out, &h, 64);
    *ptr_out = p;
    return PB_OK;
}

extern "C" int pb_peer_open(const void* handle64, void** ptr_out) {
    PB_REQUIRE(handle64 && ptr_out, PB_ERR_INVALID, "pb_peer_open: null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    void* p = nullptr;
    PB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *ptr_out = p;
    return PB_OK;
}

extern "C" int pb_peer_close(void* ptr) {
    if (ptr) PB_CUDA(cudaIpcCloseMemHandle(ptr));
    return PB_OK;
}

extern "C" int pb_peer_free(void* ptr) {
    if (ptr) PB_CUDA(cudaFree(ptr));
    return PB_OK;
}

extern "C" size_t pb_peer_buffer_bytes(int64_t capacity_floats) {
    return (size_t)PB_PEER_HEADER_BYTES + 2 * (size_t)capacity_floats * sizeof(float);
}

namespace {
__global__ void __launch_bounds__(1024) k_peer_allreduce(pb_peer_comm c, float* flat, int64_t n) {
    pb_peer_allreduce_sum(c, flat, n);
}
__global__ void __launch_bounds__(512) k_peer_allreduce_slices(pb_peer_comm c, float* flat, int64_t n, double* sumsq) {
    pb_peer_allreduce_slice(c, flat, n, sumsq);
}
}  // namespace

// Sliced form: PB_PEER_SLICES CTAs, each sums one slice over all ranks and leaves the slice's sum of squares in
// sumsq_parts[0..16).  The epoch counter is advanced by the pb_clip_adam_parts call that must follow in the same stream.
extern "C" int pb_peer_allreduce_parts(const pb_peer_comm* comm, float* flat, int64_t n, double* sumsq_parts, void* stream) {
    PB_REQUIRE(comm && flat && n >= 1 && sumsq_parts, PB_ERR_INVALID, "pb_peer_allreduce_parts: bad arguments");
    PB_REQUIRE(comm->world >= 1 && comm->world <= PB_PEER_MAX_RANKS && comm->rank >= 0 && comm->rank < comm->world &&
                   comm->epoch && n <= comm->capacity,
               PB_ERR_INVALID, "pb_peer_allreduce_parts: bad communicator (world %d rank %d capacity %lld, n %lld)", comm->world,
               comm->rank, (long long)comm->capacity, (long long)n);
    for (int r = 0; r < comm->world; ++r) PB_REQUIRE(comm->base[r], PB_ERR_INVALID, "pb_peer_allreduce_parts: peer %d not mapped", r);
    k_peer_allreduce_slices<<<PB_PEER_SLICES, 512, 0, (cudaStream_t)stream>>>(*comm, flat, n, sumsq_parts);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
extern "C" int32_t pb_peer_slices(void) { return PB_PEER_SLICES; }

// In-place sum of flat[0..n) over all ranks (every rank must call it the same number of times).  One CTA.
extern "C" int pb_peer_allreduce(const pb_peer_comm* comm, float* flat, int64_t n, void* stream) {
    PB_REQUIRE(comm && flat && n >= 1, PB_ERR_INVALID, "pb_peer_allreduce: bad arguments");
    PB_REQUIRE(comm->world >= 1 && comm->world <= PB_PEER_MAX_RANKS && comm->rank >= 0 && comm->rank < comm->world &&
                   comm->epoch && n <= comm->capacity,
               PB_ERR_INVALID, "pb_peer_allreduce: bad communicator (world %d rank %d capacity %lld, n %lld)", comm->world,
               comm->rank, (long long)comm->capacity, (long long)n);
    for (int r = 0; r < comm->world; ++r) PB_REQUIRE(comm->base[r], PB_ERR_INVALID, "pb_peer_allreduce: peer %d not mapped", r);
    k_peer_allreduce<<<1, 1024, 0, (cudaStream_t)stream>>>(*comm, flat, n);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
