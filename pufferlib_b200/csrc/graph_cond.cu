// graph_cond.cu -- the PPO early stop (target_kl, clean_pufferl.py:256-258) decided on the device, and the conditional
// (IF) graph nodes that let a captured train() skip the epochs after it.
//
// pb_kl_stop is one thread: it forms the last minibatch's approx_kl, compares it with target_kl in fp32 as torch does
// for `tensor > float`, records the decision and the epochs it lets run, and, inside a captured graph, sets the
// conditional handle that gates the next epoch's IF node.  The pb_graph_* helpers add those IF nodes to a stream
// capture (CUDA 12.4+ conditional nodes); a handle belongs to one conditional node, so each IF node has its own, and
// every handle is created on the root graph of the capture, which contains all the IF nodes.  cudaGraphSetConditional is
// a device-runtime builtin: it compiles without relocatable device code and needs no cudadevrt.
#include "pb_common.cuh"

__global__ void __launch_bounds__(1) k_kl_stop(const float* __restrict__ approx_kl, const double* __restrict__ kl_sum,
                                               int64_t rows, const float* __restrict__ target_kl, int32_t epoch, int32_t* state,
                                               cudaGraphConditionalHandle handle, int32_t use_handle) {
    bool stop;
    if (epoch > 0 && state[0] != 0) {
        stop = true;                      // an earlier epoch of this call stopped: stays stopped
    } else {
        // the fused loss's value: fp64 mean of the row sum, rounded once to fp32 (fused_ppo_loss: (stats / m).float())
        const float kl = approx_kl ? *approx_kl : __double2float_rn(*kl_sum / (double)rows);
        stop = kl > *target_kl;           // NaN compares false: never stops
        state[0] = stop ? 1 : 0;
        state[1] = epoch + (stop ? 1 : 2);
    }
    if (use_handle) cudaGraphSetConditional(handle, stop ? 0u : 1u);
}

extern "C" int pb_kl_stop(const float* approx_kl, const double* kl_sum, int64_t rows, const float* target_kl, int32_t epoch,
                          int32_t* state, uint64_t cond_handle, int32_t use_handle, void* stream) {
    PB_REQUIRE((approx_kl != nullptr) != (kl_sum != nullptr), PB_ERR_INVALID,
               "pb_kl_stop: give exactly one of approx_kl and kl_sum");
    PB_REQUIRE(!kl_sum || rows >= 1, PB_ERR_INVALID, "pb_kl_stop: kl_sum needs rows >= 1 (got %lld)", (long long)rows);
    PB_REQUIRE(state && target_kl, PB_ERR_INVALID, "pb_kl_stop: null state or target_kl");
    PB_REQUIRE(((uintptr_t)state % 4) == 0 && ((uintptr_t)approx_kl % 4) == 0 && ((uintptr_t)kl_sum % 8) == 0 &&
                   ((uintptr_t)target_kl % 4) == 0,
               PB_ERR_INVALID, "pb_kl_stop: misaligned pointer");
    PB_REQUIRE(epoch >= 0, PB_ERR_INVALID, "pb_kl_stop: epoch %d < 0", epoch);
    k_kl_stop<<<1, 1, 0, (cudaStream_t)stream>>>(approx_kl, kl_sum, rows, target_kl, epoch, state,
                                                 (cudaGraphConditionalHandle)cond_handle, use_handle);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

// The graph `stream` is capturing into, and the nodes its next node will depend on.
static int capture_info(cudaStream_t s, const char* who, cudaGraph_t* graph, const cudaGraphNode_t** deps, size_t* n_deps) {
    PB_REQUIRE(s != nullptr, PB_ERR_INVALID, "%s: the legacy default stream cannot be captured", who);
    cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
    unsigned long long id = 0;
    PB_CUDA(cudaStreamGetCaptureInfo(s, &status, &id, graph, deps, n_deps));
    PB_REQUIRE(status == cudaStreamCaptureStatusActive, PB_ERR_STATE, "%s: the stream is not capturing a graph", who);
    return PB_OK;
}

extern "C" int pb_graph_cond_create(void* stream, uint32_t default_value, uint64_t* handle_out) {
    PB_REQUIRE(handle_out, PB_ERR_INVALID, "pb_graph_cond_create: null handle_out");
    cudaGraph_t graph = nullptr;
    int rc = capture_info((cudaStream_t)stream, "pb_graph_cond_create", &graph, nullptr, nullptr);
    if (rc) return rc;
    cudaGraphConditionalHandle h = 0;
    // every launch of the graph starts with default_value (cudaGraphCondAssignDefault)
    PB_CUDA(cudaGraphConditionalHandleCreate(&h, graph, default_value, cudaGraphCondAssignDefault));
    *handle_out = (uint64_t)h;
    return PB_OK;
}

extern "C" int pb_graph_if_begin(uint64_t cond_handle, void* stream, void* body_stream) {
    cudaStream_t s = (cudaStream_t)stream, b = (cudaStream_t)body_stream;
    PB_REQUIRE(b != nullptr && b != s, PB_ERR_INVALID, "pb_graph_if_begin: body_stream must be a second, non-default stream");
    cudaStreamCaptureStatus body_status = cudaStreamCaptureStatusNone;
    PB_CUDA(cudaStreamIsCapturing(b, &body_status));
    PB_REQUIRE(body_status == cudaStreamCaptureStatusNone, PB_ERR_STATE, "pb_graph_if_begin: body_stream is already capturing");
    // the dependency array belongs to the capture and is only valid until the next call on it: add the node right away
    cudaGraph_t graph = nullptr;
    const cudaGraphNode_t* deps = nullptr;
    size_t n_deps = 0;
    int rc = capture_info(s, "pb_graph_if_begin", &graph, &deps, &n_deps);
    if (rc) return rc;

    cudaGraphNodeParams p = {};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = (cudaGraphConditionalHandle)cond_handle;
    p.conditional.type = cudaGraphCondTypeIf;
    p.conditional.size = 1;
    cudaGraphNode_t node = nullptr;
    PB_CUDA(cudaGraphAddNode(&node, graph, deps, n_deps, &p));
    PB_CUDA(cudaStreamUpdateCaptureDependencies(s, &node, 1, cudaStreamSetCaptureDependencies));
    PB_CUDA(cudaStreamBeginCaptureToGraph(b, p.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                          cudaStreamCaptureModeGlobal));
    return PB_OK;
}

extern "C" int pb_stream_create(void** stream_out) {
    PB_REQUIRE(stream_out, PB_ERR_INVALID, "pb_stream_create: null stream_out");
    cudaStream_t s = nullptr;
    PB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    *stream_out = (void*)s;
    return PB_OK;
}

extern "C" int pb_stream_destroy(void* stream) {
    if (stream) PB_CUDA(cudaStreamDestroy((cudaStream_t)stream));
    return PB_OK;
}

extern "C" int pb_graph_if_end(void* body_stream) {
    cudaStream_t b = (cudaStream_t)body_stream;
    PB_REQUIRE(b != nullptr, PB_ERR_INVALID, "pb_graph_if_end: null body_stream");
    cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
    PB_CUDA(cudaStreamIsCapturing(b, &status));
    PB_REQUIRE(status != cudaStreamCaptureStatusNone, PB_ERR_STATE, "pb_graph_if_end: body_stream is not capturing");
    cudaGraph_t body = nullptr;
    PB_CUDA(cudaStreamEndCapture(b, &body));   // the IF node's own body graph: owned by the node, nothing to free
    return PB_OK;
}
