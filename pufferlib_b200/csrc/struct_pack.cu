// struct_pack.cu -- batch pack / unpack of structured (Dict / Tuple) observations into C-aligned records (sm_90a).
//
// Replaces, for N samples at once on the device, reference pufferlib/extensions.pyx:19-30 (`emulate`: the
// recursive per-leaf `np_struct[key][()] = sample` into an `np.dtype(..., align=True)` record,
// reference pufferlib/emulation.py:68-80) and :32-49 (`nativize`, the inverse).  The layout (leaf byte offsets
// and sizes incl. alignment padding) is computed on the host by pufferlib_b200/emulation.py with numpy's own rules.
// One warp per record: lanes stride over the record's bytes, find the covering leaf (<= 32 leaves, warp-uniform
// table in registers/constant bank) and move one byte each -- 32 consecutive bytes per warp request, so global
// traffic is sector-coalesced on the record side; padding bytes are written as zero.
#include "pb_common.cuh"

namespace {

struct PackParams {
    pb_struct_layout lay;
    const unsigned char* leaf[32];
    unsigned char* leaf_out[32];
    unsigned char* rec;
    int64_t rec_stride;
    int64_t n;
};

template <bool PACK>
__global__ void __launch_bounds__(256) k_struct(const __grid_constant__ PackParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t e = warp; e < p.n; e += nwarps) {
        unsigned char* rec = p.rec + e * p.rec_stride;
        for (int b = lane; b < p.lay.record_bytes; b += 32) {
            int l = -1;
#pragma unroll 1
            for (int k = 0; k < p.lay.n_leaves; ++k)
                if (b >= p.lay.offset[k] && b < p.lay.offset[k] + p.lay.nbytes[k]) { l = k; break; }
            if (PACK) {
                rec[b] = l >= 0 ? p.leaf[l][e * p.lay.nbytes[l] + (b - p.lay.offset[l])] : (unsigned char)0;
            } else if (l >= 0) {
                p.leaf_out[l][e * p.lay.nbytes[l] + (b - p.lay.offset[l])] = rec[b];
            }
        }
    }
}

int check_layout(const pb_struct_layout* lay, const char* who) {
    PB_REQUIRE(lay, PB_ERR_INVALID, "%s: null layout", who);
    PB_REQUIRE(lay->n_leaves >= 1 && lay->n_leaves <= 32 && lay->record_bytes >= 1, PB_ERR_INVALID,
               "%s: bad layout (n_leaves=%d, record_bytes=%d)", who, lay->n_leaves, lay->record_bytes);
    for (int k = 0; k < lay->n_leaves; ++k)
        PB_REQUIRE(lay->offset[k] >= 0 && lay->nbytes[k] >= 1 && lay->offset[k] + lay->nbytes[k] <= lay->record_bytes,
                   PB_ERR_INVALID, "%s: leaf %d out of the record", who, k);
    return PB_OK;
}

int grid_for(int64_t n) {
    int64_t blocks = pb_ceil_div(n, 8);
    const int64_t cap = (int64_t)PB_NUM_SMS * 8;
    return (int)(blocks > cap ? cap : (blocks < 1 ? 1 : blocks));
}

}  // namespace

extern "C" int pb_struct_pack(const pb_struct_layout* layout, const void* const* leaves_host, void* records,
                              int64_t record_stride, int64_t n, void* stream) {
    int rc = check_layout(layout, "pb_struct_pack");
    if (rc) return rc;
    PB_REQUIRE(n >= 0, PB_ERR_INVALID, "pb_struct_pack: negative n");
    if (n == 0) return PB_OK;
    PB_REQUIRE(leaves_host && records && record_stride >= layout->record_bytes, PB_ERR_INVALID,
               "pb_struct_pack: null pointer or record_stride < record_bytes");
    PackParams p{};
    p.lay = *layout;
    for (int k = 0; k < layout->n_leaves; ++k) {
        PB_REQUIRE(leaves_host[k], PB_ERR_INVALID, "pb_struct_pack: leaf %d is null", k);
        p.leaf[k] = (const unsigned char*)leaves_host[k];
    }
    p.rec = (unsigned char*)records; p.rec_stride = record_stride; p.n = n;
    k_struct<true><<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}

extern "C" int pb_struct_unpack(const pb_struct_layout* layout, const void* records, int64_t record_stride,
                                void* const* leaves_host, int64_t n, void* stream) {
    int rc = check_layout(layout, "pb_struct_unpack");
    if (rc) return rc;
    PB_REQUIRE(n >= 0, PB_ERR_INVALID, "pb_struct_unpack: negative n");
    if (n == 0) return PB_OK;
    PB_REQUIRE(leaves_host && records && record_stride >= layout->record_bytes, PB_ERR_INVALID,
               "pb_struct_unpack: null pointer or record_stride < record_bytes");
    PackParams p{};
    p.lay = *layout;
    for (int k = 0; k < layout->n_leaves; ++k) {
        PB_REQUIRE(leaves_host[k], PB_ERR_INVALID, "pb_struct_unpack: leaf %d is null", k);
        p.leaf_out[k] = (unsigned char*)leaves_host[k];
    }
    p.rec = (unsigned char*)records; p.rec_stride = record_stride; p.n = n;
    k_struct<false><<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(p);
    PB_LAUNCH_CHECK();
    return PB_OK;
}
