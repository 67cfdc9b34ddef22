// fast_slic_b200/csrc/capi_message.cu -- the extern "C" entry points of message passing over superpixel graphs
// (message_passing.cuh): edge_gather, edge_softmax and aggregate, forward and backward.  Stateless (device pointers,
// caller-provided scratch), asynchronous on the caller's stream, never synchronise.
#include <limits.h>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "message_passing.cuh"

enum { MP_SUM = 0, MP_MEAN = 1, MP_MAX = 2 };

static bool mp_args_ok(long long N, long long E, int C, int H) {
    return N >= 0 && N <= INT_MAX && E >= 0 && E <= INT_MAX && C >= 1 && H >= 1 && C % H == 0;
}

// Checks the arguments and the non-null pointers (d_targets unless E is 0); returns early (FSLIC_OK) when there is
// nothing to do
#define MP_BEGIN(N, E, C, H, work, ...)                                                               \
    if (!mp_args_ok(N, E, C, H)) return set_err(FSLIC_EINVAL, "bad N, E, C or H");                  \
    if (!(work)) return FSLIC_OK;                                                                     \
    if ((E) > 0 && !d_targets) return set_err(FSLIC_EINVAL, "NULL argument");                       \
    {                                                                                                 \
        const void* req__[] = {__VA_ARGS__};                                                          \
        for (const void* r__ : req__)                                                                 \
            if (!r__) return set_err(FSLIC_EINVAL, "NULL argument");                                  \
    }                                                                                                 \
    USE_DEVICE(device);                                                                               \
    cudaStream_t st = (cudaStream_t)stream

// Warps of 8 per CTA over `warps` items
static inline long warp_grid(long warps, int device) { return grid_for(warps * 32, device); }

// The transposed order's scratch: sort keys and values, their sorted copies, the row of every entry (4 bytes each per
// entry), the column offsets (4 bytes per node + 4), the sort's temporary storage and, for the mean, grad_out / deg.
struct MpScratch {
    uint32_t *key, *skey, *val, *sval, *rowof, *tptr;
    float* scaled;
    void* temp;
    size_t temp_bytes, total;
};

static MpScratch mp_layout(long long N, long long E, int C, bool scaled, void* base) {
    MpScratch s;
    Carve c(base);
    s.key = c.take<uint32_t>((size_t)E * 4);
    s.skey = c.take<uint32_t>((size_t)E * 4);
    s.val = c.take<uint32_t>((size_t)E * 4);
    s.sval = c.take<uint32_t>((size_t)E * 4);
    s.rowof = c.take<uint32_t>((size_t)E * 4);
    s.tptr = c.take<uint32_t>((size_t)(N + 1) * 4);
    s.scaled = c.take<float>(scaled ? (size_t)N * C * 4 : 0);
    s.temp_bytes = align_up(radix_pairs_temp_bytes<uint32_t, uint32_t>(E, 32), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

// The transposed order: rowof, then one stable radix sort of the entries by target (invalid targets keyed N, past every
// node) and the column offsets tptr [N+1] by binary search
static int mp_transpose(const MpScratch& s, const long long* indptr, const long long* tgt, long N, long E, int device,
                        cudaStream_t st) {
    if (E == 0) {
        CK(cudaMemsetAsync(s.tptr, 0, (size_t)(N + 1) * 4, st));
        return FSLIC_OK;
    }
    k_mp_keys<<<(int)grid_for(E, device), 256, 0, st>>>(indptr, tgt, N, E, s.key, s.val, s.rowof);
    const int bits = bit_length((unsigned long long)N);
    size_t temp_bytes = s.temp_bytes;
    if (radix_pairs_temp_bytes<uint32_t, uint32_t>(E, bits) > temp_bytes)
        return set_err(FSLIC_ECUDA, "radix sort temporary storage");
    if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.key, s.skey, s.val, s.sval, (int)E, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the entry targets failed");
    k_mp_bounds<<<(int)grid_for(N + 1, device), 256, 0, st>>>(s.skey, N, E, s.tptr);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_mp_gather(int device, long long N, long long E, int C, int end, const long long* d_indptr,
                                    const long long* d_targets, const float* d_x, float* d_out, void* stream) {
    if (end != 0 && end != 1) return set_err(FSLIC_EINVAL, "end must be 0 (target) or 1 (source)");
    MP_BEGIN(N, E, C, 1, N > 0 && E > 0, d_indptr, d_x, d_out);
    if (end == 0)
        k_mp_gather_target<<<(int)grid_for(E * C, device), 256, 0, st>>>(d_targets, d_x, N, E, C, d_out);
    else
        k_mp_gather_source<<<(int)warp_grid(N, device), 256, 0, st>>>(d_indptr, d_targets, d_x, N, E, C, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" size_t fslic_b200_mp_gather_backward_scratch_bytes(long long N, long long E) {
    if (!mp_args_ok(N, E, 1, 1)) return (size_t)-1;
    return mp_layout(N, E, 1, false, nullptr).total;
}

extern "C" int fslic_b200_mp_gather_backward(int device, long long N, long long E, int C, int end,
                                             const long long* d_indptr, const long long* d_targets,
                                             const float* d_grad_out, float* d_grad_x, void* d_scratch,
                                             size_t scratch_bytes, void* stream) {
    if (end != 0 && end != 1) return set_err(FSLIC_EINVAL, "end must be 0 (target) or 1 (source)");
    MP_BEGIN(N, E, C, 1, N > 0, d_indptr, d_grad_x);
    if (E > 0 && !d_grad_out) return set_err(FSLIC_EINVAL, "NULL argument");
    if (end == 1) {
        k_mp_sum<MP_ROWS><<<(int)warp_grid(N, device), 256, 0, st>>>(d_indptr, d_targets, nullptr, nullptr, nullptr,
                                                                     d_grad_out, nullptr, nullptr, N, E, C, 1,
                                                                     d_grad_x, nullptr, nullptr);
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    if (!d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < fslic_b200_mp_gather_backward_scratch_bytes(N, E))
        return set_err(FSLIC_EINVAL, "scratch too small");
    const MpScratch s = mp_layout(N, E, C, false, d_scratch);
    const int rc = mp_transpose(s, d_indptr, d_targets, N, E, device, st);
    if (rc != FSLIC_OK) return rc;
    k_mp_sum<MP_COLS><<<(int)warp_grid(N, device), 256, 0, st>>>(d_indptr, d_targets, s.tptr, s.sval, s.rowof,
                                                                 d_grad_out, nullptr, nullptr, N, E, C, 1, d_grad_x,
                                                                 nullptr, nullptr);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_mp_softmax(int device, long long N, long long E, int H, const long long* d_indptr,
                                     const long long* d_targets, const float* d_scores, float* d_out, void* stream) {
    MP_BEGIN(N, E, H, H, N > 0 && E > 0, d_indptr, d_scores, d_out);
    k_mp_softmax<<<(int)grid_for(N * H, device), 256, 0, st>>>(d_indptr, d_targets, d_scores, N, E, H, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_mp_softmax_backward(int device, long long N, long long E, int H, const long long* d_indptr,
                                              const long long* d_targets, const float* d_out, const float* d_grad_out,
                                              float* d_grad_scores, void* stream) {
    MP_BEGIN(N, E, H, H, N > 0 && E > 0, d_indptr, d_out, d_grad_out, d_grad_scores);
    k_mp_softmax_bwd<<<(int)grid_for(N * H, device), 256, 0, st>>>(d_indptr, d_targets, d_out, d_grad_out, N, E, H,
                                                                   d_grad_scores);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_mp_aggregate(int device, long long N, long long E, int C, int H, int reduce,
                                       const long long* d_indptr, const long long* d_targets, const float* d_x,
                                       const float* d_weight, float* d_out, int32_t* d_deg, int32_t* d_amax,
                                       void* stream) {
    if (reduce < MP_SUM || reduce > MP_MAX) return set_err(FSLIC_EINVAL, "reduce must be 0 (sum), 1 (mean) or 2 (max)");
    MP_BEGIN(N, E, C, H, N > 0, d_indptr, d_x, d_out);
    if (reduce == MP_MEAN && !d_deg) return set_err(FSLIC_EINVAL, "NULL argument");
    if (reduce == MP_MAX && !d_amax) return set_err(FSLIC_EINVAL, "NULL argument");
    const int grid = (int)warp_grid(N, device);
    if (reduce == MP_MAX)
        k_mp_sum<MP_AGG_MAX><<<grid, 256, 0, st>>>(d_indptr, d_targets, nullptr, nullptr, nullptr, d_x, d_weight,
                                                   nullptr, N, E, C, H, d_out, nullptr, d_amax);
    else
        k_mp_sum<MP_AGG><<<grid, 256, 0, st>>>(d_indptr, d_targets, nullptr, nullptr, nullptr, d_x, d_weight, nullptr,
                                               N, E, C, H, d_out, reduce == MP_MEAN ? d_deg : nullptr, nullptr);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" size_t fslic_b200_mp_aggregate_backward_scratch_bytes(long long N, long long E, int C, int reduce) {
    if (!mp_args_ok(N, E, C, 1) || reduce < MP_SUM || reduce > MP_MAX) return (size_t)-1;
    return mp_layout(N, E, C, reduce == MP_MEAN, nullptr).total;
}

extern "C" int fslic_b200_mp_aggregate_backward(int device, long long N, long long E, int C, int H, int reduce,
                                                const long long* d_indptr, const long long* d_targets,
                                                const float* d_x, const float* d_weight, const int32_t* d_deg,
                                                const int32_t* d_amax, const float* d_grad_out, float* d_grad_x,
                                                float* d_grad_weight, void* d_scratch, size_t scratch_bytes,
                                                void* stream) {
    if (reduce < MP_SUM || reduce > MP_MAX) return set_err(FSLIC_EINVAL, "reduce must be 0 (sum), 1 (mean) or 2 (max)");
    MP_BEGIN(N, E, C, H, N > 0, d_indptr, d_x, d_grad_out, d_scratch);
    if ((reduce == MP_MEAN && !d_deg) || (reduce == MP_MAX && !d_amax) || (d_grad_weight && !d_weight))
        return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < fslic_b200_mp_aggregate_backward_scratch_bytes(N, E, C, reduce))
        return set_err(FSLIC_EINVAL, "scratch too small");
    const MpScratch s = mp_layout(N, E, C, reduce == MP_MEAN, d_scratch);
    const int32_t* amax = reduce == MP_MAX ? d_amax : nullptr;
    const float* g = d_grad_out;
    if (reduce == MP_MEAN) {
        k_mp_scale<<<(int)grid_for(N * C, device), 256, 0, st>>>(d_grad_out, d_deg, N, C, s.scaled);
        g = s.scaled;
    }
    const int rc = mp_transpose(s, d_indptr, d_targets, N, E, device, st);
    if (rc != FSLIC_OK) return rc;
    if (d_grad_x)
        k_mp_sum<MP_COLS_AGG><<<(int)warp_grid(N, device), 256, 0, st>>>(d_indptr, d_targets, s.tptr, s.sval, s.rowof,
                                                                         g, d_weight, amax, N, E, C, H, d_grad_x,
                                                                         nullptr, nullptr);
    if (d_grad_weight && E > 0)
        k_mp_grad_weight<<<(int)warp_grid(E, device), 256, 0, st>>>(d_targets, s.rowof, g, d_x, amax, N, E, C, H,
                                                                    d_grad_weight);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
