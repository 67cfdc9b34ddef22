// fast_slic_b200/csrc/capi_pool.cu -- the extern "C" entry points of superpixel pooling (pool.cuh): pool, unpool,
// paint_argmax and paint over a batch of label maps.  Stateless (device pointers, caller-provided scratch), asynchronous
// on the caller's stream, never synchronise.
#include <limits.h>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "pool.cuh"
#include "pool_stage.h"

PoolScratch pool_layout(long long n, long long nk, void* base) {
    PoolScratch s;
    Carve c(base);
    s.key = c.take<uint32_t>((size_t)n * 4);
    s.skey = c.take<uint32_t>((size_t)n * 4);
    s.val = c.take<uint32_t>((size_t)n * 4);
    s.sval = c.take<uint32_t>((size_t)n * 4);
    s.seg_start = c.take<uint32_t>((size_t)nk * 4);
    s.seg_end = c.take<uint32_t>((size_t)nk * 4);
    s.temp_bytes = align_up(radix_pairs_temp_bytes<uint32_t, uint32_t>(n, 32), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

int pool_sorted_segments(const PoolScratch& s, long long n, int batch, int K, int C, long hw, const float* feat,
                         int mean, float* out, int32_t* counts, int device, cudaStream_t st) {
    const long nk = (long)batch * K;
    const int bits = 16 + bit_length((unsigned long long)(batch - 1));
    CK(cudaMemsetAsync(s.seg_start, 0, (size_t)nk * 4, st));
    CK(cudaMemsetAsync(s.seg_end, 0, (size_t)nk * 4, st));
    if (n > 0) {
        if (radix_pairs_temp_bytes<uint32_t, uint32_t>(n, bits) > s.temp_bytes)
            return set_err(FSLIC_ECUDA, "radix sort temporary storage");
        size_t temp_bytes = s.temp_bytes;
        if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.key, s.skey, s.val, s.sval, (int)n, 0, bits, st) !=
            cudaSuccess)
            return set_err(FSLIC_ECUDA, "radix sort of the pixel keys failed");
        k_pool_bounds<<<(int)grid_for(n, device), 256, 0, st>>>(s.skey, n, K, s.seg_start, s.seg_end);
    }
    k_pool_segments<<<(unsigned)((nk + 7) / 8), 256, 0, st>>>(s.seg_start, s.seg_end, s.sval, feat, nk, K, C, hw, mean,
                                                             out, counts);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" size_t fslic_b200_pool_batch_scratch_bytes(int batch, int H, int W, int K) {
    if (!labels_shape_ok(batch, H, W, K)) return (size_t)-1;
    const long long n = (long long)batch * H * W;
    if (n == 0) return 256;
    if (n > INT_MAX || batch > 65536) return (size_t)-1;  // one radix sort of 32-bit keys: split the batch
    return pool_layout(n, (long long)batch * K, nullptr).total;
}

extern "C" int fslic_b200_pool_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                     const float* d_features, int mean, float* d_out, int32_t* d_counts, void* d_scratch,
                                     size_t scratch_bytes, void* stream) {
    if (!labels_shape_ok(batch, H, W, K) || C < 1) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or K");
    const long long n = (long long)batch * H * W;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_features || !d_out || !d_counts || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_pool_batch_scratch_bytes(batch, H, W, K);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long hw = (long)H * W, nk = (long)batch * K;
    const PoolScratch s = pool_layout(n, nk, d_scratch);
    k_pool_keys<<<(int)grid_for(n, device), 256, 0, st>>>(d_labels, hw, n, K, s.key, s.val);
    return pool_sorted_segments(s, n, batch, K, C, hw, d_features, mean ? 1 : 0, d_out, d_counts, device, st);
}

extern "C" int fslic_b200_pool_unpool_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                            const float* d_values, const int32_t* d_divisor, float* d_out, void* stream) {
    if (!labels_shape_ok(batch, H, W, K) || C < 1) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or K");
    const long n = (long)batch * H * W;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_values || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    k_pool_unpool<<<(int)grid_for(n, device), 256, 0, (cudaStream_t)stream>>>(d_labels, d_values, d_divisor, (long)H * W, n, C,
                                                                              K, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_pool_paint_argmax_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                                  const float* d_q, int32_t* d_node_class, int16_t* d_out, void* stream) {
    if (!labels_shape_ok(batch, H, W, K) || C < 1 || C > 32767) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or K");
    const long n = (long)batch * H * W;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_q || !d_node_class || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long nk = (long)batch * K;
    k_pool_node_argmax<<<(int)grid_for(nk, device), 256, 0, st>>>(d_q, nk, C, K, d_node_class);
    k_pool_paint<<<(int)grid_for(n, device), 256, 0, st>>>(d_labels, d_node_class, (long)H * W, n, K, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_pool_paint_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                          const int32_t* d_table, int16_t* d_out, void* stream) {
    if (!labels_shape_ok(batch, H, W, K)) return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    const long n = (long)batch * H * W;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_table || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    k_pool_paint<<<(int)grid_for(n, device), 256, 0, (cudaStream_t)stream>>>(d_labels, d_table, (long)H * W, n, K, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
