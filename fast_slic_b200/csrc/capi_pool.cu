// fast_slic_b200/csrc/capi_pool.cu -- the extern "C" entry points of superpixel pooling (pool.cuh): pool, unpool,
// paint_argmax and paint over a batch of label maps.  Stateless (device pointers, caller-provided scratch), asynchronous
// on the caller's stream, never synchronise.
#include <limits.h>

#include <cub/device/device_radix_sort.cuh>

#include "capi_common.h"
#include "pool.cuh"

static size_t pool_sort_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)items, 0, 32);
    return bytes;
}

static bool pool_shape_ok(int batch, int H, int W, int K) {
    return batch >= 0 && H >= 0 && W >= 0 && K >= 1 && K <= 65534;
}

// Keys, pixel indices and their sorted copies (4 bytes each per pixel), the segment bounds (8 bytes per superpixel)
// and the sort's temporary storage (sized for all 32 key bits).
extern "C" size_t fslic_b200_pool_batch_scratch_bytes(int batch, int H, int W, int K) {
    if (!pool_shape_ok(batch, H, W, K)) return (size_t)-1;
    const long long n = (long long)batch * H * W;
    if (n == 0) return 256;
    if (n > INT_MAX || batch > 65536) return (size_t)-1;  // one radix sort of 32-bit keys: split the batch
    const size_t nk = (size_t)batch * K;
    return align_up((size_t)n * 4, 256) * 4 + align_up(nk * 4, 256) * 2 + align_up(pool_sort_temp_bytes(n), 256);
}

extern "C" int fslic_b200_pool_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                     const float* d_features, int mean, float* d_out, int32_t* d_counts, void* d_scratch,
                                     size_t scratch_bytes, void* stream) {
    if (!pool_shape_ok(batch, H, W, K) || C < 1) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or K");
    const long long n = (long long)batch * H * W;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_features || !d_out || !d_counts || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_pool_batch_scratch_bytes(batch, H, W, K);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long hw = (long)H * W, nk = (long)batch * K;
    unsigned char* p = static_cast<unsigned char*>(d_scratch);
    uint32_t* key = reinterpret_cast<uint32_t*>(p); p += align_up((size_t)n * 4, 256);
    uint32_t* skey = reinterpret_cast<uint32_t*>(p); p += align_up((size_t)n * 4, 256);
    uint32_t* val = reinterpret_cast<uint32_t*>(p); p += align_up((size_t)n * 4, 256);
    uint32_t* sval = reinterpret_cast<uint32_t*>(p); p += align_up((size_t)n * 4, 256);
    uint32_t* seg_start = reinterpret_cast<uint32_t*>(p); p += align_up((size_t)nk * 4, 256);
    uint32_t* seg_end = reinterpret_cast<uint32_t*>(p); p += align_up((size_t)nk * 4, 256);
    size_t temp_bytes = align_up(pool_sort_temp_bytes(n), 256);
    void* temp = p;
    const int bits = 16 + bit_length((unsigned long long)(batch - 1));
    size_t temp_used = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, temp_used, key, skey, val, sval, (int)n, 0, bits, st);
    if (temp_used > temp_bytes) return set_err(FSLIC_ECUDA, "radix sort temporary storage");
    k_pool_keys<<<(int)grid_for(n, device), 256, 0, st>>>(d_labels, hw, n, K, key, val);
    if (cub::DeviceRadixSort::SortPairs(temp, temp_bytes, key, skey, val, sval, (int)n, 0, bits, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the pixel keys failed");
    CK(cudaMemsetAsync(seg_start, 0, (size_t)nk * 4, st));
    CK(cudaMemsetAsync(seg_end, 0, (size_t)nk * 4, st));
    k_pool_bounds<<<(int)grid_for(n, device), 256, 0, st>>>(skey, n, K, seg_start, seg_end);
    k_pool_segments<<<(unsigned)((nk + 7) / 8), 256, 0, st>>>(seg_start, seg_end, sval, d_features, nk, K, C, hw, mean ? 1 : 0,
                                                             d_out, d_counts);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_pool_unpool_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                            const float* d_values, const int32_t* d_divisor, float* d_out, void* stream) {
    if (!pool_shape_ok(batch, H, W, K) || C < 1) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or K");
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
    if (!pool_shape_ok(batch, H, W, K) || C < 1 || C > 32767) return set_err(FSLIC_EINVAL, "bad batch, H, W, C or K");
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
    if (!pool_shape_ok(batch, H, W, K)) return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    const long n = (long)batch * H * W;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_table || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    k_pool_paint<<<(int)grid_for(n, device), 256, 0, (cudaStream_t)stream>>>(d_labels, d_table, (long)H * W, n, K, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
