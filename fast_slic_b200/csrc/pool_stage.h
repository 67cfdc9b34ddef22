// fast_slic_b200/csrc/pool_stage.h -- the sort-and-sum stage of superpixel pooling (capi_pool.cu, kernels in
// pool.cuh) for the translation units that pool their own (image, label) keys: one stable radix sort of the keys with
// the pixel indices as values, the segment bounds, then k_pool_segments.  So every pooled sum in the library has one
// summation order (DESIGN.md section 4.12).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <cuda_runtime.h>

// Keys, pixel indices and their sorted copies (4 bytes each per key), the segment bounds (8 bytes per superpixel)
// and the sort's temporary storage (sized for all 32 key bits).
struct PoolScratch {
    uint32_t *key, *skey, *val, *sval, *seg_start, *seg_end;
    void* temp;
    size_t temp_bytes, total;
};

// The layout for up to n keys over nk = batch * K superpixels from `base` (null: sizes only, in .total)
PoolScratch pool_layout(long long n, long long nk, void* base);

// s.key / s.val hold n keys (image << 16 | label, 0xffff for no superpixel) and pixel indices, in raster order inside
// each image: out [batch, C, K] = the sums (or with `mean` the means) over feat [batch, C, hw], counts [batch, K].
// n may be 0 (every superpixel empty).  n <= INT_MAX, batch <= 65536.
int pool_sorted_segments(const PoolScratch& s, long long n, int batch, int K, int C, long hw, const float* feat,
                         int mean, float* out, int32_t* counts, int device, cudaStream_t st);
