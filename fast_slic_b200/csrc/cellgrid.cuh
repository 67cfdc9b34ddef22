// fast_slic_b200/csrc/cellgrid.cuh -- device helpers of the seed grid and the cell grid that the u16 path
// (lab.cuh, prepare.cuh), float_slic.cuh and soft_slic.cuh share.  No kernels: any translation unit may include it.
#pragma once
#include "common.cuh"

// One channel's term of the squared feature distance: fc + (x - mu)^2, each operation rounded on its own
__device__ __forceinline__ float fs_acc(float fc, float x, float mu) {
    const float t = __fsub_rn(x, mu);
    return __fadd_rn(fc, __fmul_rn(t, t));
}

// The packed assign key of candidate k at distance d: bits(d) << 32 | k, a NaN distance having the bits 0x7fffffff, so
// the smallest key is the nearest candidate with ties to the lower k (float_slic.cuh)
__device__ __forceinline__ unsigned long long dist_key(float d, int k) {
    const uint32_t bits = isnan(d) ? 0x7fffffffu : __float_as_uint(d);
    return (unsigned long long)bits << 32 | (uint32_t)k;
}

// The seed centre (cy, cx) of cluster k on the grid of BaseContext::initialize_clusters (context.cpp:43-86): walks
// the row bands to find the band / column its index falls in (O(sqrt K)).  Also k_fs_seed's (float_slic.cuh).
__device__ __forceinline__ void init_grid_centre(int k, int H, int W, int K, int& cy_out, int& cx_out) {
    const int n_y = (int)sqrt((double)K);
    const int base_n = K / n_y, remainder = K % n_y;
    const int h = (H + n_y - 1) / n_y;
    // rows 0,2,4,.. get the first extras, then 1,3,5,.. (context.cpp:49-57)
    const int n_even = (n_y + 1) / 2;
    int acc = 0, cy = H / 2, cx = W / 2;
    bool found = false;
    for (int i = 0; i < H && !found; i += h) {
        int bi = i / h;
        if (bi > n_y - 1) bi = n_y - 1;
        int order = (bi % 2 == 0) ? (bi / 2) : (n_even + bi / 2);  // position of this row in the hand-out order
        int extra = 0;
        if (n_y == 1) extra = remainder;  // row = 1 % 1 = 0 keeps receiving (cannot happen: K % 1 == 0)
        else extra = (order < remainder) ? 1 : 0;
        const int n_x = base_n + extra;
        const int w = (W + n_x - 1) / n_x;
        const int cnt = (W + w - 1) / w;  // centres this band actually emits
        if (k < acc + cnt) {
            const int j = (k - acc) * w;
            cy = min(max(i + h / 2, 0), H - 1);
            cx = min(max(j + w / 2, 0), W - 1);
            found = true;
        }
        acc += cnt;
    }
    // k >= acc: padded with (H/2, W/2) (context.cpp:80-86)
    cy_out = cy;
    cx_out = cx;
}

// Exclusive scan of the cell histogram s_cnt[0, ncnt) by the whole block, between two barriers.  Every thread
// owns a run of consecutive cells, and one block-wide scan adds up the run totals.  Afterwards s_cnt[c] and cs[c] both
// hold the first slot of cell c: s_cnt becomes the fill pointer of the scatter, cs is the cell_start the assign kernels
// read.  s_warp holds one int per warp of the block.
__device__ __forceinline__ void scan_cells(int* s_cnt, int* s_warp, int* __restrict__ cs, int ncnt, int tid, int nt) {
    __syncthreads();
    const int per = (ncnt + nt - 1) / nt;
    const int c0 = tid * per;
    int local = 0;
    for (int u = 0; u < per; u++) {
        const int c = c0 + u;
        if (c < ncnt) local += s_cnt[c];
    }
    int x = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(FSLIC_FULL, x, o);
        if ((tid & 31) >= o) x += y;
    }
    if ((tid & 31) == 31) s_warp[tid >> 5] = x;
    __syncthreads();
    if (tid < 32) {
        const int nw = nt >> 5;
        int w = (tid < nw) ? s_warp[tid] : 0;
        int z = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(FSLIC_FULL, z, o);
            if (tid >= o) z += y;
        }
        if (tid < nw) s_warp[tid] = z - w;
    }
    __syncthreads();
    int run = s_warp[tid >> 5] + x - local;  // exclusive prefix of this thread's first cell
    for (int u = 0; u < per; u++) {
        const int c = c0 + u;
        if (c < ncnt) {
            const int v = s_cnt[c];
            s_cnt[c] = run;
            cs[c] = run;
            run += v;
        }
    }
    __syncthreads();
}
