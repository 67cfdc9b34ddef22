// crf_feed.cuh -- the SimpleCRF's per-frame input built on the device (capi_crf.cu's fslic_b200_crfdev_* entry points):
// cluster records, adjacency CSR and unaries, each equal bit for bit to what the host path (SimpleCRF.push_slic_frame
// and the unary setters of fast_slic_b200/crf.py, capi_crf.cu's fslic_b200_crf_*) stores for the same input.
// Defines non-inline kernels: include it (and crf.cuh) from capi_crf.cu only.
#pragma once
#include <stdint.h>
#include <cub/block/block_scan.cuh>
#include "common.cuh"
#include "glibc_logf.cuh"
#include "crf.cuh"

// numpy's float64 -> int32 cast on x86 (cvttsd2si): truncation, and INT_MIN for NaN, ±inf and anything whose truncation
// is outside the int32 range.  CUDA's conversion saturates and maps NaN to 0, so those cases are spelled out.
__device__ __forceinline__ int32_t feed_x86_trunc_i32(double d) {
    return d > -2147483649.0 && d < 2147483648.0 ? (int32_t)d : INT32_MIN;
}

// push_slic_frame's records: to_yxmrgb() (float64) .astype(np.int32), then set_yxmrgb stores y, x, r, g, b as float32
// (round to nearest) and num_members as uint32 (wrapping), `number` = index as uint16, every other field zero.
__device__ __forceinline__ float feed_coord(float v) { return __int2float_rn(feed_x86_trunc_i32((double)v)); }

// The destinations of up to CRF_GROUP_MAX pushed frames (crf.cuh), blockIdx.y = frame of the launch.
struct FeedFramePtrs {
    fslic_cluster* clusters;
    float *unary, *q0, *q1;
    int32_t *offsets, *nbr;
};
struct FeedFrameSet {
    FeedFramePtrs f[CRF_GROUP_MAX];
};

// One thread per node of each frame: records src[blockIdx.y] ([N]) go to frame blockIdx.y.  Also fills the frame's
// unaries with `unbiased` (set_unbiased: logf(C), the host's constant) and zeroes both q buffers, as push_frame does.
__global__ void __launch_bounds__(256) k_feed_nodes(const fslic_cluster* __restrict__ src,
                                                    const __grid_constant__ FeedFrameSet dst, int N, int C,
                                                    float unbiased) {
    const FeedFramePtrs& d = dst.f[blockIdx.y];
    src += (long long)blockIdx.y * N;
    const long long CN = (long long)C * N;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < CN || t < N;
         t += (long long)gridDim.x * blockDim.x) {
        if (t < N) {
            const fslic_cluster s = src[t];
            fslic_cluster o;
            o.y = feed_coord(s.y);
            o.x = feed_coord(s.x);
            o.r = feed_coord(s.r);
            o.g = feed_coord(s.g);
            o.b = feed_coord(s.b);
            o.a = 0.0f;
            o.number = (uint16_t)t;
            o.is_active = 0;
            o.is_updatable = 0;
            o.num_members = (uint32_t)feed_x86_trunc_i32((double)s.num_members);
            d.clusters[t] = o;
        }
        if (t < CN) {
            d.unary[t] = unbiased;
            d.q0[t] = 0.0f;
            d.q1[t] = 0.0f;
        }
    }
}

// counts[K] / neighbors[K][12] of graph blockIdx.y of the batch -> frame blockIdx.y's CSR: offsets = exclusive scan of
// the counts, the neighbours row by row in list order (what set_connectivity makes of a NodeConnectivity).  One CTA of
// FEED_CSR_THREADS per frame; thread t owns the contiguous rows [t * per, (t + 1) * per).
#define FEED_CSR_THREADS 1024
__global__ void __launch_bounds__(FEED_CSR_THREADS) k_feed_csr(const int32_t* __restrict__ counts,
                                                               const uint32_t* __restrict__ neighbors, int K,
                                                               const __grid_constant__ FeedFrameSet dst) {
    typedef cub::BlockScan<int, FEED_CSR_THREADS> Scan;
    __shared__ typename Scan::TempStorage scan_tmp;
    counts += (long long)blockIdx.y * K;
    neighbors += (long long)blockIdx.y * K * CONN_MAX;
    int32_t* __restrict__ offsets = dst.f[blockIdx.y].offsets;
    int32_t* __restrict__ nbr = dst.f[blockIdx.y].nbr;
    const int per = (K + FEED_CSR_THREADS - 1) / FEED_CSR_THREADS;
    const int r0 = min(K, (int)threadIdx.x * per), r1 = min(K, r0 + per);
    int own = 0;
    for (int i = r0; i < r1; i++) own += counts[i];
    int base;
    Scan(scan_tmp).ExclusiveSum(own, base);
    if (threadIdx.x == 0) offsets[0] = 0;
    for (int i = r0; i < r1; i++) {
        const int n = counts[i];
        for (int v = 0; v < n; v++) nbr[base + v] = (int32_t)neighbors[(long long)i * CONN_MAX + v];
        base += n;
        offsets[i + 1] = base;
    }
}

// set_proba of frame blockIdx.y from p[blockIdx.y] (n = C * N values each): unary = -logf(p), glibc's logf and x86's
// sign flip.  Only the unary pointers of the set are used.
__global__ void __launch_bounds__(256) k_feed_proba(const float* __restrict__ p, const __grid_constant__ CrfFrameQSet set,
                                                    long long n) {
    float* __restrict__ unary = set.f[blockIdx.y].unary;
    p += (long long)blockIdx.y * n;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
        unary[k] = glogf::neg_logf(p[k]);
}

// set_mask, first launch: *bad = 1 if any class is outside [0, C) (*bad is zeroed before)
__global__ void __launch_bounds__(256) k_feed_mask_check(const int32_t* __restrict__ classes, int N, int C, int* bad) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x)
        if (classes[i] < 0 || classes[i] >= C) *bad = 1;
}

// set_mask, second launch: every (class, node) gets the inactive unary, node i's own class the active one
__global__ void __launch_bounds__(256) k_feed_mask(const int32_t* __restrict__ classes, int N, int C, float active_unary,
                                                   float inactive_unary, float* __restrict__ unary) {
    const long long CN = (long long)C * N;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < CN; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k % N), c = (int)(k / N);
        unary[k] = classes[i] == c ? active_unary : inactive_unary;
    }
}

__global__ void k_logf_debug(uint32_t first, long long n, float* out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = glogf::logf(__uint_as_float(first + (uint32_t)i));
}
