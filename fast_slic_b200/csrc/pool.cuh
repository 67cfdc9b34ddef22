// fast_slic_b200/csrc/pool.cuh -- superpixel pooling over a batch of label maps (DESIGN.md section 4.12): per-superpixel
// sums / means of float feature maps, the gather back to pixels (unpool) and the per-pixel class of a per-superpixel
// score table (paint_argmax).  No counterpart in the reference.  No float atomics: every image's sums are added in one
// fixed order that depends on nothing but that image's labels and features.
//
// Summation order of the sum over superpixel k of image b (the members of k in raster order m_0, m_1, ...):
//   lane l of one warp adds m_l, m_{l+32}, m_{l+64}, ... left to right, starting from +0.0;
//   then five butterfly steps, for o = 16, 8, 4, 2, 1: v_l = v_l + v_{l xor o} (addition commutes, so the 32 lanes hold
//   the same value after every step); the result is lane 0's value.
// The members come in raster order out of one stable radix sort of the keys (image << 16 | label) with the pixel index
// as the value.  A label outside [0, K) gets the label 0xffff, which no superpixel has (K <= 65534), and is dropped.
#pragma once
#include "common.cuh"

#define POOL_NO_LABEL 0xffffu

// keys[t] = (image in the call << 16) | label (0xffff outside [0, K)), vals[t] = the pixel index in its image, over the
// n = batch * hw pixels of the call
__global__ void __launch_bounds__(256) k_pool_keys(const uint16_t* __restrict__ lab, long hw, long n, int K,
                                                    uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const long b = t / hw;
        const uint32_t l = lab[t];
        keys[t] = (uint32_t)b << 16 | (l < (uint32_t)K ? l : POOL_NO_LABEL);
        vals[t] = (uint32_t)(t - b * hw);
    }
}

// Segment bounds of the sorted keys: seg_start / seg_end [batch * K] (zeroed before, so an empty superpixel is [0, 0))
// receive the first and one-past-last sorted position of each (image, label).
__global__ void __launch_bounds__(256) k_pool_bounds(const uint32_t* __restrict__ skey, long n, int K,
                                                      uint32_t* __restrict__ seg_start, uint32_t* __restrict__ seg_end) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const uint32_t key = skey[i];
        const uint32_t l = key & 0xffffu;
        if (l == POOL_NO_LABEL) continue;
        const long seg = (long)(key >> 16) * K + l;
        if (i == 0 || skey[i - 1] != key) seg_start[seg] = (uint32_t)i;
        if (i == n - 1 || skey[i + 1] != key) seg_end[seg] = (uint32_t)(i + 1);
    }
}

// The butterfly over the warp's 32 lane sums, then lane 0 writes the sum or the mean to *o
__device__ __forceinline__ void pool_finish(float acc, int lane, uint32_t cnt, float fcnt, int mean, float* o) {
#pragma unroll
    for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(FSLIC_FULL, acc, off);
    if (lane == 0) *o = mean ? (cnt ? __fdiv_rn(acc, fcnt) : 0.0f) : acc;
}

// One warp per (image, label) segment, nseg = batch * K: out [batch, C, K] = the sum in the order above, or with `mean`
// sum / (float)count (one correctly rounded division, count converted round-to-nearest; 0 for an empty superpixel);
// counts [batch, K] = the segment's length.  members: the sorted pixel indices; feat [batch, C, hw].
__global__ void __launch_bounds__(256) k_pool_segments(const uint32_t* __restrict__ seg_start,
                                                        const uint32_t* __restrict__ seg_end,
                                                        const uint32_t* __restrict__ members,
                                                        const float* __restrict__ feat, long nseg, int K, int C, long hw,
                                                        int mean, float* __restrict__ out, int32_t* __restrict__ counts) {
    const long seg = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (seg >= nseg) return;  // the whole warp leaves together
    const long b = seg / K, k = seg - b * K;
    const uint32_t s = seg_start[seg], e = seg_end[seg];
    const uint32_t cnt = e - s;
    if (lane == 0) counts[seg] = (int32_t)cnt;
    const float fcnt = __uint2float_rn(cnt);
    const float* f = feat + b * C * hw;
    float* o = out + b * C * K + k;
    // four channels per pass over the members (one index load feeds four gathers), then the rest one at a time; each
    // channel's accumulator sees the same sequence either way
    int c = 0;
    for (; c + 4 <= C; c += 4) {
        const float* fc = f + (long)c * hw;
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll 2
        for (uint32_t i = s + lane; i < e; i += 32) {
            const uint32_t m = members[i];
#pragma unroll
            for (int u = 0; u < 4; u++) acc[u] += __ldg(fc + u * hw + m);
        }
#pragma unroll
        for (int u = 0; u < 4; u++) pool_finish(acc[u], lane, cnt, fcnt, mean, o + (long)(c + u) * K);
    }
    for (; c < C; c++) {
        const float* fc = f + (long)c * hw;
        float acc = 0.0f;
#pragma unroll 4
        for (uint32_t i = s + lane; i < e; i += 32) acc += __ldg(fc + members[i]);
        pool_finish(acc, lane, cnt, fcnt, mean, o + (long)c * K);
    }
}

// out [batch, C, hw] = values [batch, C, K] at each pixel's label, divided by (float)divisor[b, label] when divisor is
// given (the backward of the mean); 0 where the label is outside [0, K).  One pixel per thread, all channels.
__global__ void __launch_bounds__(256) k_pool_unpool(const uint16_t* __restrict__ lab, const float* __restrict__ values,
                                                      const int32_t* __restrict__ divisor, long hw, long n, int C, int K,
                                                      float* __restrict__ out) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const long b = t / hw, p = t - b * hw;
        const uint32_t l = lab[t];
        float* o = out + b * C * hw + p;
        if (l >= (uint32_t)K) {
            for (int c = 0; c < C; c++) o[(long)c * hw] = 0.0f;
            continue;
        }
        const float* v = values + b * C * K + l;
        if (divisor) {
            const float d = __int2float_rn(divisor[b * K + l]);
            for (int c = 0; c < C; c++) o[(long)c * hw] = __fdiv_rn(__ldg(v + (long)c * K), d);
        } else {
            for (int c = 0; c < C; c++) o[(long)c * hw] = __ldg(v + (long)c * K);
        }
    }
}

// cls [batch, K] = the first index of the maximum of q[b, :, k] over C, a NaN counting as the maximum (torch.argmax)
__global__ void __launch_bounds__(256) k_pool_node_argmax(const float* __restrict__ q, long nk, int C, int K,
                                                           int32_t* __restrict__ cls) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nk; t += (long)gridDim.x * blockDim.x) {
        const long b = t / K, k = t - b * K;
        const float* qq = q + b * C * K + k;
        float best = qq[0];
        int bi = 0;
        for (int c = 1; c < C && !isnan(best); c++) {
            const float v = qq[(long)c * K];
            if (isnan(v) || v > best) {
                best = v;
                bi = c;
            }
        }
        cls[t] = bi;
    }
}

// out [batch, hw] = cls[b, label] of each pixel, -1 where the label is outside [0, K)
__global__ void __launch_bounds__(256) k_pool_paint(const uint16_t* __restrict__ lab, const int32_t* __restrict__ cls,
                                                     long hw, long n, int K, int16_t* __restrict__ out) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const uint32_t l = lab[t];
        out[t] = l < (uint32_t)K ? (int16_t)cls[t / hw * K + l] : (int16_t)-1;
    }
}
