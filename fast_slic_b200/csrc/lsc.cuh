// fast_slic_b200/csrc/lsc.cuh -- LSC (linear spectral clustering): the reference's ContextLSC (src/lsc.cpp, lsc.h)
// with num_threads = 1, the only thread count whose result is defined (DESIGN.md section 4.9).
//
// BaseContext::iterate (context.cpp:109-197) runs unchanged -- the Lab kernel, the colour re-seed, the scheduler's
// (phase, k) visiting order over the cell grid, the integer update through `acc`, connectivity enforcement -- and LSC
// overrides three hooks, each a kernel here:
//   before_iteration   k_lsc_means       the ten feature means: one serial float sum over H*W pixels per (image,
//                                        feature), all 10 B chains at once (lsc.cpp:138-150)
//                      k_lsc_features    weight w = fma chain of mean_f * feat_f, features divided by w (:151-161)
//                      k_lsc_centroids   initial centroid features over the (2 (S/4) + 1)^2 window (:165-195)
//   assign_clusters    k_assign_lsc      d = sum_f (feat_f - centroid_f)^2 over the (2S+1)^2 window (:197-224)
//   after_update       k_lsc_after_update  raster-order sums of w * feat_f and w per cluster (:226-307)
// Correctness first, in the style of realdist.cuh: every float operation is an explicit __f*_rn / __fmaf_rn intrinsic in
// the order of the reference's object code (g++ -O3 -mfma), so labels and clusters are bit-identical to it.
//
// Feature tables (lsc.cpp:69-101) are computed on the host with glibc's sincos, as the reference does, and read from
// `tab`: [0, 256) L cos, [256, 512) L sin, [512, 768) colour cos, [768, 1024) colour sin, then W x-cos, W x-sin,
// H y-cos, H y-sin.
#pragma once
#include <cfloat>
#include <climits>
#include "assign.cuh"

#define LSC_NF 10  // features: L cos, L sin, a cos, a sin, b cos, b sin, x cos, x sin, y cos, y sin (lsc.h:12)
#define LSC_CF 12  // floats per centroid record on the device (10 features, padded to three 16-byte loads)
#define LSC_TAB_FIXED 1024

__device__ __forceinline__ float lsc_raw(const float* __restrict__ tab, int H, int W, int f, uint32_t q, int i, int j) {
    switch (f) {  // lsc.cpp:107-135
        case 0: return tab[q & 0xff];
        case 1: return tab[256 + (q & 0xff)];
        case 2: return tab[512 + ((q >> 8) & 0xff)];
        case 3: return tab[768 + ((q >> 8) & 0xff)];
        case 4: return tab[512 + ((q >> 16) & 0xff)];
        case 5: return tab[768 + ((q >> 16) & 0xff)];
        case 6: return tab[LSC_TAB_FIXED + j];
        case 7: return tab[LSC_TAB_FIXED + W + j];
        case 8: return tab[LSC_TAB_FIXED + 2 * W + i];
        default: return tab[LSC_TAB_FIXED + 2 * W + H + i];
    }
}

// One warp per (image, feature): the mean is one dependent chain of H*W float adds in raster order (lsc.cpp:143-149),
// which no reassociation may shorten.  All lanes load and look up 32 * LSC_MU pixels one block ahead and stage them in
// shared memory; every lane then runs the same add chain over 16-byte broadcast reads, so the loads stay off the
// chain and the chain's latency (one FADD per pixel) is the kernel's time.
#define LSC_MU 8
__global__ void __launch_bounds__(32) k_lsc_means(const uint32_t* __restrict__ quad, const float* __restrict__ tab, int H,
                                                  int W, float* __restrict__ means) {
    __shared__ __align__(16) float buf[32 * LSC_MU];
    const int b = blockIdx.x / LSC_NF, f = blockIdx.x % LSC_NF, lane = threadIdx.x;
    const long N = (long)H * W;
    const uint32_t* q = quad + (size_t)b * N;
    auto load = [&](long base, float* v) {
#pragma unroll
        for (int u = 0; u < LSC_MU; u++) {
            const long p = base + u * 32 + lane;
            v[u] = 0.f;
            if (p < N) {
                const int i = (int)(p / W), j = (int)(p - (long)i * W);
                v[u] = lsc_raw(tab, H, W, f, __ldg(q + p), i, j);
            }
        }
    };
    float nxt[LSC_MU];
    load(0, nxt);
    float s = 0.f;
    for (long base = 0; base < N; base += 32 * LSC_MU) {
        __syncwarp();
#pragma unroll
        for (int u = 0; u < LSC_MU; u++) buf[u * 32 + lane] = nxt[u];
        __syncwarp();
        load(base + 32 * LSC_MU, nxt);  // the next block's loads are in flight during this block's chain
        const float4* b4 = reinterpret_cast<const float4*>(buf);
        if (base + 32 * LSC_MU <= N) {
#pragma unroll
            for (int t = 0; t < 8 * LSC_MU; t++) {
                const float4 v = b4[t];
                s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(s, v.x), v.y), v.z), v.w);
            }
        } else {
            for (long t = 0; t < N - base; t++) s = __fadd_rn(s, buf[t]);
        }
    }
    if (lane == 0) means[b * LSC_NF + f] = __fdiv_rn(s, (float)N);  // sum / len: int -> float, float division
}

// One thread per pixel: w = fma(mean_9, feat_9, ... fma(mean_0, feat_0, 0)) (lsc.cpp:154-160, fused by the reference's
// object code), then every feature divided by w (normalize_features, :309-316).  Writes the normalised planes
// feat [B][10][N] and w [B][N].
__global__ void __launch_bounds__(256) k_lsc_features(const uint32_t* __restrict__ quad, const float* __restrict__ tab,
                                                      int H, int W, int B, const float* __restrict__ means,
                                                      float* __restrict__ feat, float* __restrict__ wts) {
    const long N = (long)H * W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < N * B; t += (long)gridDim.x * blockDim.x) {
        const int b = (int)(t / N);
        const long p = t - (long)b * N;
        const int i = (int)(p / W), j = (int)(p - (long)i * W);
        const uint32_t q = quad[t];
        float x[LSC_NF];
        float w = 0.f;
#pragma unroll
        for (int f = 0; f < LSC_NF; f++) {
            x[f] = lsc_raw(tab, H, W, f, q, i, j);
            w = __fmaf_rn(means[b * LSC_NF + f], x[f], w);
        }
        wts[t] = w;
#pragma unroll
        for (int f = 0; f < LSC_NF; f++) feat[((size_t)b * LSC_NF + f) * N + p] = __fdiv_rn(x[f], w);
    }
}

// Per-cluster bounding box of the labels on the current pass's rows (k_assign_lsc<true> fills it, k_lsc_after_update
// reads and clears it).  Empty = {INT_MAX, INT_MAX, -1, -1}.
struct __align__(16) LscBox {
    int y0, x0, y1, x1;
};

// One thread per (image, cluster): the mean normalised feature over the window (2 (S/4) + 1)^2 around the truncated,
// unclamped centre, clamped to the image, summed in raster order; the pixel count is a float sum of 1.0f like the
// reference's (lsc.cpp:176-193) -- an empty window gives 0/0.  Also clears the cluster's bounding box.
__global__ void __launch_bounds__(256) k_lsc_centroids(const float* __restrict__ feat, int H, int W, int K, int S, int B,
                                                       const fslic_cluster* __restrict__ clusters, float* __restrict__ cf,
                                                       float* __restrict__ cf_init, LscBox* __restrict__ box) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * K) return;
    const int b = t / K;
    const long N = (long)H * W;
    const fslic_cluster c = clusters[t];
    const int cy = (int)c.y, cx = (int)c.x, r = S / 4;
    const int y_lo = max(cy - r, 0), y_hi = min(cy + r + 1, H);
    const int x_lo = max(cx - r, 0), x_hi = min(cx + r + 1, W);
    float acc[LSC_NF];
#pragma unroll
    for (int f = 0; f < LSC_NF; f++) acc[f] = 0.f;
    float cnt = 0.f;
    const float* fb = feat + (size_t)b * LSC_NF * N;
    for (int i = y_lo; i < y_hi; i++)
        for (int j = x_lo; j < x_hi; j++) {
            const long p = (long)i * W + j;
#pragma unroll
            for (int f = 0; f < LSC_NF; f++) acc[f] = __fadd_rn(acc[f], fb[(size_t)f * N + p]);
            cnt = __fadd_rn(cnt, 1.0f);
        }
#pragma unroll
    for (int f = 0; f < LSC_NF; f++) {
        const float v = __fdiv_rn(acc[f], cnt);
        cf[(size_t)t * LSC_CF + f] = v;
        cf_init[(size_t)t * LSC_NF + f] = v;
    }
    box[t] = LscBox{INT_MAX, INT_MAX, -1, -1};
}

// The LSC distance between a pixel's features x and a centroid's c: the reference's fused chain fma(diff, diff, d)
// from 0 over the ten features (lsc.cpp:212-216).  A candidate counts only if d < FLT_MAX (the reference's
// `min_dist > dist` against FLT_MAX, context.cpp:204: false for NaN -- an emptied cluster's 0/0 centroid -- and +inf);
// d >= 0, so its bits order like its value.  Used by k_assign_lsc and k_trace_pass.
__device__ __forceinline__ bool lsc_dist(const float* x, const float* c, uint32_t& bits) {
    float d = 0.f;
#pragma unroll
    for (int f = 0; f < LSC_NF; f++) {
        const float diff = __fsub_rn(x[f], c[f]);
        d = __fmaf_rn(diff, diff, d);
    }
    bits = __float_as_uint(d);
    return d < FLT_MAX;
}

// The assign pass: one thread per pixel of the pass's rows gathers over the cell grid like k_assign_real (same window
// test as its variant 0: the truncated, clamped centre of CInfo, |di|, |dj| <= S) and takes the minimum of (d, phase, k)
// with lsc_dist.  Keeping / clearing the label where no window covers the pixel is k_assign_real's rule.  UPDATE: the
// integer sums of the update and the label bounding boxes.
template <bool UPDATE>
__global__ void __launch_bounds__(256) k_assign_lsc(AssignParams ap, const uint32_t* __restrict__ quad,
                                                    uint16_t* __restrict__ labels, const CInfo* __restrict__ cinfo,
                                                    const int* __restrict__ cell_start, const float* __restrict__ feat,
                                                    const float* __restrict__ cf, unsigned long long* __restrict__ acc,
                                                    LscBox* __restrict__ box) {
    const long total = (long)ap.nsub * ap.W * ap.B;
    const int S = ap.S, W = ap.W, H = ap.H;
    const long N = (long)H * W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        int b, i, j;
        pass_pixel(ap, t, b, i, j);
        const size_t img_off = (size_t)b * N;
        const long p = (long)i * W + j;
        float x[LSC_NF];
#pragma unroll
        for (int f = 0; f < LSC_NF; f++) x[f] = feat[((size_t)b * LSC_NF + f) * N + p];
        const float4* cfb = reinterpret_cast<const float4*>(cf + (size_t)b * ap.K * LSC_CF);
        const auto dist = [&](const CInfo& r, uint32_t& d) {
            const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
            if (abs(i - cy) > S || abs(j - cx) > S) return false;
            const int k = r.sortkey & 0xffff;
            const float4 c0 = __ldg(cfb + (size_t)k * 3), c1 = __ldg(cfb + (size_t)k * 3 + 1),
                         c2 = __ldg(cfb + (size_t)k * 3 + 2);
            const float c[LSC_NF] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w, c2.x, c2.y};
            return lsc_dist(x, c, d);
        };
        const unsigned long long best =
            gather_min(ap, i, j, S, cinfo + (size_t)b * ap.K, cell_start + (size_t)b * (ap.ncell + 1), dist);
        const uint32_t label = store_label<false>(ap, best, i, labels + img_off + p);
        if (UPDATE) {
            if (label != 0xFFFF) acc_add_pixel(acc + (size_t)b * ap.K * 4, label, i, j, quad[img_off + p]);
            // bounding boxes: one set of atomics per run of equal labels in the warp (image and label together)
            const unsigned act = __activemask();
            const unsigned grp = __match_any_sync(act, ((unsigned)b << 16) | label);
            const int y0 = (int)__reduce_min_sync(grp, (unsigned)i), y1 = (int)__reduce_max_sync(grp, (unsigned)i);
            const int x0 = (int)__reduce_min_sync(grp, (unsigned)j), x1 = (int)__reduce_max_sync(grp, (unsigned)j);
            if (label != 0xFFFF && (threadIdx.x & 31) == __ffs(grp) - 1) {
                LscBox* bx = box + (size_t)b * ap.K + label;
                atomicMin(&bx->y0, y0);
                atomicMin(&bx->x0, x0);
                atomicMax(&bx->y1, y1);
                atomicMax(&bx->x1, x1);
            }
        }
    }
}

// after_update (lsc.cpp:226-307) with one thread: for each cluster, over the pixels labelled with it on the pass's rows
// in raster order, sum_f = fma(w, feat_f, sum_f) and sum_w = sum_w + w; the centroid becomes (0 + sum_f) / (0 + sum_w)
// -- 0/0 = NaN for a cluster without pixels.  Every cluster is updatable here (`preemptive` is not combined with LSC).
// One warp per (image, cluster) walks the cluster's bounding box: lanes read 32 labels of a row, the matching pixels'
// weight and features go through shared memory, and lane f < 10 keeps sum_f, lane 10 sum_w -- one accumulator per
// lane, no float atomics.  Clears the box for the next pass.
#define LSC_AU_WARPS 8
__global__ void __launch_bounds__(LSC_AU_WARPS * 32) k_lsc_after_update(int H, int W, int K, int B, int stride,
                                                                        const uint16_t* __restrict__ labels,
                                                                        const float* __restrict__ feat,
                                                                        const float* __restrict__ wts,
                                                                        float* __restrict__ cf, LscBox* __restrict__ box) {
    __shared__ float sm[LSC_AU_WARPS][LSC_NF + 1][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * LSC_AU_WARPS + warp;
    if (t >= B * K) return;
    const int b = t / K, k = t - b * K;
    const long N = (long)H * W;
    const LscBox bx = box[t];
    float a = 0.f;
    for (int i = bx.y0; i <= bx.y1; i += stride) {
        const size_t row = (size_t)b * N + (size_t)i * W;
        for (int x = bx.x0; x <= bx.x1; x += 32) {
            const int j = x + lane;
            const bool in = j <= bx.x1 && labels[row + j] == (uint16_t)k;
            const unsigned m = __ballot_sync(FSLIC_FULL, in);
            if (!m) continue;
            if (in) {
                const long p = (long)i * W + j;
                sm[warp][LSC_NF][lane] = wts[row + j];
#pragma unroll
                for (int f = 0; f < LSC_NF; f++) sm[warp][f][lane] = feat[((size_t)b * LSC_NF + f) * N + p];
            }
            __syncwarp();
            for (unsigned mm = m; mm; mm &= mm - 1) {
                const int s = __ffs(mm) - 1;
                const float w = sm[warp][LSC_NF][s];
                if (lane < LSC_NF)
                    a = __fmaf_rn(w, sm[warp][lane][s], a);
                else if (lane == LSC_NF)
                    a = __fadd_rn(a, w);
            }
            __syncwarp();
        }
    }
    const float wsum = __fadd_rn(0.f, __shfl_sync(FSLIC_FULL, a, LSC_NF));
    if (lane < LSC_NF) cf[(size_t)t * LSC_CF + lane] = __fdiv_rn(__fadd_rn(0.f, a), wsum);
    if (lane == 0) box[t] = LscBox{INT_MAX, INT_MAX, -1, -1};
}
