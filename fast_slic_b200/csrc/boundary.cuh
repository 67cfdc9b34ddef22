// fast_slic_b200/csrc/boundary.cuh -- statistics of pixel maps along the shared boundaries of region adjacency edges
// (DESIGN.md section 4.17): per graph entry and channel, the mean, min and max of the values at both ends of every
// boundary pixel pair of the entry's two labels, and the number of such pairs.  No counterpart in the reference.  No
// float atomics: each statistic is computed by one warp in one fixed order.
//
// Pixel pairs are those of region adjacency (rag.cuh): the right and down neighbour, with connectivity 8 also the
// down-right and down-left one.  Slot s = t * D + d (D = 2 or 4) is direction d of the call's pixel t = b * hw + p, so
// slots increase with (image, pair ordinal p * D + d).  One call runs in two steps, with one host read between them:
//   select      the boundary slots (both labels in [0, K) and different), in slot order (cub::DeviceSelect::If, which
//               keeps the order), and their number, which the caller reads back;
//   stats       k_boundary_keys       the key (image << 32 | lo << 16 | hi) of each selected slot;
//               (stable radix sort of the keys, the slot as the value: each key's pairs stay in ordinal order)
//               k_boundary_heads      flags the positions where the key changes;
//               (cub::DeviceSelect::Flagged of those positions: the start of every run of one key)
//               k_boundary_entry_keys the same key for each graph entry whose image is in the call, all ones otherwise;
//               (radix sort of the entry keys, the entry index as the value)
//               k_boundary_init       (the first call of a batch only) NaN and a count of 0 in every row;
//               k_boundary_runs       one warp per run: the entries with its key (two binary searches), then per
//                                     channel the sum, min and max of the run's 2n values, written to those entries.
// Summation order of a run (pool.cuh's): value j of the run is the anchor (j even) or the other pixel (j odd) of pair
// j / 2; lane l adds values l, l + 32, ... left to right from +0.0, five butterfly steps combine the lanes, and the mean
// is lane 0's sum / (float)(2n).  min / max use the total order of non-NaN floats with -0.0 < +0.0 (as ordered ints);
// any NaN makes them NaN.
#pragma once
#include <limits.h>

#include "common.cuh"

#define BOUNDARY_NO_KEY 0xffffffffffffffffull

// Neighbour offset of direction d inside an image of width W: right, down, down-right, down-left
__device__ __forceinline__ int boundary_offset(int d, int W) {
    return d == 0 ? 1 : (d == 1 ? W : (d == 2 ? W + 1 : W - 1));
}

// The predicate of the select: slot s is a pixel pair whose two labels are in [0, K) and differ
struct BoundaryPair {
    const uint16_t* lab;
    uint32_t hw, W, H, K;
    int shift;  // log2 D
    __device__ __forceinline__ bool operator()(uint32_t s) const {
        const uint32_t t = s >> shift, d = s & ((1u << shift) - 1);
        const uint32_t p = t % hw, i = p / W, j = p - i * W;
        const uint32_t di = d == 0 ? 0 : 1;
        if (i + di >= H) return false;
        if ((d == 0 || d == 2) && j + 1 >= W) return false;
        if (d == 3 && j == 0) return false;
        const uint32_t a = lab[t];
        if (a >= K) return false;
        const uint32_t g = lab[t + boundary_offset((int)d, (int)W)];
        return g < K && g != a;
    }
};

// head[i] = 1 where position i of the sorted keys begins a run of one key, else 0
__global__ void __launch_bounds__(256) k_boundary_heads(const unsigned long long* __restrict__ skey, long pairs,
                                                         uint8_t* __restrict__ head) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += (long)gridDim.x * blockDim.x)
        head[i] = i == 0 || skey[i] != skey[i - 1];
}

// key[i] = (image in the call) << 32 | lo << 16 | hi of selected slot sel[i]
__global__ void __launch_bounds__(256) k_boundary_keys(const uint32_t* __restrict__ sel, long pairs,
                                                        const uint16_t* __restrict__ lab, uint32_t hw, int W, int shift,
                                                        unsigned long long* __restrict__ key) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += (long)gridDim.x * blockDim.x) {
        const uint32_t s = sel[i], t = s >> shift, d = s & ((1u << shift) - 1);
        const uint32_t a = lab[t], g = lab[t + boundary_offset((int)d, W)];
        key[i] = (unsigned long long)(t / hw) << 32 | (a < g ? a << 16 | g : g << 16 | a);
    }
}

// ekey[e] = the key of entry (src[e], dst[e]) when both are nodes of one image in [image_base, image_base + batch) and
// differ, all ones otherwise; eidx[e] = e
__global__ void __launch_bounds__(256) k_boundary_entry_keys(const long long* __restrict__ src,
                                                              const long long* __restrict__ dst, long long edges,
                                                              long long nodes, int K, long long image_base, int batch,
                                                              unsigned long long* __restrict__ ekey,
                                                              uint32_t* __restrict__ eidx) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < edges; e += (long long)gridDim.x * blockDim.x) {
        const long long u = src[e], v = dst[e];
        unsigned long long key = BOUNDARY_NO_KEY;
        if (u >= 0 && v >= 0 && u < nodes && v < nodes && u != v) {
            const long long b = u / K;
            if (v / K == b && b >= image_base && b < image_base + batch) {
                const uint32_t lu = (uint32_t)(u - b * K), lv = (uint32_t)(v - b * K);
                key = (unsigned long long)(b - image_base) << 32 | (lu < lv ? lu << 16 | lv : lv << 16 | lu);
            }
        }
        ekey[e] = key;
        eidx[e] = (uint32_t)e;
    }
}

// mean, min, max [edges, C] = NaN, count [edges] = 0
__global__ void __launch_bounds__(256) k_boundary_init(long long edges, int C, float* __restrict__ mean,
                                                        float* __restrict__ mn, float* __restrict__ mx,
                                                        int32_t* __restrict__ count) {
    const float nan = __int_as_float(0x7fffffff);
    const long long n = edges * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        mean[i] = nan;
        mn[i] = nan;
        mx[i] = nan;
        if (i < edges) count[i] = 0;
    }
}

// The total order of non-NaN floats, -0.0 < +0.0, as signed ints (an involution: it also maps back)
__device__ __forceinline__ int boundary_okey(int i) { return i ^ ((i >> 31) & 0x7fffffff); }

// First position of sorted keys [0, n) that is >= key
__device__ __forceinline__ int boundary_lower_bound(const unsigned long long* __restrict__ k, int n,
                                                    unsigned long long key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
        if (k[mid] < key)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}

// The butterfly sum, the warp min / max and the NaN flag of one channel -> (mean, min, max)
__device__ __forceinline__ void boundary_finish(float acc, int lo, int hi, bool nan, float f2n, float* m, float* a,
                                                float* b) {
#pragma unroll
    for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(FSLIC_FULL, acc, off);
    lo = __reduce_min_sync(FSLIC_FULL, lo);
    hi = __reduce_max_sync(FSLIC_FULL, hi);
    const bool any_nan = __any_sync(FSLIC_FULL, nan);
    *m = __fdiv_rn(acc, f2n);
    *a = any_nan ? __int_as_float(0x7fffffff) : __int_as_float(boundary_okey(lo));
    *b = any_nan ? __int_as_float(0x7fffffff) : __int_as_float(boundary_okey(hi));
}

__device__ __forceinline__ void boundary_add(float v, float& acc, int& lo, int& hi, bool& nan) {
    acc += v;
    if (isnan(v)) {
        nan = true;
    } else {
        const int k = boundary_okey(__float_as_int(v));
        lo = min(lo, k);
        hi = max(hi, k);
    }
}

// Persistent warps over the runs: run r (of *d_runs) is sorted positions [start[r], start[r + 1] or pairs); its
// entries are the sorted entry positions [m0, m1) with its key.  values [batch, C, hw] of the call's images.
__global__ void __launch_bounds__(256) k_boundary_runs(const unsigned long long* __restrict__ skey,
                                                        const uint32_t* __restrict__ sslot,
                                                        const uint32_t* __restrict__ start, const int* __restrict__ d_runs,
                                                        int pairs, const unsigned long long* __restrict__ sekey,
                                                        const uint32_t* __restrict__ seidx, int edges,
                                                        const float* __restrict__ values, int C, uint32_t hw, int W,
                                                        int shift, float* __restrict__ mean, float* __restrict__ mn,
                                                        float* __restrict__ mx, int32_t* __restrict__ count) {
    const int lane = threadIdx.x & 31;
    const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    const int runs = *d_runs;
    const uint32_t dmask = (1u << shift) - 1;
    for (long r = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < runs; r += nwarps) {
        const int s = (int)start[r], e = r + 1 < runs ? (int)start[r + 1] : pairs;
        const unsigned long long key = skey[s];
        // lane 0: the first entry with the key, lane 1: the first after them
        int pos = 0;
        if (lane < 2) pos = boundary_lower_bound(sekey, edges, key + (unsigned long long)lane);
        const int m0 = __shfl_sync(FSLIC_FULL, pos, 0), m = __shfl_sync(FSLIC_FULL, pos, 1) - m0;
        if (m == 0) continue;  // no entry asks for this boundary (the whole warp skips it)
        const uint32_t n = (uint32_t)(e - s), nv = 2 * n;
        const float f2n = __uint2float_rn(nv);
        const uint32_t base = (uint32_t)(key >> 32) * hw;
        const float* f = values + (long)(key >> 32) * C * hw;
        for (int k = lane; k < m; k += 32) count[seidx[m0 + k]] = (int32_t)n;
        int c = 0;
        // four channels per pass over the pairs (one slot load feeds four gathers), then the rest one at a time; each
        // channel's accumulators see the same sequence either way
        for (; c + 4 <= C; c += 4) {
            const float* fc = f + (long)c * hw;
            float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
            int lo[4] = {INT_MAX, INT_MAX, INT_MAX, INT_MAX}, hi[4] = {INT_MIN, INT_MIN, INT_MIN, INT_MIN};
            bool nan[4] = {false, false, false, false};
            for (uint32_t j = lane; j < nv; j += 32) {
                const uint32_t slot = sslot[s + (j >> 1)], t = slot >> shift;
                const uint32_t p = t - base + ((j & 1) ? boundary_offset((int)(slot & dmask), W) : 0);
#pragma unroll
                for (int u = 0; u < 4; u++) boundary_add(__ldg(fc + (long)u * hw + p), acc[u], lo[u], hi[u], nan[u]);
            }
            float rm[4], ra[4], rb[4];
#pragma unroll
            for (int u = 0; u < 4; u++) boundary_finish(acc[u], lo[u], hi[u], nan[u], f2n, &rm[u], &ra[u], &rb[u]);
            // lane 4 k + u writes channel c + u of the k-th entry
            for (int q = lane; q < 4 * m; q += 32) {
                const int u = q & 3;
                const long o = (long)seidx[m0 + (q >> 2)] * C + c + u;
                mean[o] = u == 0 ? rm[0] : u == 1 ? rm[1] : u == 2 ? rm[2] : rm[3];
                mn[o] = u == 0 ? ra[0] : u == 1 ? ra[1] : u == 2 ? ra[2] : ra[3];
                mx[o] = u == 0 ? rb[0] : u == 1 ? rb[1] : u == 2 ? rb[2] : rb[3];
            }
        }
        for (; c < C; c++) {
            const float* fc = f + (long)c * hw;
            float acc = 0.0f;
            int lo = INT_MAX, hi = INT_MIN;
            bool nan = false;
            for (uint32_t j = lane; j < nv; j += 32) {
                const uint32_t slot = sslot[s + (j >> 1)], t = slot >> shift;
                const uint32_t p = t - base + ((j & 1) ? boundary_offset((int)(slot & dmask), W) : 0);
                boundary_add(__ldg(fc + p), acc, lo, hi, nan);
            }
            float rm, ra, rb;
            boundary_finish(acc, lo, hi, nan, f2n, &rm, &ra, &rb);
            for (int k = lane; k < m; k += 32) {
                const long o = (long)seidx[m0 + k] * C + c;
                mean[o] = rm;
                mn[o] = ra;
                mx[o] = rb;
            }
        }
    }
}

// ---- Volumes (DESIGN.md section 4.24): label volumes u16 [batch, D, H, W] and values f32 [batch, C, D, H, W], the
// voxel pairs of region adjacency (rag.cuh's k_rag3d_discover): each voxel (the anchor) with its forward neighbours
// (dz, dy, dx) of BOUNDARY3D_DIRS, the first 3 (connectivity 6), 9 (18) or 13 (26).  Pair ordinal = anchor * Ndir + d.
// The selection is sized per voxel, not per voxel pair:
//   select      k_boundary3d_mask     a 13-bit mask of each voxel's boundary directions (2 bytes per voxel);
//               (cub::DeviceSelect::Flagged of the voxels with a mask, in voxel order, 4 bytes per voxel, and
//               cub::DeviceReduce::Sum of popc(mask): the caller reads back the voxel count and the pair count)
//   stats       (cub::DeviceScan::ExclusiveSum of popc(mask) over the selected voxels: each voxel's first pair)
//               k_boundary3d_expand   one record per boundary pair in ordinal order: key, position, anchor, direction;
//               (stable radix sort of the keys, the position as the value; then the 2-D heads, run starts and entry
//               keys above)
//               k_boundary3d_runs     k_boundary_runs with the other voxel at anchor + off[d].
// Every forward offset dz * H * W + dy * W + dx of a pair that exists is positive.
struct Boundary3dDirs {
    int off[13];  // dz * H * W + dy * W + dx of each direction, host-built for the call's H, W
};

__device__ __forceinline__ int boundary3d_dir(int d, int a) {
    constexpr int8_t dirs[13][3] = {{0, 0, 1}, {0, 1, 0},  {1, 0, 0},  {0, 1, 1},  {0, 1, -1},
                                    {1, 1, 0}, {1, -1, 0}, {1, 0, 1},  {1, 0, -1}, {1, 1, 1},
                                    {1, 1, -1}, {1, -1, 1}, {1, -1, -1}};
    return dirs[d][a];
}

// mask[t] = bit d set where voxel t's pair in direction d exists, both labels are in [0, K) and they differ
template <int NDIR>
__global__ void __launch_bounds__(256) k_boundary3d_mask(const uint16_t* __restrict__ lab, uint32_t dhw, int D, int H,
                                                          int W, uint32_t n, int K, Boundary3dDirs dirs,
                                                          uint16_t* __restrict__ mask) {
    const uint32_t hw = (uint32_t)H * (uint32_t)W;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const uint32_t p = t % dhw, z = p / hw, r = p - z * hw, y = r / (uint32_t)W, x = r - y * (uint32_t)W;
        const uint32_t s = lab[t];
        uint32_t m = 0;
        if (s < (uint32_t)K) {
#pragma unroll
            for (int d = 0; d < NDIR; d++) {
                const int dz = boundary3d_dir(d, 0), dy = boundary3d_dir(d, 1), dx = boundary3d_dir(d, 2);
                if ((int)z + dz < D && (int)y + dy >= 0 && (int)y + dy < H && (int)x + dx >= 0 && (int)x + dx < W) {
                    const uint32_t g = lab[t + dirs.off[d]];
                    if (g < (uint32_t)K && g != s) m |= 1u << d;
                }
            }
        }
        mask[t] = (uint16_t)m;
    }
}

// counts[0] = the selected voxel count (the pair sum writes counts[1])
__global__ void k_boundary3d_count(const int* __restrict__ nsel, long long* __restrict__ counts) { counts[0] = *nsel; }

// popc of the mask of selected voxel i
struct Boundary3dPopc {
    const uint16_t* mask;
    const uint32_t* sel;
    __device__ __forceinline__ uint32_t operator()(uint32_t i) const { return (uint32_t)__popc(mask[sel[i]]); }
};

// popc of the mask of voxel t, 64-bit: the pair count of a call can exceed 2^32
struct Boundary3dPopc64 {
    const uint16_t* mask;
    __device__ __forceinline__ unsigned long long operator()(uint32_t t) const {
        return (unsigned long long)__popc(mask[t]);
    }
};

// Selected voxel i (first pair first[i]): for each of its boundary directions d in increasing order, the record at
// q = first[i] + j: key (image << 32 | lo << 16 | hi), pos = q, anchor = the voxel, dir = d
__global__ void __launch_bounds__(256) k_boundary3d_expand(const uint32_t* __restrict__ sel, uint32_t voxels,
                                                            const uint16_t* __restrict__ mask,
                                                            const uint32_t* __restrict__ first,
                                                            const uint16_t* __restrict__ lab, uint32_t dhw,
                                                            Boundary3dDirs dirs, unsigned long long* __restrict__ key,
                                                            uint32_t* __restrict__ pos, uint32_t* __restrict__ anchor,
                                                            uint8_t* __restrict__ dir) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < voxels; i += gridDim.x * blockDim.x) {
        const uint32_t t = sel[i], a = lab[t];
        const unsigned long long image = (unsigned long long)(t / dhw) << 32;
        uint32_t m = mask[t], q = first[i];
        while (m) {
            const int d = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t g = lab[t + dirs.off[d]];
            key[q] = image | (a < g ? a << 16 | g : g << 16 | a);
            pos[q] = q;
            anchor[q] = t;
            dir[q] = (uint8_t)d;
            q++;
        }
    }
}

// k_boundary_runs for volumes: run r of *d_runs is sorted positions [start[r], start[r + 1] or pairs); pair spos[i]
// has its anchor voxel anchor[.] and the other voxel anchor + off[dir[.]].  values [batch, C, dhw].
__global__ void __launch_bounds__(256) k_boundary3d_runs(const unsigned long long* __restrict__ skey,
                                                          const uint32_t* __restrict__ spos,
                                                          const uint32_t* __restrict__ anchor,
                                                          const uint8_t* __restrict__ dir,
                                                          const uint32_t* __restrict__ start,
                                                          const int* __restrict__ d_runs, int pairs,
                                                          const unsigned long long* __restrict__ sekey,
                                                          const uint32_t* __restrict__ seidx, int edges,
                                                          const float* __restrict__ values, int C, uint32_t dhw,
                                                          Boundary3dDirs dirs, float* __restrict__ mean,
                                                          float* __restrict__ mn, float* __restrict__ mx,
                                                          int32_t* __restrict__ count) {
    const int lane = threadIdx.x & 31;
    const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    const int runs = *d_runs;
    for (long r = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < runs; r += nwarps) {
        const int s = (int)start[r], e = r + 1 < runs ? (int)start[r + 1] : pairs;
        const unsigned long long key = skey[s];
        int pos = 0;
        if (lane < 2) pos = boundary_lower_bound(sekey, edges, key + (unsigned long long)lane);
        const int m0 = __shfl_sync(FSLIC_FULL, pos, 0), m = __shfl_sync(FSLIC_FULL, pos, 1) - m0;
        if (m == 0) continue;
        const uint32_t n = (uint32_t)(e - s), nv = 2 * n;
        const float f2n = __uint2float_rn(nv);
        const uint32_t base = (uint32_t)(key >> 32) * dhw;
        const float* f = values + (long)(key >> 32) * C * dhw;
        for (int k = lane; k < m; k += 32) count[seidx[m0 + k]] = (int32_t)n;
        int c = 0;
        for (; c + 4 <= C; c += 4) {
            const float* fc = f + (long)c * dhw;
            float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
            int lo[4] = {INT_MAX, INT_MAX, INT_MAX, INT_MAX}, hi[4] = {INT_MIN, INT_MIN, INT_MIN, INT_MIN};
            bool nan[4] = {false, false, false, false};
            for (uint32_t j = lane; j < nv; j += 32) {
                const uint32_t q = spos[s + (j >> 1)];
                const uint32_t p = anchor[q] - base + ((j & 1) ? (uint32_t)dirs.off[dir[q]] : 0u);
#pragma unroll
                for (int u = 0; u < 4; u++) boundary_add(__ldg(fc + (long)u * dhw + p), acc[u], lo[u], hi[u], nan[u]);
            }
            float rm[4], ra[4], rb[4];
#pragma unroll
            for (int u = 0; u < 4; u++) boundary_finish(acc[u], lo[u], hi[u], nan[u], f2n, &rm[u], &ra[u], &rb[u]);
            for (int q = lane; q < 4 * m; q += 32) {
                const int u = q & 3;
                const long o = (long)seidx[m0 + (q >> 2)] * C + c + u;
                mean[o] = u == 0 ? rm[0] : u == 1 ? rm[1] : u == 2 ? rm[2] : rm[3];
                mn[o] = u == 0 ? ra[0] : u == 1 ? ra[1] : u == 2 ? ra[2] : ra[3];
                mx[o] = u == 0 ? rb[0] : u == 1 ? rb[1] : u == 2 ? rb[2] : rb[3];
            }
        }
        for (; c < C; c++) {
            const float* fc = f + (long)c * dhw;
            float acc = 0.0f;
            int lo = INT_MAX, hi = INT_MIN;
            bool nan = false;
            for (uint32_t j = lane; j < nv; j += 32) {
                const uint32_t q = spos[s + (j >> 1)];
                const uint32_t p = anchor[q] - base + ((j & 1) ? (uint32_t)dirs.off[dir[q]] : 0u);
                boundary_add(__ldg(fc + p), acc, lo, hi, nan);
            }
            float rm, ra, rb;
            boundary_finish(acc, lo, hi, nan, f2n, &rm, &ra, &rb);
            for (int k = lane; k < m; k += 32) {
                const long o = (long)seidx[m0 + k] * C + c;
                mean[o] = rm;
                mn[o] = ra;
                mx[o] = rb;
            }
        }
    }
}
