// fast_slic_b200/csrc/knn.cuh -- exact k-nearest-neighbour graphs over the feature points of superpixels (DESIGN.md
// section 4.18).  No counterpart in the reference (its get_knn_connectivity has no defined result).
//
// Node n = b * K + i is row i of image b's points [K][D].  It is a candidate when it is present and its D coordinates
// are finite.  The distance of two nodes is s = ((+0 + t_0 * t_0) + t_1 * t_1) + ..., t_c = p_i[c] - p_j[c], every
// operation rounded to nearest on its own (no FMA contraction), so s(i, j) and s(j, i) are the same bits, s >= +0 and s
// is never NaN.  Candidates of one image are ordered by the 64-bit key float_bits(s) << 32 | j: s >= +0, so the raw bits
// order like the floats, and one integer compare gives the (s, j) order.  Node i's neighbours are the first
// min(k, P_b - 1) other candidates of its image under that order.
//
// One call runs in two steps, with one host read of the edge total between them:
//   count   k_knn_flags          candidacy of every node of the call;
//           (cub::DeviceSelect::Flagged of the candidates, in node order)
//           k_knn_starts         where each image's candidates begin in that list;
//           k_knn_pack           each candidate's coordinates, zero-padded to DP (a power of two >= 4; the padding
//                                adds +0 * +0 = +0 to s, which leaves its bits unchanged);
//           k_knn_select<KC, DP> one thread per candidate query: the best k keys over tiles of the image's candidates
//                                staged in shared memory, written in j order, the row count;
//     directed:  (cub::DeviceScan::ExclusiveSum of the row counts) and k_knn_rows: indptr and the total;
//     symmetric: k_knn_pairs        both directions of every selected edge as row << 16 | target, the distance as
//                                   the value, all ones for an unused slot;
//                (cub::DeviceRadixSort::SortPairs over the bits in use, cub::DeviceSelect::UniqueByKey: a pair found
//                from both ends has the same key and the same distance bits)
//                k_knn_unique_rows: indptr from the sorted keys by binary search, and the total;
//   fill    k_knn_emit_directed / k_knn_emit_symmetric: edge_index and distance.
#pragma once
#include <stdint.h>

#include "common.cuh"

#define KNN_NO_KEY 0xffffffffffffffffull
#define KNN_THREADS 128
// Shared memory of one select CTA's candidate tile: 32 KB of coordinates (8192 / DP candidates) and their indices
#define KNN_TILE_FLOATS 8192

__global__ void k_knn_flags(const float* __restrict__ points, const uint8_t* __restrict__ present, long nodes, int D,
                            uint8_t* __restrict__ flags) {
    for (long n = blockIdx.x * (long)blockDim.x + threadIdx.x; n < nodes; n += (long)gridDim.x * blockDim.x) {
        bool ok = present == nullptr || present[n] != 0;
        for (int c = 0; c < D && ok; c++) ok = isfinite(points[n * D + c]);
        flags[n] = ok ? 1 : 0;
    }
}

// starts[b] = the first candidate of image b (b in [0, batch]): a lower bound of b * K in the ordered candidate list
__global__ void k_knn_starts(const uint32_t* __restrict__ cand, const int* __restrict__ ncand, int batch, int K,
                             int* __restrict__ starts) {
    const int n = *ncand;
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b <= batch; b += gridDim.x * blockDim.x) {
        const uint32_t target = (uint32_t)b * (uint32_t)K;
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (cand[mid] < target) lo = mid + 1;
            else hi = mid;
        }
        starts[b] = lo;
    }
}

__global__ void k_knn_pack(const float* __restrict__ points, const uint32_t* __restrict__ cand,
                           const int* __restrict__ ncand, int D, int DP, float* __restrict__ packed) {
    const long items = (long)*ncand * DP;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < items; t += (long)gridDim.x * blockDim.x) {
        const long q = t / DP;
        const int c = (int)(t - q * DP);
        packed[t] = c < D ? points[(long)cand[q] * D + c] : 0.0f;
    }
}

// Replaces the largest key, best[0], with key and moves it down the descending list to its place.  The lists are
// kept over KC registers with constant indices only: best[0, k) holds the k best keys (+1, all ones for none yet),
// best[k, KC) holds 0, below every key + 1, which never moves.
template <int KC>
__device__ __forceinline__ void knn_insert(unsigned long long (&best)[KC], unsigned long long key) {
    best[0] = key;
#pragma unroll
    for (int i = 0; i + 1 < KC; i++) {
        const unsigned long long a = best[i], b = best[i + 1];
        best[i] = a < b ? b : a;
        best[i + 1] = a < b ? a : b;
    }
}

// One thread per candidate query of image blockIdx.y (and every gridDim.y-th image after it), KNN_THREADS queries per
// CTA.  Writes row_count[row] = min(k, P - 1) and the row's neighbours in ascending j to idx / dist [row * k + i], row
// the query's node in the call.  The k best keys live in KC >= k registers (knn_insert).
template <int KC, int DP>
__global__ void __launch_bounds__(KNN_THREADS) k_knn_select(const float* __restrict__ packed,
                                                           const uint32_t* __restrict__ cand,
                                                           const int* __restrict__ starts, int batch, int K, int k,
                                                           int* __restrict__ row_count, uint32_t* __restrict__ idx,
                                                           float* __restrict__ dist) {
    constexpr int TILE = KNN_TILE_FLOATS / DP;
    __shared__ __align__(16) float tile[KNN_TILE_FLOATS];
    __shared__ uint32_t tile_j[TILE];
    for (int b = blockIdx.y; b < batch; b += gridDim.y) {
        const int start = starts[b], P = starts[b + 1] - start;
        const int q0 = blockIdx.x * KNN_THREADS;
        if (q0 >= P) continue;  // uniform over the CTA
        const int qi = q0 + (int)threadIdx.x;
        const bool live = qi < P;
        float q[DP];
#pragma unroll
        for (int c = 0; c < DP; c += 4) {
            const float4 v = live ? *reinterpret_cast<const float4*>(packed + (long)(start + qi) * DP + c)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
            q[c] = v.x;
            q[c + 1] = v.y;
            q[c + 2] = v.z;
            q[c + 3] = v.w;
        }
        unsigned long long best[KC];
#pragma unroll
        for (int i = 0; i < KC; i++) best[i] = i < k ? KNN_NO_KEY : 0ull;
        for (int t0 = 0; t0 < P; t0 += TILE) {
            const int n = P - t0 < TILE ? P - t0 : TILE;
            __syncthreads();
            const float4* src = reinterpret_cast<const float4*>(packed + (long)(start + t0) * DP);
            for (int v = threadIdx.x; v < n * (DP / 4); v += KNN_THREADS)
                reinterpret_cast<float4*>(tile)[v] = src[v];
            for (int v = threadIdx.x; v < n; v += KNN_THREADS) tile_j[v] = cand[start + t0 + v] - (uint32_t)b * K;
            __syncthreads();
            if (!live) continue;
#pragma unroll 2
            for (int jj = 0; jj < n; jj++) {
                const float4* p = reinterpret_cast<const float4*>(tile + jj * DP);
                float s = 0.0f;
#pragma unroll
                for (int c = 0; c < DP; c += 4) {
                    const float4 v = p[c / 4];
                    float t = __fsub_rn(q[c], v.x);
                    s = __fadd_rn(s, __fmul_rn(t, t));
                    t = __fsub_rn(q[c + 1], v.y);
                    s = __fadd_rn(s, __fmul_rn(t, t));
                    t = __fsub_rn(q[c + 2], v.z);
                    s = __fadd_rn(s, __fmul_rn(t, t));
                    t = __fsub_rn(q[c + 3], v.w);
                    s = __fadd_rn(s, __fmul_rn(t, t));
                }
                const unsigned long long key = ((unsigned long long)__float_as_uint(s) << 32 | tile_j[jj]) + 1;
                if (key < best[0] && t0 + jj != qi) knn_insert<KC>(best, key);
            }
        }
        if (!live) continue;
        const int cnt = P - 1 < k ? P - 1 : k;
        // the row in ascending target order: each neighbour goes to its rank by j among the row's cnt neighbours
        const long row = (long)cand[start + qi];
        row_count[row] = cnt;
#pragma unroll
        for (int i = 0; i < KC; i++) {
            const bool real = best[i] != 0 && best[i] != KNN_NO_KEY;
            if (real) {
                const uint32_t j = (uint32_t)(best[i] - 1);
                int rank = 0;
#pragma unroll
                for (int m = 0; m < KC; m++) rank += best[m] != 0 && best[m] != KNN_NO_KEY && (uint32_t)(best[m] - 1) < j;
                idx[row * k + rank] = j;
                dist[row * k + rank] = __uint_as_float((uint32_t)((best[i] - 1) >> 32));
            }
        }
    }
}

// Directed: indptr[r] = edge_base + offs[r] for the call's rows r in [0, nodes]; the total after the last
__global__ void k_knn_rows(const int* __restrict__ offs, long nodes, long long edge_base, long long* __restrict__ indptr,
                           long long* __restrict__ total) {
    for (long r = blockIdx.x * (long)blockDim.x + threadIdx.x; r <= nodes; r += (long)gridDim.x * blockDim.x) {
        indptr[r] = edge_base + offs[r];
        if (r == nodes) *total = offs[r];
    }
}

// Symmetric: both directions of slot (row, i) at 2 * slot and 2 * slot + 1 as row << 16 | target, all ones for a slot
// past the row's count
__global__ void k_knn_pairs(const int* __restrict__ row_count, const uint32_t* __restrict__ idx,
                            const float* __restrict__ dist, long nodes, int K, int k,
                            unsigned long long* __restrict__ keys, float* __restrict__ vals) {
    const long slots = nodes * k;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < slots; t += (long)gridDim.x * blockDim.x) {
        const long row = t / k;
        const int i = (int)(t - row * k);
        unsigned long long a = KNN_NO_KEY, r = KNN_NO_KEY;
        float s = 0.0f;
        if (i < row_count[row]) {
            const unsigned long long j = idx[t], base = (unsigned long long)(row / K) * K, local = row - base;
            a = (unsigned long long)row << 16 | j;
            r = (base + j) << 16 | local;
            s = dist[t];
        }
        keys[2 * t] = a;
        keys[2 * t + 1] = r;
        vals[2 * t] = s;
        vals[2 * t + 1] = s;
    }
}

// Symmetric: indptr[r] = edge_base + the first unique key at or after r << 16, for the call's rows r in [0, nodes]; the
// total (unique keys below the all-ones sentinel) after the last
__global__ void k_knn_unique_rows(const unsigned long long* __restrict__ ukeys, const int* __restrict__ nunique,
                                  long nodes, long long edge_base, long long* __restrict__ indptr,
                                  long long* __restrict__ total) {
    const int n = *nunique;
    for (long r = blockIdx.x * (long)blockDim.x + threadIdx.x; r <= nodes; r += (long)gridDim.x * blockDim.x) {
        const unsigned long long target = (unsigned long long)r << 16;
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ukeys[mid] < target) lo = mid + 1;
            else hi = mid;
        }
        indptr[r] = edge_base + lo;
        if (r == nodes) *total = lo;
    }
}

__global__ void k_knn_emit_directed(const int* __restrict__ row_count, const int* __restrict__ offs,
                                    const uint32_t* __restrict__ idx, const float* __restrict__ dist, long nodes, int K,
                                    int k, long long node_base, long long* __restrict__ src, long long* __restrict__ dst,
                                    float* __restrict__ distance) {
    const long slots = nodes * k;
    for (long t = blockIdx.x * (long)blockDim.x + threadIdx.x; t < slots; t += (long)gridDim.x * blockDim.x) {
        const long row = t / k;
        const int i = (int)(t - row * k);
        if (i < row_count[row]) {
            const long e = offs[row] + i;
            src[e] = node_base + row;
            dst[e] = node_base + (row / K) * K + idx[t];
            distance[e] = dist[t];
        }
    }
}

__global__ void k_knn_emit_symmetric(const unsigned long long* __restrict__ ukeys, const float* __restrict__ uvals,
                                     long edges, int K, long long node_base, long long* __restrict__ src,
                                     long long* __restrict__ dst, float* __restrict__ distance) {
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < edges; e += (long)gridDim.x * blockDim.x) {
        const unsigned long long key = ukeys[e];
        const long long row = (long long)(key >> 16);
        src[e] = node_base + row;
        dst[e] = node_base + (row / K) * K + (long long)(key & 0xffff);
        distance[e] = uvals[e];
    }
}
