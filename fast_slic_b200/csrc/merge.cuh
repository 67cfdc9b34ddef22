// fast_slic_b200/csrc/merge.cuh -- single-linkage merging of superpixels over a region adjacency graph (DESIGN.md section
// 4.16): the minimum spanning forest of each image by Boruvka, then a threshold or region-count cut of it.  No
// counterpart in the reference.
//
// Node n = b * K + k is label k of image b, present when a pixel of image b carries k.  An undirected edge {lo, hi} of
// image b (local ids, lo < hi) with float weight w has the key
//   merge_wkey(w) << 32 | lo << 16 | hi,
// where merge_wkey maps float32 to uint32 in order (-0 to +0).  Keys are unique inside an image, so every atomicMin
// below picks the same edge however the threads interleave, and the forest and its order are unique.  All union-find
// links put the larger root under the smaller, so parent pointers only decrease, no cycle can form and every root is
// the smallest id of its tree.
#pragma once
#include "common.cuh"

#define MERGE_NO_KEY 0xffffffffffffffffull
#define MERGE_ROUNDS 16  // each round at least halves the trees of every component: 2^16 > 65534 nodes

__device__ __forceinline__ uint32_t merge_wkey(float w) {
    const uint32_t u = w == 0.0f ? 0u : __float_as_uint(w);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float merge_weight(uint32_t wk) {
    return __uint_as_float((wk & 0x80000000u) ? (wk & 0x7fffffffu) : ~wk);
}

// Parent pointers change under concurrent links: read them past L1
__device__ __forceinline__ int merge_find(int* parent, int x) {
    for (;;) {
        const int p = *(volatile int*)&parent[x];
        if (p == x) return x;
        x = p;
    }
}

// Links the trees of a and b, the larger root under the smaller, with a CAS that succeeds only while that root is
// still a root.  Returns whether this call made the link (false: a and b were already in one tree).
__device__ __forceinline__ bool merge_union(int* parent, int a, int b) {
    for (;;) {
        a = merge_find(parent, a);
        b = merge_find(parent, b);
        if (a == b) return false;
        if (a < b) {
            const int t = a;
            a = b;
            b = t;
        }
        if (atomicCAS(&parent[a], a, b) == a) return true;
    }
}

// present [n_nodes] and P [batch] zeroed before: present[b*K + k] = 1 where a pixel of image b carries k, P[b] = the
// number of such k.  The plain load first keeps the atomics to about one per node.
__global__ void __launch_bounds__(256) k_merge_presence(const uint16_t* __restrict__ lab, long hw, long n, int K,
                                                         int* present, int* P) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const uint32_t l = lab[t];
        if (l >= (uint32_t)K) continue;
        const long b = t / hw;
        int* f = present + b * K + l;
        if (!*(volatile int*)f && atomicExch(f, 1) == 0) atomicAdd(P + b, 1);
    }
}

// parent[x] = x, best[x] = no key
__global__ void __launch_bounds__(256) k_merge_init(long n_nodes, int* __restrict__ parent,
                                                     unsigned long long* __restrict__ best) {
    for (long x = (long)blockIdx.x * blockDim.x + threadIdx.x; x < n_nodes; x += (long)gridDim.x * blockDim.x) {
        parent[x] = (int)x;
        best[x] = MERGE_NO_KEY;
    }
}

// Rounds after one that linked nothing do nothing: the forest is complete
__device__ __forceinline__ bool merge_round_done(const int* linked, int round) {
    return round > 0 && !*(volatile const int*)&linked[round - 1];
}

// Boruvka, step 1: every tree root takes the smallest key of the edges that leave its tree.  Only entries with
// src < dst are read; an entry is skipped when an endpoint is outside [0, n_nodes), the endpoints lie in different
// images, an endpoint is not present or the weight is NaN.  parent is flat here (every node points at its root).
__global__ void __launch_bounds__(256) k_merge_choose(int round, const int* __restrict__ linked,
                                                       const long long* __restrict__ src,
                                                       const long long* __restrict__ dst,
                                                       const float* __restrict__ weight, long long edges,
                                                       long long n_nodes, int K, const int* __restrict__ present,
                                                       const int* __restrict__ parent,
                                                       unsigned long long* __restrict__ best) {
    if (merge_round_done(linked, round)) return;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < edges;
         e += (long long)gridDim.x * blockDim.x) {
        const long long u = src[e], v = dst[e];
        if (u < 0 || u >= v || v >= n_nodes) continue;
        const long long b = u / K;
        if (v >= (b + 1) * K || !present[u] || !present[v]) continue;
        const float w = weight[e];
        if (isnan(w)) continue;
        const int ru = parent[u], rv = parent[v];
        if (ru == rv) continue;
        const unsigned long long key =
            (unsigned long long)merge_wkey(w) << 32 | (unsigned long long)(u - b * K) << 16 | (unsigned long long)(v - b * K);
        atomicMin(best + ru, key);
        atomicMin(best + rv, key);
    }
}

// Boruvka, step 2: each root links its tree along its chosen edge.  Two roots that chose the same edge link once, so
// the union that makes the link appends the edge to its image's slice [b*K, b*K + count[b]) of the forest table.
// A root is recognised by its key: best is set at roots only, and parent changes under the concurrent links.
__global__ void __launch_bounds__(256) k_merge_link(int round, int* linked, long n_nodes, int K, int* parent,
                                                     const unsigned long long* __restrict__ best,
                                                     unsigned long long* __restrict__ table, int* count) {
    if (merge_round_done(linked, round)) return;
    for (long x = (long)blockIdx.x * blockDim.x + threadIdx.x; x < n_nodes; x += (long)gridDim.x * blockDim.x) {
        const unsigned long long key = best[x];
        if (key == MERGE_NO_KEY) continue;
        const long b = x / K;
        const int lo = (int)(key >> 16 & 0xffffu), hi = (int)(key & 0xffffu);
        if (merge_union(parent, (int)(b * K + lo), (int)(b * K + hi))) {
            table[b * K + atomicAdd(count + b, 1)] = key;
            linked[round] = 1;
        }
    }
}

// Boruvka, step 3 (and the end of the cut): every node points at its root; best is cleared for the next round.
// Concurrent rewrites only replace a pointer by its root, so every walk still ends there.
__global__ void __launch_bounds__(256) k_merge_flatten(int round, const int* __restrict__ linked, long n_nodes,
                                                        int* parent, unsigned long long* __restrict__ best) {
    if (merge_round_done(linked, round)) return;
    for (long x = (long)blockIdx.x * blockDim.x + threadIdx.x; x < n_nodes; x += (long)gridDim.x * blockDim.x) {
        parent[x] = merge_find(parent, (int)x);
        best[x] = MERGE_NO_KEY;
    }
}

// The cut: union the prefix of each image's forest edges in key order.  threshold: the edges with (double)w < t (the
// slice need not be sorted: which edges pass does not depend on their order); num_regions = R: the first
// max(0, P[b] - R) edges of the sorted slice.  parent is reset to the identity before.
__global__ void __launch_bounds__(256) k_merge_cut(long n_nodes, int K, int by_count, double threshold, int num_regions,
                                                    const unsigned long long* __restrict__ table,
                                                    const int* __restrict__ count, const int* __restrict__ P,
                                                    int* parent) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_nodes; i += (long)gridDim.x * blockDim.x) {
        const long b = i / K;
        const int j = (int)(i - b * K);
        if (j >= count[b]) continue;
        const unsigned long long key = table[i];
        if (by_count ? j >= P[b] - num_regions : !((double)merge_weight((uint32_t)(key >> 32)) < threshold)) continue;
        merge_union(parent, (int)(b * K + (key >> 16 & 0xffffu)), (int)(b * K + (key & 0xffffu)));
    }
}

// flag[x] = 1 for a present root (the smallest id of its region), flag[n_nodes] = 0: the scan gives each region its
// number and each image its total
__global__ void __launch_bounds__(256) k_merge_roots(long n_nodes, const int* __restrict__ present,
                                                      const int* __restrict__ parent, int* __restrict__ flag) {
    for (long x = (long)blockIdx.x * blockDim.x + threadIdx.x; x <= n_nodes; x += (long)gridDim.x * blockDim.x)
        flag[x] = x < n_nodes && present[x] && parent[x] == (int)x;
}

// region[x] = the number of x's root in its image (pos: the exclusive scan of flag), -1 for a node that is not
// present; num_regions[b] = the present roots of image b
__global__ void __launch_bounds__(256) k_merge_number(long n_nodes, int K, const int* __restrict__ present,
                                                       const int* __restrict__ parent, const int* __restrict__ pos,
                                                       int32_t* __restrict__ region, int32_t* __restrict__ num_regions) {
    for (long x = (long)blockIdx.x * blockDim.x + threadIdx.x; x < n_nodes; x += (long)gridDim.x * blockDim.x) {
        const long b = x / K, base = b * K;
        region[x] = present[x] ? pos[parent[x]] - pos[base] : -1;
        if (x == base) num_regions[b] = pos[base + K] - pos[base];
    }
}

// Segment bounds of the forest sort: image b's edges are table[b*K, b*K + count[b])
__global__ void __launch_bounds__(256) k_merge_segments(int batch, int K, const int* __restrict__ count,
                                                         int* __restrict__ seg_begin, int* __restrict__ seg_end) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < batch; b += gridDim.x * blockDim.x) {
        seg_begin[b] = b * K;
        seg_end[b] = b * K + count[b];
    }
}
