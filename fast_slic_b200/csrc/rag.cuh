// fast_slic_b200/csrc/rag.cuh -- region adjacency graphs of a batch of label maps (DESIGN.md section 4.13): every pair
// of superpixels that touch, weighted by the number of adjacent pixel pairs between them, as CSR rows sorted by target.
// No counterpart in the reference.  All integer: the result is exact and independent of the launch order.
//
// Image b of a call owns the slice [b*T, (b+1)*T) of an open-addressing table of label-pair keys (a << 16 | c, a < c)
// and their pixel-pair counts:
//   k_rag_discover  one thread per pixel, 2 (connectivity 4) or 4 (connectivity 8) pixel pairs each: right and down,
//                   plus down-right and down-left.  Lanes of a warp holding the same (image, key) add once (MATCH.ANY);
//                   the leader claims a slot with one CAS and adds the count with one atomicAdd.  Past max_probes the
//                   image's overflow flag is set;
//   k_rag3d_discover the same over volumes (section 4.23): one thread per voxel, 3, 9 or 13 voxel pairs each
//                   (connectivity 6, 18, 26), feeding the same tables; every later step is shared;
//   k_rag_degree    every occupied slot adds 1 to the degree of both of its labels;
//   (exclusive scan of the degrees: the call-local CSR row offsets)
//   k_rag_finish    the caller's row offsets (shifted by the edges of earlier calls) and the call's edge total;
//   k_rag_scatter   every occupied slot files its two directed edges, keys row << 16 | target, at the next free place
//                   of their rows (in whatever order the atomics give);
//   (radix sort of the edge keys, the count as the value: rows in order, each by target -- keys are unique, so the
//   order is too)
//   k_rag_emit      the source and target node ids of the sorted keys.
#pragma once
#include "common.cuh"

#define RAG_EMPTY 0xffffffffu  // no key is all ones: a < c <= 65533

template <int CONN>
__global__ void __launch_bounds__(256) k_rag_discover(const uint16_t* __restrict__ lab, long hw, int H, int W, long n, int K,
                                                       uint32_t* __restrict__ tkey, uint32_t* __restrict__ tcnt, uint32_t T,
                                                       uint32_t max_probes, long long* __restrict__ overflow) {
    const long step = (long)gridDim.x * blockDim.x;
    const long nround = (n + step - 1) / step * step;  // whole warps stay in the loop: the warp intrinsics need all lanes
    const int lane = threadIdx.x & 31;
    const uint32_t tmask = T - 1;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nround; t += step) {
        long b = 0;
        int i = 0, j = 0;
        uint32_t s = 0xffffu;
        if (t < n) {
            // 32-bit divisions where they suffice (hw <= 2^29), a 64-bit one only for calls of 2^32 pixels or more
            b = n <= (long)UINT32_MAX ? (long)((uint32_t)t / (uint32_t)hw) : t / hw;
            const uint32_t p = (uint32_t)(t - b * hw);
            i = (int)(p / (uint32_t)W);
            j = (int)(p - (uint32_t)i * (uint32_t)W);
            s = lab[t];
        }
#pragma unroll
        for (int d = 0; d < CONN / 2; d++) {
            // d = 0: right, 1: down, 2: down-right, 3: down-left
            const int di = d == 0 ? 0 : 1, dj = d == 0 ? 1 : (d == 1 ? 0 : (d == 2 ? 1 : -1));
            unsigned long long key = ~0ull;
            if (s < (uint32_t)K && i + di < H && j + dj >= 0 && j + dj < W) {
                const uint32_t g = lab[t + (long)di * W + dj];
                if (g < (uint32_t)K && g != s) key = (unsigned long long)b << 32 | (s < g ? s << 16 | g : g << 16 | s);
            }
            if (!__any_sync(FSLIC_FULL, key != ~0ull)) continue;  // most warps: no boundary in this direction
            const unsigned peers = __match_any_sync(FSLIC_FULL, key);
            if (key == ~0ull || lane != __ffs(peers) - 1) continue;
            const uint32_t k32 = (uint32_t)key;
            uint32_t* ks = tkey + b * T;
            uint32_t h = conn_hash(k32) & tmask;
            for (uint32_t probes = 0;; probes++) {
                if (probes >= max_probes) {
                    overflow[b] = 1;
                    break;
                }
                const uint32_t old = atomicCAS(&ks[h], RAG_EMPTY, k32);
                if (old == RAG_EMPTY || old == k32) {
                    atomicAdd(&tcnt[b * T + h], (uint32_t)__popc(peers));
                    break;
                }
                h = (h + 1) & tmask;
            }
        }
    }
}

// k_rag_discover's insert of one direction as a function for k_rag3d_discover (the 2-D kernel keeps its own copy, so
// its code is unchanged), called by all 32 lanes: lanes holding the same (image, key) add once (MATCH.ANY), the leader
// claims a slot of image b's table with one CAS and adds the lane count; past max_probes the image's flag is set.  A
// key of ~0 is no pair.
__device__ __forceinline__ void rag_add(unsigned long long key, int lane, long b, uint32_t* __restrict__ tkey,
                                        uint32_t* __restrict__ tcnt, uint32_t T, uint32_t max_probes,
                                        long long* __restrict__ overflow) {
    const unsigned peers = __match_any_sync(FSLIC_FULL, key);
    if (key == ~0ull || lane != __ffs(peers) - 1) return;
    const uint32_t k32 = (uint32_t)key;
    const uint32_t tmask = T - 1;
    uint32_t* ks = tkey + b * T;
    uint32_t h = conn_hash(k32) & tmask;
    for (uint32_t probes = 0;; probes++) {
        if (probes >= max_probes) {
            overflow[b] = 1;
            break;
        }
        const uint32_t old = atomicCAS(&ks[h], RAG_EMPTY, k32);
        if (old == RAG_EMPTY || old == k32) {
            atomicAdd(&tcnt[b * T + h], (uint32_t)__popc(peers));
            break;
        }
        h = (h + 1) & tmask;
    }
}

// k_rag_discover over volumes: one thread per voxel, 3 (connectivity 6), 9 (18) or 13 (26) voxel pairs each.  Every
// direction is tested first and one warp vote skips warps whose voxels all lie inside one label (most of a supervoxel
// map); the rest go through the same per-direction vote, match and table insert as the 2-D kernel.
template <int CONN>
__global__ void __launch_bounds__(256) k_rag3d_discover(const uint16_t* __restrict__ lab, long dhw, int D, int H, int W,
                                                         long n, int K, uint32_t* __restrict__ tkey,
                                                         uint32_t* __restrict__ tcnt, uint32_t T, uint32_t max_probes,
                                                         long long* __restrict__ overflow) {
    // the forward half of the 3x3x3 neighbourhood (first non-zero offset positive), (dz, dy, dx): connectivity 6 takes
    // the first 3 (faces), 18 the first 9 (and edges), 26 all 13 (and corners)
    constexpr int NDIR = CONN == 6 ? 3 : (CONN == 18 ? 9 : 13);
    constexpr int8_t dirs[13][3] = {{0, 0, 1}, {0, 1, 0},  {1, 0, 0},  {0, 1, 1},  {0, 1, -1},
                                    {1, 1, 0}, {1, -1, 0}, {1, 0, 1},  {1, 0, -1}, {1, 1, 1},
                                    {1, 1, -1}, {1, -1, 1}, {1, -1, -1}};
    const long step = (long)gridDim.x * blockDim.x;
    const long nround = (n + step - 1) / step * step;  // whole warps stay in the loop: the warp intrinsics need all lanes
    const int lane = threadIdx.x & 31;
    const uint32_t hw = (uint32_t)H * (uint32_t)W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nround; t += step) {
        long b = 0;
        int z = 0, y = 0, x = 0;
        uint32_t s = 0xffffu;
        if (t < n) {
            // 32-bit divisions where they suffice (dhw <= 2^29), a 64-bit one only for calls of 2^32 voxels or more
            b = n <= (long)UINT32_MAX ? (long)((uint32_t)t / (uint32_t)dhw) : t / dhw;
            const uint32_t p = (uint32_t)(t - b * dhw);
            z = (int)(p / hw);
            const uint32_t r = p - (uint32_t)z * hw;
            y = (int)(r / (uint32_t)W);
            x = (int)(r - (uint32_t)y * (uint32_t)W);
            s = lab[t];
        }
        // bit d: the pair in direction d is valid and its labels differ
        uint32_t diff = 0;
#pragma unroll
        for (int d = 0; d < NDIR; d++) {
            const int dz = dirs[d][0], dy = dirs[d][1], dx = dirs[d][2];
            if (s < (uint32_t)K && z + dz < D && y + dy >= 0 && y + dy < H && x + dx >= 0 && x + dx < W) {
                const uint32_t g = lab[t + (long)dz * hw + (long)dy * W + dx];
                if (g < (uint32_t)K && g != s) diff |= 1u << d;
            }
        }
        if (!__any_sync(FSLIC_FULL, diff != 0)) continue;  // most warps: no boundary in any direction
#pragma unroll
        for (int d = 0; d < NDIR; d++) {
            if (!__any_sync(FSLIC_FULL, diff >> d & 1u)) continue;
            unsigned long long key = ~0ull;
            if (diff >> d & 1u) {  // the neighbour again, from L1
                const uint32_t g = lab[t + (long)dirs[d][0] * hw + (long)dirs[d][1] * W + dirs[d][2]];
                key = (unsigned long long)b << 32 | (s < g ? s << 16 | g : g << 16 | s);
            }
            rag_add(key, lane, b, tkey, tcnt, T, max_probes, overflow);
        }
    }
}

// deg [batch*K] (zeroed before): the number of distinct neighbours of each (image, label)
__global__ void __launch_bounds__(256) k_rag_degree(const uint32_t* __restrict__ tkey, long nslots, int tshift, int K,
                                                     unsigned long long* __restrict__ deg) {
    for (long s = (long)blockIdx.x * blockDim.x + threadIdx.x; s < nslots; s += (long)gridDim.x * blockDim.x) {
        const uint32_t key = tkey[s];
        if (key == RAG_EMPTY) continue;
        const long row = (s >> tshift) * K;
        atomicAdd(&deg[row + (key >> 16)], 1ull);
        atomicAdd(&deg[row + (key & 0xffffu)], 1ull);
    }
}

// indptr[r] = local[r] + edge_base for the nk + 1 row offsets; *total = local[nk], the call's directed edge count
__global__ void __launch_bounds__(256) k_rag_finish(const long long* __restrict__ local, long nk, long long edge_base,
                                                     long long* __restrict__ indptr, long long* __restrict__ total) {
    for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r <= nk; r += (long)gridDim.x * blockDim.x) {
        indptr[r] = local[r] + edge_base;
        if (r == nk) *total = local[nk];
    }
}

// Each occupied slot {u, c} of image b, count w: the edges (row b*K+u, target c) and (row b*K+c, target u) as keys
// row << 16 | target, at local[row] + cursor[row]++ of their rows; val gets the count.
__global__ void __launch_bounds__(256) k_rag_scatter(const uint32_t* __restrict__ tkey, const uint32_t* __restrict__ tcnt,
                                                      long nslots, int tshift, int K, const long long* __restrict__ local,
                                                      unsigned long long* __restrict__ cursor,
                                                      unsigned long long* __restrict__ ekey, int32_t* __restrict__ val) {
    for (long s = (long)blockIdx.x * blockDim.x + threadIdx.x; s < nslots; s += (long)gridDim.x * blockDim.x) {
        const uint32_t key = tkey[s];
        if (key == RAG_EMPTY) continue;
        const long base = (s >> tshift) * K;
        const uint32_t u = key >> 16, c = key & 0xffffu;
        const int32_t w = (int32_t)tcnt[s];
        const long long pu = local[base + u] + (long long)atomicAdd(&cursor[base + u], 1ull);
        const long long pc = local[base + c] + (long long)atomicAdd(&cursor[base + c], 1ull);
        ekey[pu] = (unsigned long long)(base + u) << 16 | c;
        val[pu] = w;
        ekey[pc] = (unsigned long long)(base + c) << 16 | u;
        val[pc] = w;
    }
}

// The sorted edge keys -> src = node_base + row, dst = node_base + the row's image * K + target
__global__ void __launch_bounds__(256) k_rag_emit(const unsigned long long* __restrict__ skey, long long edges, int K,
                                                   long long node_base, long long* __restrict__ src,
                                                   long long* __restrict__ dst) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < edges; e += (long long)gridDim.x * blockDim.x) {
        const unsigned long long key = skey[e];
        const long long row = (long long)(key >> 16);
        src[e] = node_base + row;
        dst[e] = node_base + row / K * K + (long long)(key & 0xffffu);
    }
}
