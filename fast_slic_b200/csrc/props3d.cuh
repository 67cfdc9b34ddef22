// fast_slic_b200/csrc/props3d.cuh -- supervoxel shapes (DESIGN.md section 4.23): per (volume, label) the voxel count,
// bounding box, raw first and second moments, surface (faces to another label or outside the volume) and its
// volume-edge part, then the centroid and central second moments in float64.  The volume form of props.cuh, with the
// same shared-table scheme.  Integer only up to the finishing kernel, whose float64 steps are each one IEEE-rounded
// operation: every result is exact and independent of the launch order.
//
//   k_props3d_init    one thread per node: zero sums, bbox minima at INT_MAX, maxima at 0;
//   k_props3d_tiles   one CTA per tile of PROPS3D_TILE_ROWS rows x PROPS3D_TILE_WORDS * 32 columns of one slice; each
//                     warp walks one 32-column word down the tile's rows, loading the voxels in front (z - 1) and behind
//                     (z + 1) of each.  Per row a ballot of "label differs from the left neighbour" splits the word into
//                     runs; the head lane of each run adds its closed-form moments, box and faces to a shared table keyed
//                     by label (shared atomics), or straight to global memory when the table has no slot for it.  Each
//                     table entry is flushed to global memory once per tile;
//   k_props3d_finish  one thread per node: centroid and covariance from the integer sums, empty boxes zeroed.
#pragma once
#include <limits.h>

#include "common.cuh"

#define PROPS3D_TILE_ROWS 32
#define PROPS3D_TILE_WORDS 8                     // one word per warp of the 256-thread CTA
#define PROPS3D_TABLE 256                        // table slots, a power of two
#define PROPS3D_PROBES 16                        // slots tried before a run goes to global memory
#define PROPS3D_EMPTY 0xffffffffu
#define PROPS3D_MOMENTS 9                        // sum z, y, x, z^2, zy, zx, y^2, yx, x^2

// The global outputs of one call, node n = b*K + k
struct Props3dOut {
    int32_t* area;                  // [n]
    int32_t* bbox;                  // [n][6]: z0, y0, x0 (min, inclusive), z1, y1, x1 (max, exclusive)
    unsigned long long* moments;    // [n][9] (int64; every sum is non-negative)
    unsigned long long* surface;    // [n] (int64)
    int32_t* border;                // [n]
};

// What one run, or one table entry, adds to a node.  A tile has 8192 voxels of 6 faces, so its surface fits 32 bits.
struct Props3dAdd {
    uint32_t area, surface, border;
    int lo[3], hi[3];
    unsigned long long m[PROPS3D_MOMENTS];
};

__device__ __forceinline__ void props3d_to_global(const Props3dOut& o, long n, const Props3dAdd& a) {
    atomicAdd(&o.area[n], (int)a.area);
    atomicAdd(&o.surface[n], (unsigned long long)a.surface);
    atomicAdd(&o.border[n], (int)a.border);
#pragma unroll
    for (int f = 0; f < 3; f++) {
        atomicMin(&o.bbox[n * 6 + f], a.lo[f]);
        atomicMax(&o.bbox[n * 6 + 3 + f], a.hi[f]);
    }
#pragma unroll
    for (int f = 0; f < PROPS3D_MOMENTS; f++) atomicAdd(&o.moments[n * PROPS3D_MOMENTS + f], a.m[f]);
}

__global__ void __launch_bounds__(256) k_props3d_init(long nodes, Props3dOut o) {
    for (long n = (long)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (long)gridDim.x * blockDim.x) {
        o.area[n] = 0;
        o.surface[n] = 0;
        o.border[n] = 0;
#pragma unroll
        for (int f = 0; f < 3; f++) {
            o.bbox[n * 6 + f] = INT_MAX;
            o.bbox[n * 6 + 3 + f] = 0;
        }
#pragma unroll
        for (int f = 0; f < PROPS3D_MOMENTS; f++) o.moments[n * PROPS3D_MOMENTS + f] = 0;
    }
}

// Sum of c^2 for c in [0, n], n >= -1
__device__ __forceinline__ unsigned long long props3d_sq_sum(long long n) {
    return (unsigned long long)(n * (n + 1) * (2 * n + 1) / 6);
}

// The shared table of one CTA: slot s holds label key[s] of the current tile (PROPS3D_EMPTY when free)
struct Props3dTable {
    uint32_t key[PROPS3D_TABLE];
    uint32_t area[PROPS3D_TABLE], surface[PROPS3D_TABLE], border[PROPS3D_TABLE];
    int lo[3][PROPS3D_TABLE], hi[3][PROPS3D_TABLE];
    unsigned long long m[PROPS3D_MOMENTS][PROPS3D_TABLE];
};

__device__ __forceinline__ void props3d_slot_reset(Props3dTable& t, int s) {
    t.key[s] = PROPS3D_EMPTY;
    t.area[s] = t.surface[s] = t.border[s] = 0;
#pragma unroll
    for (int f = 0; f < 3; f++) {
        t.lo[f][s] = INT_MAX;
        t.hi[f][s] = 0;
    }
#pragma unroll
    for (int f = 0; f < PROPS3D_MOMENTS; f++) t.m[f][s] = 0;
}

// The slot of label k in the table, claimed if k is new; -1 when PROPS3D_PROBES slots are taken by other labels
__device__ __forceinline__ int props3d_slot(Props3dTable& t, uint32_t k) {
    int s = (int)((k * 2654435761u) >> 24) & (PROPS3D_TABLE - 1);
    for (int p = 0; p < PROPS3D_PROBES; p++) {
        const uint32_t cur = *(volatile uint32_t*)&t.key[s];
        if (cur == k) return s;
        if (cur == PROPS3D_EMPTY) {
            const uint32_t old = atomicCAS(&t.key[s], PROPS3D_EMPTY, k);
            if (old == PROPS3D_EMPTY || old == k) return s;
        }
        s = (s + 1) & (PROPS3D_TABLE - 1);
    }
    return -1;
}

__device__ __forceinline__ void props3d_to_table(Props3dTable& t, int s, const Props3dAdd& a) {
    atomicAdd(&t.area[s], a.area);
    atomicAdd(&t.surface[s], a.surface);
    atomicAdd(&t.border[s], a.border);
#pragma unroll
    for (int f = 0; f < 3; f++) {
        atomicMin(&t.lo[f][s], a.lo[f]);
        atomicMax(&t.hi[f][s], a.hi[f]);
    }
#pragma unroll
    for (int f = 0; f < PROPS3D_MOMENTS; f++) atomicAdd(&t.m[f][s], a.m[f]);
}

// Grid: y over volumes (looping past 65535), x over the tiles of a volume (D slices of ceil(H / PROPS3D_TILE_ROWS)
// rows of ceil(Wd / PROPS3D_TILE_WORDS) tiles).  256 threads.  Outputs initialised by k_props3d_init.
__global__ void __launch_bounds__(256) k_props3d_tiles(const uint16_t* __restrict__ lab, int batch, int D, int H, int W,
                                                       int K, Props3dOut o) {
    __shared__ Props3dTable t;
    const int Wd = (W + 31) / 32, tcols = (Wd + PROPS3D_TILE_WORDS - 1) / PROPS3D_TILE_WORDS;
    const int trows = (H + PROPS3D_TILE_ROWS - 1) / PROPS3D_TILE_ROWS, slice_tiles = trows * tcols;
    const int tiles = D * slice_tiles;
    const long hw = (long)H * W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    props3d_slot_reset(t, threadIdx.x);
    __syncthreads();
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const uint16_t* l = lab + b * (hw * D);
        const long node0 = b * (long)K;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int z = tile / slice_tiles, r = tile - z * slice_tiles;
            const int ty = r / tcols, w = (r - ty * tcols) * PROPS3D_TILE_WORDS + warp;
            const int i0 = ty * PROPS3D_TILE_ROWS, i1 = min(H, i0 + PROPS3D_TILE_ROWS);
            const uint16_t* ls = l + z * hw;  // this slice
            // warp-uniform: the warp's word, walked down rows i0 .. i1 - 1
            if (w < Wd) {
                const int j = w * 32 + lane;
                const bool in = j < W;
                const uint32_t valid = __ballot_sync(FSLIC_FULL, in);
                const int last = 31 - __clz(valid);
                const bool has_front = z > 0, has_back = z + 1 < D;
                uint32_t up = 0, cur = 0;
                if (in && i0 > 0) up = ls[(long)(i0 - 1) * W + j];
                if (in) cur = ls[(long)i0 * W + j];
                for (int i = i0; i < i1; i++) {
                    const long p = (long)i * W + j;
                    uint32_t down = 0, front = 0, back = 0;
                    if (in && i + 1 < H) down = ls[p + W];
                    if (in && has_front) front = ls[p - hw];
                    if (in && has_back) back = ls[p + hw];
                    // the real neighbours across the word's edges
                    uint32_t left = __shfl_up_sync(FSLIC_FULL, cur, 1), right = __shfl_down_sync(FSLIC_FULL, cur, 1);
                    if (lane == 0 && in && j > 0) left = ls[p - 1];
                    if (lane == last && j + 1 < W) right = ls[p + 1];
                    const bool ldiff = j == 0 || left != cur, rdiff = j + 1 == W || right != cur;
                    const uint32_t heads = __ballot_sync(FSLIC_FULL, in && (lane == 0 || left != cur));
                    const uint32_t U = __ballot_sync(FSLIC_FULL, in && (i == 0 || up != cur));
                    const uint32_t Dn = __ballot_sync(FSLIC_FULL, in && (i + 1 == H || down != cur));
                    const uint32_t F = __ballot_sync(FSLIC_FULL, in && (!has_front || front != cur));
                    const uint32_t Bk = __ballot_sync(FSLIC_FULL, in && (!has_back || back != cur));
                    const uint32_t R = __ballot_sync(FSLIC_FULL, in && rdiff);
                    if ((heads >> lane & 1u) && cur < (uint32_t)K) {
                        const uint32_t above = heads & ~((2u << lane) - 1u);
                        const int tail = above ? __ffs(above) - 2 : last;
                        const uint32_t run = ((2u << tail) - 1u) & ~((1u << lane) - 1u);
                        const long long a = j, e = j + (tail - lane), m = e - a + 1, y = i, zz = z;
                        const unsigned long long sx = (unsigned long long)((a + e) * m / 2);
                        Props3dAdd add;
                        add.area = (uint32_t)m;
                        add.surface = __popc(U & run) + __popc(Dn & run) + __popc(F & run) + __popc(Bk & run) +
                                      (ldiff ? 1u : 0u) + (R >> tail & 1u);
                        add.border = (z == 0 ? (uint32_t)m : 0u) + (z + 1 == D ? (uint32_t)m : 0u) +
                                     (i == 0 ? (uint32_t)m : 0u) + (i + 1 == H ? (uint32_t)m : 0u) +
                                     (a == 0 ? 1u : 0u) + (e + 1 == W ? 1u : 0u);
                        add.lo[0] = z;
                        add.lo[1] = i;
                        add.lo[2] = (int)a;
                        add.hi[0] = z + 1;
                        add.hi[1] = i + 1;
                        add.hi[2] = (int)e + 1;
                        add.m[0] = (unsigned long long)(zz * m);
                        add.m[1] = (unsigned long long)(y * m);
                        add.m[2] = sx;
                        add.m[3] = (unsigned long long)(zz * zz * m);
                        add.m[4] = (unsigned long long)(zz * y * m);
                        add.m[5] = (unsigned long long)zz * sx;
                        add.m[6] = (unsigned long long)(y * y * m);
                        add.m[7] = (unsigned long long)y * sx;
                        add.m[8] = props3d_sq_sum(e) - props3d_sq_sum(a - 1);
                        const int s = props3d_slot(t, cur);
                        if (s >= 0)
                            props3d_to_table(t, s, add);
                        else
                            props3d_to_global(o, node0 + cur, add);
                    }
                    up = cur;
                    cur = down;
                }
            }
            __syncthreads();
            // flush: one slot per thread, then free it for the next tile
            const uint32_t k = t.key[threadIdx.x];
            if (k != PROPS3D_EMPTY) {
                const int s = threadIdx.x;
                Props3dAdd a;
                a.area = t.area[s];
                a.surface = t.surface[s];
                a.border = t.border[s];
#pragma unroll
                for (int f = 0; f < 3; f++) {
                    a.lo[f] = t.lo[f][s];
                    a.hi[f] = t.hi[f][s];
                }
#pragma unroll
                for (int f = 0; f < PROPS3D_MOMENTS; f++) a.m[f] = t.m[f][s];
                props3d_to_global(o, node0 + k, a);
                props3d_slot_reset(t, s);
            }
            __syncthreads();
        }
    }
}

// One thread per node: centroid (sum z / n, sum y / n, sum x / n) and covariance (zz, zy, zx, yy, yx, xx), each
// sum ab / n - c_a c_b, each step one correctly rounded float64 operation; 0.0 and a zero box for an empty node
__global__ void __launch_bounds__(256) k_props3d_finish(long nodes, Props3dOut o, double* __restrict__ centroid,
                                                        double* __restrict__ covariance) {
    constexpr int A[6] = {0, 0, 0, 1, 1, 2}, B[6] = {0, 1, 2, 1, 2, 2};  // the axes of covariance entry f
    for (long n = (long)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (long)gridDim.x * blockDim.x) {
        const int area = o.area[n];
        double c[3] = {0.0, 0.0, 0.0}, v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        if (area == 0) {
#pragma unroll
            for (int f = 0; f < 6; f++) o.bbox[n * 6 + f] = 0;
        } else {
            const double a = (double)area;  // exact: area <= 2^29
            const unsigned long long* m = o.moments + n * PROPS3D_MOMENTS;
            double q[PROPS3D_MOMENTS];
#pragma unroll
            for (int f = 0; f < PROPS3D_MOMENTS; f++) q[f] = __ddiv_rn(__ll2double_rn((long long)m[f]), a);
#pragma unroll
            for (int f = 0; f < 3; f++) c[f] = q[f];
#pragma unroll
            for (int f = 0; f < 6; f++) v[f] = __dsub_rn(q[3 + f], __dmul_rn(c[A[f]], c[B[f]]));
        }
#pragma unroll
        for (int f = 0; f < 3; f++) centroid[n * 3 + f] = c[f];
#pragma unroll
        for (int f = 0; f < 6; f++) covariance[n * 6 + f] = v[f];
    }
}
