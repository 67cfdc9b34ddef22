// fast_slic_b200/csrc/props.cuh -- superpixel shapes (DESIGN.md section 4.15): per (image, label) the area, bounding
// box, raw first and second moments, crack perimeter and its image-edge part, then the centroid and central second
// moments in float64.  No counterpart in the reference.  Integer only up to the finishing kernel, whose float64 steps
// are each one IEEE-rounded operation: every result is exact and independent of the launch order.
//
//   k_props_init    one thread per node: zero sums, bbox minima at INT_MAX, maxima at 0;
//   k_props_tiles   one CTA per tile of PROPS_TILE_ROWS rows x PROPS_TILE_WORDS * 32 columns of one image; each warp
//                   walks one 32-column word down the tile's rows.  Per row a ballot of "label differs from the left
//                   neighbour" splits the word into runs; the head lane of each run adds its closed-form moments, box
//                   and perimeter sides to a shared table keyed by label (shared atomics), or straight to global
//                   memory when the table has no slot for it.  Each table entry is flushed to global memory once per
//                   tile (64-bit atomicAdd, 32-bit atomicAdd / atomicMin / atomicMax);
//   k_props_finish  one thread per node: centroid and covariance from the integer sums, empty boxes zeroed.
#pragma once
#include <limits.h>

#include "common.cuh"

#define PROPS_TILE_ROWS 32
#define PROPS_TILE_WORDS 8                     // one word per warp of the 256-thread CTA
#define PROPS_TABLE 256                        // table slots, a power of two
#define PROPS_PROBES 16                        // slots tried before a run goes to global memory
#define PROPS_EMPTY 0xffffffffu
#define PROPS_MOMENTS 5                        // sum y, sum x, sum y^2, sum xy, sum x^2

// The global outputs of one call, node n = b*K + k
struct PropsOut {
    int32_t* area;                  // [n]
    int32_t* bbox;                  // [n][4]: y0, x0 (min, inclusive), y1, x1 (max, exclusive)
    unsigned long long* moments;    // [n][5] (int64; every sum is non-negative)
    int32_t* perimeter;             // [n]
    int32_t* border;                // [n]
};

// What one run, or one table entry, adds to a node
struct PropsAdd {
    uint32_t area, perimeter, border;
    int y0, x0, y1, x1;
    unsigned long long m[PROPS_MOMENTS];
};

__device__ __forceinline__ void props_to_global(const PropsOut& o, long n, const PropsAdd& a) {
    atomicAdd(&o.area[n], (int)a.area);
    atomicAdd(&o.perimeter[n], (int)a.perimeter);
    atomicAdd(&o.border[n], (int)a.border);
    atomicMin(&o.bbox[n * 4 + 0], a.y0);
    atomicMin(&o.bbox[n * 4 + 1], a.x0);
    atomicMax(&o.bbox[n * 4 + 2], a.y1);
    atomicMax(&o.bbox[n * 4 + 3], a.x1);
#pragma unroll
    for (int f = 0; f < PROPS_MOMENTS; f++) atomicAdd(&o.moments[n * PROPS_MOMENTS + f], a.m[f]);
}

__global__ void __launch_bounds__(256) k_props_init(long nodes, PropsOut o) {
    for (long n = (long)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (long)gridDim.x * blockDim.x) {
        o.area[n] = 0;
        o.perimeter[n] = 0;
        o.border[n] = 0;
        o.bbox[n * 4 + 0] = INT_MAX;
        o.bbox[n * 4 + 1] = INT_MAX;
        o.bbox[n * 4 + 2] = 0;
        o.bbox[n * 4 + 3] = 0;
#pragma unroll
        for (int f = 0; f < PROPS_MOMENTS; f++) o.moments[n * PROPS_MOMENTS + f] = 0;
    }
}

// Sum of c^2 for c in [0, n], n >= -1
__device__ __forceinline__ unsigned long long props_sq_sum(long long n) {
    return (unsigned long long)(n * (n + 1) * (2 * n + 1) / 6);
}

// The shared table of one CTA: slot s holds label key[s] of the current tile (PROPS_EMPTY when free)
struct PropsTable {
    uint32_t key[PROPS_TABLE];
    uint32_t area[PROPS_TABLE], perimeter[PROPS_TABLE], border[PROPS_TABLE];
    int y0[PROPS_TABLE], x0[PROPS_TABLE], y1[PROPS_TABLE], x1[PROPS_TABLE];
    unsigned long long m[PROPS_MOMENTS][PROPS_TABLE];
};

__device__ __forceinline__ void props_slot_reset(PropsTable& t, int s) {
    t.key[s] = PROPS_EMPTY;
    t.area[s] = t.perimeter[s] = t.border[s] = 0;
    t.y0[s] = t.x0[s] = INT_MAX;
    t.y1[s] = t.x1[s] = 0;
#pragma unroll
    for (int f = 0; f < PROPS_MOMENTS; f++) t.m[f][s] = 0;
}

// The slot of label k in the table, claimed if k is new; -1 when PROPS_PROBES slots are taken by other labels
__device__ __forceinline__ int props_slot(PropsTable& t, uint32_t k) {
    int s = (int)((k * 2654435761u) >> 24) & (PROPS_TABLE - 1);
    for (int p = 0; p < PROPS_PROBES; p++) {
        const uint32_t cur = *(volatile uint32_t*)&t.key[s];
        if (cur == k) return s;
        if (cur == PROPS_EMPTY) {
            const uint32_t old = atomicCAS(&t.key[s], PROPS_EMPTY, k);
            if (old == PROPS_EMPTY || old == k) return s;
        }
        s = (s + 1) & (PROPS_TABLE - 1);
    }
    return -1;
}

__device__ __forceinline__ void props_to_table(PropsTable& t, int s, const PropsAdd& a) {
    atomicAdd(&t.area[s], a.area);
    atomicAdd(&t.perimeter[s], a.perimeter);
    atomicAdd(&t.border[s], a.border);
    atomicMin(&t.y0[s], a.y0);
    atomicMin(&t.x0[s], a.x0);
    atomicMax(&t.y1[s], a.y1);
    atomicMax(&t.x1[s], a.x1);
#pragma unroll
    for (int f = 0; f < PROPS_MOMENTS; f++) atomicAdd(&t.m[f][s], a.m[f]);
}

// Grid: y over images (looping past 65535), x over the tiles of an image (ceil(H / PROPS_TILE_ROWS) rows of
// ceil(Wd / PROPS_TILE_WORDS) tiles).  256 threads.  Outputs initialised by k_props_init.
__global__ void __launch_bounds__(256) k_props_tiles(const uint16_t* __restrict__ lab, int batch, int H, int W, int K,
                                                     PropsOut o) {
    __shared__ PropsTable t;
    const int Wd = (W + 31) / 32, tcols = (Wd + PROPS_TILE_WORDS - 1) / PROPS_TILE_WORDS;
    const int tiles = ((H + PROPS_TILE_ROWS - 1) / PROPS_TILE_ROWS) * tcols;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    props_slot_reset(t, threadIdx.x);
    __syncthreads();
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const uint16_t* l = lab + b * ((long)H * W);
        const long node0 = b * (long)K;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const int ty = tile / tcols, w = (tile - ty * tcols) * PROPS_TILE_WORDS + warp;
            const int i0 = ty * PROPS_TILE_ROWS, i1 = min(H, i0 + PROPS_TILE_ROWS);
            // warp-uniform: the warp's word, walked down rows i0 .. i1 - 1
            if (w < Wd) {
                const int j = w * 32 + lane;
                const bool in = j < W;
                const uint32_t valid = __ballot_sync(FSLIC_FULL, in);
                const int last = 31 - __clz(valid);
                uint32_t up = 0, cur = 0;
                if (in && i0 > 0) up = l[(long)(i0 - 1) * W + j];
                if (in) cur = l[(long)i0 * W + j];
                for (int i = i0; i < i1; i++) {
                    const long p = (long)i * W + j;
                    uint32_t down = 0;
                    if (in && i + 1 < H) down = l[p + W];
                    // the real neighbours across the word's edges
                    uint32_t left = __shfl_up_sync(FSLIC_FULL, cur, 1), right = __shfl_down_sync(FSLIC_FULL, cur, 1);
                    if (lane == 0 && in && j > 0) left = l[p - 1];
                    if (lane == last && j + 1 < W) right = l[p + 1];
                    const bool ldiff = j == 0 || left != cur, rdiff = j + 1 == W || right != cur;
                    const uint32_t heads = __ballot_sync(FSLIC_FULL, in && (lane == 0 || left != cur));
                    const uint32_t U = __ballot_sync(FSLIC_FULL, in && (i == 0 || up != cur));
                    const uint32_t D = __ballot_sync(FSLIC_FULL, in && (i + 1 == H || down != cur));
                    const uint32_t R = __ballot_sync(FSLIC_FULL, in && rdiff);
                    if ((heads >> lane & 1u) && cur < (uint32_t)K) {
                        const uint32_t above = heads & ~((2u << lane) - 1u);
                        const int tail = above ? __ffs(above) - 2 : last;
                        const uint32_t run = ((2u << tail) - 1u) & ~((1u << lane) - 1u);
                        const long long a = j, e = j + (tail - lane), m = e - a + 1, y = i;
                        const unsigned long long sx = (unsigned long long)((a + e) * m / 2);
                        PropsAdd add;
                        add.area = (uint32_t)m;
                        add.perimeter = __popc(U & run) + __popc(D & run) + (ldiff ? 1u : 0u) + (R >> tail & 1u);
                        add.border = (i == 0 ? (uint32_t)m : 0u) + (i + 1 == H ? (uint32_t)m : 0u) + (a == 0 ? 1u : 0u) +
                                     (e + 1 == W ? 1u : 0u);
                        add.y0 = i;
                        add.x0 = (int)a;
                        add.y1 = i + 1;
                        add.x1 = (int)e + 1;
                        add.m[0] = (unsigned long long)(y * m);
                        add.m[1] = sx;
                        add.m[2] = (unsigned long long)(y * y * m);
                        add.m[3] = (unsigned long long)y * sx;
                        add.m[4] = props_sq_sum(e) - props_sq_sum(a - 1);
                        const int s = props_slot(t, cur);
                        if (s >= 0)
                            props_to_table(t, s, add);
                        else
                            props_to_global(o, node0 + cur, add);
                    }
                    up = cur;
                    cur = down;
                }
            }
            __syncthreads();
            // flush: one slot per thread, then free it for the next tile
            const uint32_t k = t.key[threadIdx.x];
            if (k != PROPS_EMPTY) {
                const int s = threadIdx.x;
                PropsAdd a;
                a.area = t.area[s];
                a.perimeter = t.perimeter[s];
                a.border = t.border[s];
                a.y0 = t.y0[s];
                a.x0 = t.x0[s];
                a.y1 = t.y1[s];
                a.x1 = t.x1[s];
#pragma unroll
                for (int f = 0; f < PROPS_MOMENTS; f++) a.m[f] = t.m[f][s];
                props_to_global(o, node0 + k, a);
                props_slot_reset(t, s);
            }
            __syncthreads();
        }
    }
}

// One thread per node: centroid (sum y / n, sum x / n) and covariance (syy / n - cy cy, sxy / n - cy cx,
// sxx / n - cx cx), each step one correctly rounded float64 operation; 0.0 and a zero box for an empty node
__global__ void __launch_bounds__(256) k_props_finish(long nodes, PropsOut o, double* __restrict__ centroid,
                                                      double* __restrict__ covariance) {
    for (long n = (long)blockIdx.x * blockDim.x + threadIdx.x; n < nodes; n += (long)gridDim.x * blockDim.x) {
        const int area = o.area[n];
        double c[2] = {0.0, 0.0}, v[3] = {0.0, 0.0, 0.0};
        if (area == 0) {
#pragma unroll
            for (int f = 0; f < 4; f++) o.bbox[n * 4 + f] = 0;
        } else {
            const double a = (double)area;  // exact: area < 2^29
            const unsigned long long* m = o.moments + n * PROPS_MOMENTS;
            double q[PROPS_MOMENTS];
#pragma unroll
            for (int f = 0; f < PROPS_MOMENTS; f++) q[f] = __ddiv_rn(__ll2double_rn((long long)m[f]), a);
            c[0] = q[0];
            c[1] = q[1];
            v[0] = __dsub_rn(q[2], __dmul_rn(c[0], c[0]));
            v[1] = __dsub_rn(q[3], __dmul_rn(c[0], c[1]));
            v[2] = __dsub_rn(q[4], __dmul_rn(c[1], c[1]));
        }
        centroid[n * 2 + 0] = c[0];
        centroid[n * 2 + 1] = c[1];
#pragma unroll
        for (int f = 0; f < 3; f++) covariance[n * 3 + f] = v[f];
    }
}
