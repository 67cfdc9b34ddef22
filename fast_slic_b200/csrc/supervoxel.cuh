// fast_slic_b200/csrc/supervoxel.cuh -- SLIC over float32 volumes [B,C,D,H,W] (DESIGN.md section 4.22).  No
// counterpart in the reference.  Every float operation is one separately rounded IEEE operation (no contraction) in
// the order the contract gives, so a numpy restatement reproduces every bit:
//   distance   fc = +0; for c = 0 .. C-1: fc = fs_acc(fc, f_c, mu_c);  t_a = (float)v_a - c_a,
//              d = fc + ((w2z * (tz * tz) + w2y * (ty * ty)) + w2x * (tx * tx))
//   winner     the smallest dist_key(d, k) over the candidates |v_a - (int)c_a| <= R_a on every axis
//   update     c_a = (float)((double)sum v_a / (double)n) (exact integer sums), the feature means are pool's
//              (pool_stage.h) over the pass's voxels; a cluster without members keeps its centre and features.
//
// Centre state: pos [B,K,3] (z, y, x), feat [B,K,C].  Before every pass k_sv_grid counting-sorts the centres into
// buckets of pitch G_a >= R_a (at most SV_MAX_CELLS of them, capi_supervoxel.cu), so the candidates of a voxel lie in
// at most 3 x 3 x 3 buckets and a tile finds every centre whose window may reach it in a few ranges.
#pragma once
#include "cellgrid.cuh"
#include "common.cuh"

#define SV_TILE_W 16     // columns of an assign tile (one half-warp along a row)
#define SV_TILE_R 4      // pass rows of an assign tile
#define SV_TILE_D 4      // slices of an assign tile: one half-warp per (slice, pass row)
#define SV_THREADS (SV_TILE_W * SV_TILE_R * SV_TILE_D)
#define SV_MAXC 64       // candidates a tile keeps in registers; a tile with more goes to k_sv_assign_fallback
#define SV_CH 32         // channels of the centroid features staged in shared memory at a time
#define SV_NO_LABEL 0xffffu

struct SvParams {
    int D, H, W, C, K;
    int nd, nh, nw;            // the seed grid, K = nd * nh * nw
    int Rz, Ry, Rx;            // window radii ceil(L_a / n_a)
    int Gz, Gy, Gx;            // bucket pitches >= R_a
    int cellsY, cellsX, ncell; // buckets along y and x, and in all
    float w2z, w2y, w2x;
    int r, s, npr;             // the pass visits rows r, r + s, .., npr of them in every slice
    int tiles_x, tiles_y, tiles;  // tiles along x and along the pass rows, and per volume
};

__device__ __forceinline__ unsigned long long sv_key(float fc, int z, int y, int x, float cz, float cy, float cx,
                                                     const SvParams& p, int k) {
    const float tz = __fsub_rn((float)z, cz), ty = __fsub_rn((float)y, cy), tx = __fsub_rn((float)x, cx);
    const float sp = __fadd_rn(__fadd_rn(__fmul_rn(p.w2z, __fmul_rn(tz, tz)), __fmul_rn(p.w2y, __fmul_rn(ty, ty))),
                               __fmul_rn(p.w2x, __fmul_rn(tx, tx)));
    return dist_key(__fadd_rn(fc, sp), k);
}

__device__ __forceinline__ bool sv_in_window(int z, int y, int x, float cz, float cy, float cx, const SvParams& p) {
    return abs(z - (int)cz) <= p.Rz && abs(y - (int)cy) <= p.Ry && abs(x - (int)cx) <= p.Rx;
}

__device__ __forceinline__ int sv_cell(const SvParams& p, float cz, float cy, float cx) {
    return ((int)cz / p.Gz * p.cellsY + (int)cy / p.Gy) * p.cellsX + (int)cx / p.Gx;
}

// The integer centre of cell i of n on an axis of length L: (lo + hi - 1) / 2 of [iL/n, (i+1)L/n)
__device__ __forceinline__ int sv_centre(int i, int L, int n) {
    return (int)(((long)i * L / n + (long)(i + 1) * L / n - 1) / 2);
}

// The seeds, one thread per (volume, cluster, channel): cluster k = (iz * nh + iy) * nw + ix sits at the centre of its
// cell with the features of that voxel.  count = 0.
__global__ void __launch_bounds__(256) k_sv_seed(SvParams p, const float* __restrict__ vol, long nkc,
                                                 float* __restrict__ pos, float* __restrict__ feat,
                                                 int32_t* __restrict__ count) {
    const long n = (long)p.D * p.H * p.W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nkc; t += (long)gridDim.x * blockDim.x) {
        const long bk = t / p.C;
        const int c = (int)(t - bk * p.C);
        const long b = bk / p.K;
        const int k = (int)(bk - b * p.K);
        const int ix = k % p.nw, iy = (k / p.nw) % p.nh, iz = k / (p.nw * p.nh);
        const int z = sv_centre(iz, p.D, p.nd), y = sv_centre(iy, p.H, p.nh), x = sv_centre(ix, p.W, p.nw);
        feat[t] = vol[(b * p.C + c) * n + ((long)z * p.H + y) * p.W + x];
        if (c == 0) {
            pos[3 * bk] = (float)z;
            pos[3 * bk + 1] = (float)y;
            pos[3 * bk + 2] = (float)x;
            count[bk] = 0;
        }
    }
}

// The buckets of volume blockIdx.x: rec [K] = the cluster indices sorted by bucket, in any order inside one;
// cell_start [ncell + 1] = the first slot of each bucket.  1024 threads, (ncell + 1) ints of dynamic shared memory.
__global__ void __launch_bounds__(1024) k_sv_grid(SvParams p, const float* __restrict__ pos,
                                                  int* __restrict__ cell_start, uint32_t* __restrict__ rec) {
    extern __shared__ int s_cnt[];
    __shared__ int s_warp[32];
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const float* ps = pos + (size_t)b * p.K * 3;
    int* cs = cell_start + (size_t)b * (p.ncell + 1);
    for (int c = tid; c <= p.ncell; c += nt) s_cnt[c] = 0;
    __syncthreads();
    for (int k = tid; k < p.K; k += nt) atomicAdd(&s_cnt[sv_cell(p, ps[3 * k], ps[3 * k + 1], ps[3 * k + 2])], 1);
    scan_cells(s_cnt, s_warp, cs, p.ncell + 1, tid, nt);
    for (int k = tid; k < p.K; k += nt) {
        const int slot = atomicAdd(&s_cnt[sv_cell(p, ps[3 * k], ps[3 * k + 1], ps[3 * k + 2])], 1);
        rec[(size_t)b * p.K + slot] = (uint32_t)k;
    }
}

// The tile `tile` of a pass: its box (slices z0..z1, pass rows m0..m1, columns c0..c1) and the voxel of this thread
struct SvTile {
    int z0, z1, m0, m1, c0, c1, z, y, x;
    bool valid;
};

__device__ __forceinline__ SvTile sv_tile(const SvParams& p, int tile) {
    SvTile t;
    const int tx = tile % p.tiles_x, rest = tile / p.tiles_x;
    const int ty = rest % p.tiles_y, tz = rest / p.tiles_y;
    t.c0 = tx * SV_TILE_W;
    t.c1 = min(t.c0 + SV_TILE_W - 1, p.W - 1);
    t.m0 = ty * SV_TILE_R;
    t.m1 = min(t.m0 + SV_TILE_R - 1, p.npr - 1);
    t.z0 = tz * SV_TILE_D;
    t.z1 = min(t.z0 + SV_TILE_D - 1, p.D - 1);
    const int w = (int)(threadIdx.x / SV_TILE_W);
    const int m = t.m0 + w % SV_TILE_R;
    t.z = t.z0 + w / SV_TILE_R;
    t.x = t.c0 + (int)(threadIdx.x % SV_TILE_W);
    t.y = p.r + m * p.s;
    t.valid = m <= t.m1 && t.z <= t.z1 && t.x <= t.c1;
    return t;
}

// The channel loop of a tile with nc <= NB candidates, as fs_tile_body: every voxel reads f_c once per channel and adds
// it to one accumulator per candidate, so each (voxel, candidate) sum runs over the channels in order.  Then the window
// test, the spatial term and the smallest key.
template <int NB>
__device__ __forceinline__ void sv_tile_body(const SvParams& p, const SvTile& t, int b, int nc,
                                             const float* __restrict__ vol, const float* __restrict__ feat,
                                             const int* s_k, const float* s_c, float* s_mu,
                                             uint16_t* __restrict__ labels) {
    const long n = (long)p.D * p.H * p.W;
    const long v = ((long)t.z * p.H + t.y) * p.W + t.x;
    const float* fp = vol + (long)b * p.C * n + v;
    float acc[NB];
#pragma unroll
    for (int q = 0; q < NB; q++) acc[q] = 0.f;
    for (int cb = 0; cb < p.C; cb += SV_CH) {
        const int cn = min(SV_CH, p.C - cb);
        __syncthreads();  // the previous chunk is consumed
        for (int e = threadIdx.x; e < nc * cn; e += blockDim.x) {
            const int q = e / cn, cc = e - q * cn;
            s_mu[cc * SV_MAXC + q] = feat[((long)b * p.K + s_k[q]) * p.C + cb + cc];
        }
        __syncthreads();
#pragma unroll 2
        for (int cc = 0; cc < cn; cc++) {
            const float x = t.valid ? __ldg(fp + (long)(cb + cc) * n) : 0.f;
            const float4* mu4 = reinterpret_cast<const float4*>(s_mu + cc * SV_MAXC);
#pragma unroll
            for (int q4 = 0; q4 < NB / 4; q4++) {
                const float4 m = mu4[q4];
                acc[4 * q4 + 0] = fs_acc(acc[4 * q4 + 0], x, m.x);
                acc[4 * q4 + 1] = fs_acc(acc[4 * q4 + 1], x, m.y);
                acc[4 * q4 + 2] = fs_acc(acc[4 * q4 + 2], x, m.z);
                acc[4 * q4 + 3] = fs_acc(acc[4 * q4 + 3], x, m.w);
            }
        }
    }
    if (!t.valid) return;
    unsigned long long best = ~0ull;
#pragma unroll
    for (int q = 0; q < NB; q++) {
        if (q < nc) {
            const float cz = s_c[3 * q], cy = s_c[3 * q + 1], cx = s_c[3 * q + 2];
            if (sv_in_window(t.z, t.y, t.x, cz, cy, cx, p)) {
                const unsigned long long key = sv_key(acc[q], t.z, t.y, t.x, cz, cy, cx, p, s_k[q]);
                best = key < best ? key : best;
            }
        }
    }
    if (best != ~0ull) labels[(long)b * n + v] = (uint16_t)(uint32_t)best;
}

// The assign kernel of a pass: one CTA of SV_THREADS per tile of SV_TILE_W columns x SV_TILE_R pass rows x SV_TILE_D
// slices (grid: tiles of a volume x volumes).  A tile's candidates are the centres within R_a of its box, about
// prod_a (extent_a + 2 R_a) / cell_a + 1 of them, so a compact box keeps the count under SV_MAXC at the usual radii.  The CTA collects the centres whose window may reach the
// tile from the buckets; with more than SV_MAXC it appends the tile to ovf_list (ovf_count counts them) and leaves it
// to k_sv_assign_fallback.  A voxel without a candidate keeps its label.
__global__ void __launch_bounds__(SV_THREADS) k_sv_assign_tiles(
    SvParams p, const float* __restrict__ vol, const float* __restrict__ feat, const float* __restrict__ pos,
    const int* __restrict__ cell_start, const uint32_t* __restrict__ rec, uint16_t* __restrict__ labels,
    int* __restrict__ ovf_count, int* __restrict__ ovf_list) {
    __shared__ int s_n;
    __shared__ int s_k[SV_MAXC];
    __shared__ float s_c[3 * SV_MAXC];
    __shared__ __align__(16) float s_mu[SV_CH * SV_MAXC];
    const int b = blockIdx.y, tile = blockIdx.x;
    const SvTile t = sv_tile(p, tile);
    const int ymin = p.r + t.m0 * p.s, ymax = p.r + t.m1 * p.s;
    const int bz0 = max(t.z0 - p.Rz, 0) / p.Gz, bz1 = min(t.z1 + p.Rz, p.D - 1) / p.Gz;
    const int by0 = max(ymin - p.Ry, 0) / p.Gy, by1 = min(ymax + p.Ry, p.H - 1) / p.Gy;
    const int bx0 = max(t.c0 - p.Rx, 0) / p.Gx, bx1 = min(t.c1 + p.Rx, p.W - 1) / p.Gx;
    const int nby = by1 - by0 + 1, nrows = (bz1 - bz0 + 1) * nby;
    const int* cs = cell_start + (size_t)b * (p.ncell + 1);
    const uint32_t* rc = rec + (size_t)b * p.K;
    const float* ps = pos + (size_t)b * p.K * 3;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int q = (int)(threadIdx.x >> 5); q < nrows; q += SV_THREADS / 32) {
        const int row = ((bz0 + q / nby) * p.cellsY + by0 + q % nby) * p.cellsX;
        const int hi = cs[row + bx1 + 1];
        for (int e = cs[row + bx0] + (int)(threadIdx.x & 31); e < hi; e += 32) {
            const int k = (int)rc[e];
            const float cz = ps[3 * k], cy = ps[3 * k + 1], cx = ps[3 * k + 2];
            const int iz = (int)cz, iy = (int)cy, ix = (int)cx;
            if (iz >= t.z0 - p.Rz && iz <= t.z1 + p.Rz && iy >= ymin - p.Ry && iy <= ymax + p.Ry &&
                ix >= t.c0 - p.Rx && ix <= t.c1 + p.Rx) {
                const int slot = atomicAdd(&s_n, 1);
                if (slot < SV_MAXC) {
                    s_k[slot] = k;
                    s_c[3 * slot] = cz;
                    s_c[3 * slot + 1] = cy;
                    s_c[3 * slot + 2] = cx;
                }
            }
        }
    }
    __syncthreads();
    const int nc = s_n;
    if (nc > SV_MAXC) {
        if (threadIdx.x == 0) ovf_list[atomicAdd(ovf_count, 1)] = b * p.tiles + tile;
        return;
    }
    if (nc == 0) return;
    if (nc <= 16) sv_tile_body<16>(p, t, b, nc, vol, feat, s_k, s_c, s_mu, labels);
    else if (nc <= 32) sv_tile_body<32>(p, t, b, nc, vol, feat, s_k, s_c, s_mu, labels);
    else sv_tile_body<64>(p, t, b, nc, vol, feat, s_k, s_c, s_mu, labels);
}

// The overflow path: the tiles k_sv_assign_tiles listed, one thread per voxel, each walking the buckets its window
// touches and computing every candidate's distance with the same fs_acc / sv_key.  A grid-stride loop over the list.
__global__ void __launch_bounds__(SV_THREADS) k_sv_assign_fallback(
    SvParams p, const float* __restrict__ vol, const float* __restrict__ feat, const float* __restrict__ pos,
    const int* __restrict__ cell_start, const uint32_t* __restrict__ rec, uint16_t* __restrict__ labels,
    const int* __restrict__ ovf_count, const int* __restrict__ ovf_list) {
    const long n = (long)p.D * p.H * p.W;
    const int total = *ovf_count;
    for (int e = blockIdx.x; e < total; e += gridDim.x) {
        const int id = ovf_list[e];
        const int b = id / p.tiles;
        const SvTile t = sv_tile(p, id - b * p.tiles);
        if (!t.valid) continue;
        const int* cs = cell_start + (size_t)b * (p.ncell + 1);
        const uint32_t* rc = rec + (size_t)b * p.K;
        const float* ps = pos + (size_t)b * p.K * 3;
        const long v = ((long)t.z * p.H + t.y) * p.W + t.x;
        const float* fp = vol + (long)b * p.C * n + v;
        const int bz0 = max(t.z - p.Rz, 0) / p.Gz, bz1 = min(t.z + p.Rz, p.D - 1) / p.Gz;
        const int by0 = max(t.y - p.Ry, 0) / p.Gy, by1 = min(t.y + p.Ry, p.H - 1) / p.Gy;
        const int bx0 = max(t.x - p.Rx, 0) / p.Gx, bx1 = min(t.x + p.Rx, p.W - 1) / p.Gx;
        unsigned long long best = ~0ull;
        for (int bz = bz0; bz <= bz1; bz++) {
            for (int by = by0; by <= by1; by++) {
                const int row = (bz * p.cellsY + by) * p.cellsX;
                const int hi = cs[row + bx1 + 1];
                for (int q = cs[row + bx0]; q < hi; q++) {
                    const int k = (int)rc[q];
                    const float cz = ps[3 * k], cy = ps[3 * k + 1], cx = ps[3 * k + 2];
                    if (!sv_in_window(t.z, t.y, t.x, cz, cy, cx, p)) continue;
                    const float* mu = feat + ((long)b * p.K + k) * p.C;
                    float fc = 0.f;
                    for (int c = 0; c < p.C; c++) fc = fs_acc(fc, __ldg(fp + (long)c * n), mu[c]);
                    const unsigned long long key = sv_key(fc, t.z, t.y, t.x, cz, cy, cx, p, k);
                    best = key < best ? key : best;
                }
            }
        }
        if (best != ~0ull) labels[(long)b * n + v] = (uint16_t)(uint32_t)best;
    }
}

// The pool keys of a pass (pool_stage.h): keys[t] = volume << 16 | label (0xffff outside [0, K)), vals[t] = the voxel
// index, over the pass rows of every slice of `batch` volumes in raster order (total = batch * D * npr * W)
__global__ void __launch_bounds__(256) k_sv_keys(SvParams p, const uint16_t* __restrict__ labels, long total,
                                                 uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const long per = (long)p.D * p.npr * p.W, n = (long)p.D * p.H * p.W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long b = t / per, rem = t - b * per;
        const long zm = rem / p.W, x = rem - zm * p.W;
        const long z = zm / p.npr, m = zm - z * p.npr;
        const long v = (z * p.H + p.r + m * p.s) * p.W + x;
        const uint32_t l = labels[b * n + v];
        keys[t] = (uint32_t)b << 16 | (l < (uint32_t)p.K ? l : SV_NO_LABEL);
        vals[t] = (uint32_t)v;
    }
}

// The update after a pass, one warp per (volume, cluster) over pool's sorted segments: the exact integer sums of the
// members' z, y and x give the centre, and the pooled means (means [B,C,K]) become feat [B,K,C].  A cluster without
// members keeps both.
__global__ void __launch_bounds__(256) k_sv_update(SvParams p, long nk, const uint32_t* __restrict__ seg_start,
                                                   const uint32_t* __restrict__ seg_end,
                                                   const uint32_t* __restrict__ members, const float* __restrict__ means,
                                                   float* __restrict__ pos, float* __restrict__ feat) {
    const long seg = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (seg >= nk) return;  // the whole warp leaves together
    const uint32_t s = seg_start[seg], e = seg_end[seg];
    if (e == s) return;
    const uint32_t hw = (uint32_t)p.H * (uint32_t)p.W;
    unsigned long long sz = 0, sy = 0, sx = 0;
    for (uint32_t q = s + lane; q < e; q += 32) {
        const uint32_t v = members[q];
        const uint32_t z = v / hw, rem = v - z * hw;
        const uint32_t y = rem / (uint32_t)p.W;
        sz += z;
        sy += y;
        sx += rem - y * (uint32_t)p.W;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        sz += __shfl_xor_sync(FSLIC_FULL, sz, off);
        sy += __shfl_xor_sync(FSLIC_FULL, sy, off);
        sx += __shfl_xor_sync(FSLIC_FULL, sx, off);
    }
    if (lane == 0) {
        const double cnt = (double)(e - s);
        pos[3 * seg] = __double2float_rn(__ddiv_rn((double)sz, cnt));
        pos[3 * seg + 1] = __double2float_rn(__ddiv_rn((double)sy, cnt));
        pos[3 * seg + 2] = __double2float_rn(__ddiv_rn((double)sx, cnt));
    }
    const long b = seg / p.K, k = seg - b * p.K;
    for (int c = lane; c < p.C; c += 32) feat[seg * p.C + c] = means[(b * p.C + c) * p.K + k];
}
