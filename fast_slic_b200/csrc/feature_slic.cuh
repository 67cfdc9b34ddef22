// fast_slic_b200/csrc/feature_slic.cuh -- SLIC over float feature maps [B,C,H,W] (DESIGN.md section 4.19).  No
// counterpart in the reference.  Every float operation is one separately rounded IEEE operation (no contraction) in
// the order the contract gives, so a numpy restatement reproduces every bit:
//   distance   fc = +0; for c = 0 .. C-1: t = f_c - mu_c, fc = fc + t * t;
//              ty = i - cy, tx = j - cx, d = fc + w2 * (ty * ty + tx * tx), w2 = (compactness / S)^2
//   winner     the smallest key (bits(d) << 32 | k) over the candidates |i - (int)cy| <= S, |j - (int)cx| <= S, a NaN
//              distance having the bits 0x7fffffff: ties go to the lower k, non-finite distances lose to finite ones
//   update     cy = (float)((double)sum_i / (double)n) and the same for cx (exact integer sums), the feature means are
//              pool's (pool.cuh) over the pass's rows; a cluster without members keeps its centre and features.
//
// Centre state: pos [B,K,2] (y, x), feat [B,K,C].  Before every pass k_fs_grid sorts the centres into a cell grid of
// pitch G >= S (cellgrid.cuh's scan), so a tile finds every centre whose window may reach it in a few ranges.
#pragma once
#include "cellgrid.cuh"
#include "common.cuh"

#define FS_TILE_W 32     // columns of an assign tile (one warp along a row)
#define FS_TILE_R 8      // pass rows of an assign tile (one per warp)
#define FS_MAXC 32       // candidates a tile keeps in registers; a tile with more goes to k_fs_assign_fallback
#define FS_CH 32         // channels of the centroid features staged in shared memory at a time
#define FS_NO_LABEL 0xffffu

struct FsParams {
    int H, W, C, K, S;
    int G, cellW, ncell;
    float w2;            // (compactness / S)^2, each step rounded
    int r, s, npr;       // the pass visits rows r, r + s, .., npr of them
    int tiles_x, tiles;  // tiles per pass row band and per image
};

// The packed key of candidate k of pixel (i, j) from its feature distance fc
__device__ __forceinline__ unsigned long long fs_key(float fc, int i, int j, float cy, float cx, float w2, int k) {
    const float ty = __fsub_rn((float)i, cy), tx = __fsub_rn((float)j, cx);
    return dist_key(__fadd_rn(fc, __fmul_rn(w2, __fadd_rn(__fmul_rn(ty, ty), __fmul_rn(tx, tx)))), k);
}

__device__ __forceinline__ bool fs_in_window(int i, int j, float cy, float cx, int S) {
    return abs(i - (int)cy) <= S && abs(j - (int)cx) <= S;
}

// The seeds, one thread per (image, cluster, channel): the grid centre of initialize_clusters and the features of its
// pixel, or the clamped init_pos (fminf / fmaxf send NaN to 0) and init_feat as given.  count = 0.
__global__ void __launch_bounds__(256) k_fs_seed(const float* __restrict__ features, const float* __restrict__ init_pos,
                                                 const float* __restrict__ init_feat, long nkc, int H, int W, int C,
                                                 int K, float* __restrict__ pos, float* __restrict__ feat,
                                                 int32_t* __restrict__ count) {
    const long hw = (long)H * W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nkc; t += (long)gridDim.x * blockDim.x) {
        const long bk = t / C;
        const int c = (int)(t - bk * C);
        const long b = bk / K;
        const int k = (int)(bk - b * K);
        if (init_pos) {
            feat[t] = init_feat[t];
            if (c == 0) {
                pos[2 * bk] = fminf(fmaxf(init_pos[2 * bk], 0.f), (float)(H - 1));
                pos[2 * bk + 1] = fminf(fmaxf(init_pos[2 * bk + 1], 0.f), (float)(W - 1));
                count[bk] = 0;
            }
            continue;
        }
        int cy, cx;
        init_grid_centre(k, H, W, K, cy, cx);
        feat[t] = features[(b * C + c) * hw + (long)cy * W + cx];
        if (c == 0) {
            pos[2 * bk] = (float)cy;
            pos[2 * bk + 1] = (float)cx;
            count[bk] = 0;
        }
    }
}

// The cell grid of image blockIdx.x: rec [K] = the cluster indices sorted by the cell of ((int)cy, (int)cx), in any
// order inside a cell; cell_start [ncell + 1] = the first slot of each cell.  1024 threads, (ncell + 1) ints of
// dynamic shared memory.
__global__ void __launch_bounds__(1024) k_fs_grid(FsParams p, const float* __restrict__ pos,
                                                  int* __restrict__ cell_start, uint32_t* __restrict__ rec) {
    extern __shared__ int s_cnt[];
    __shared__ int s_warp[32];
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const float* ps = pos + (size_t)b * p.K * 2;
    int* cs = cell_start + (size_t)b * (p.ncell + 1);
    for (int c = tid; c <= p.ncell; c += nt) s_cnt[c] = 0;
    __syncthreads();
    for (int k = tid; k < p.K; k += nt) atomicAdd(&s_cnt[((int)ps[2 * k] / p.G) * p.cellW + (int)ps[2 * k + 1] / p.G], 1);
    scan_cells(s_cnt, s_warp, cs, p.ncell + 1, tid, nt);
    for (int k = tid; k < p.K; k += nt) {
        const int slot = atomicAdd(&s_cnt[((int)ps[2 * k] / p.G) * p.cellW + (int)ps[2 * k + 1] / p.G], 1);
        rec[(size_t)b * p.K + slot] = (uint32_t)k;
    }
}

// The tile `tile` of a pass: its first column and pass row, and the pixel (i, j) of thread (lane, warp)
struct FsTile {
    int c0, c1, m0, m1, i, j;
    bool valid;
};

__device__ __forceinline__ FsTile fs_tile(const FsParams& p, int tile) {
    FsTile t;
    const int tx = tile % p.tiles_x, ty = tile / p.tiles_x;
    t.c0 = tx * FS_TILE_W;
    t.c1 = min(t.c0 + FS_TILE_W - 1, p.W - 1);
    t.m0 = ty * FS_TILE_R;
    t.m1 = min(t.m0 + FS_TILE_R - 1, p.npr - 1);
    const int m = t.m0 + (int)(threadIdx.x >> 5);
    t.j = t.c0 + (int)(threadIdx.x & 31);
    t.i = p.r + m * p.s;
    t.valid = m <= t.m1 && t.j <= t.c1;
    return t;
}

// The channel loop of a tile with nc <= NB candidates: every pixel reads f_c once per channel and adds it to one
// accumulator per candidate, so each (pixel, candidate) sum runs over the channels in order.  Then the window test,
// the spatial term and the smallest key.
template <int NB>
__device__ __forceinline__ void fs_tile_body(const FsParams& p, const FsTile& t, int b, int nc,
                                             const float* __restrict__ features, const float* __restrict__ feat,
                                             const int* s_k, const float* s_cy, const float* s_cx, float* s_mu,
                                             uint16_t* __restrict__ labels) {
    const long hw = (long)p.H * p.W;
    const float* fp = features + (long)b * p.C * hw + (long)t.i * p.W + t.j;
    float acc[NB];
#pragma unroll
    for (int q = 0; q < NB; q++) acc[q] = 0.f;
    for (int cb = 0; cb < p.C; cb += FS_CH) {
        const int cn = min(FS_CH, p.C - cb);
        __syncthreads();  // the previous chunk is consumed
        for (int e = threadIdx.x; e < nc * cn; e += blockDim.x) {
            const int q = e / cn, cc = e - q * cn;
            s_mu[cc * FS_MAXC + q] = feat[((long)b * p.K + s_k[q]) * p.C + cb + cc];
        }
        __syncthreads();
#pragma unroll 4
        for (int cc = 0; cc < cn; cc++) {
            const float x = t.valid ? __ldg(fp + (long)(cb + cc) * hw) : 0.f;
            const float4* mu4 = reinterpret_cast<const float4*>(s_mu + cc * FS_MAXC);
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
        if (q < nc && fs_in_window(t.i, t.j, s_cy[q], s_cx[q], p.S)) {
            const unsigned long long key = fs_key(acc[q], t.i, t.j, s_cy[q], s_cx[q], p.w2, s_k[q]);
            best = key < best ? key : best;
        }
    }
    if (best != ~0ull) labels[(long)b * hw + (long)t.i * p.W + t.j] = (uint16_t)(uint32_t)best;
}

// The assign kernel of a pass: one CTA of FS_TILE_R warps per tile of FS_TILE_W columns x FS_TILE_R pass rows
// (grid: tiles of an image x images).  The CTA collects the centres whose window may reach the tile from the cell
// grid; with more than FS_MAXC it appends the tile to ovf_list (ovf_count counts them) and leaves it to
// k_fs_assign_fallback.  A pixel without a candidate keeps its label.
__global__ void __launch_bounds__(FS_TILE_W * FS_TILE_R) k_fs_assign_tiles(
    FsParams p, const float* __restrict__ features, const float* __restrict__ feat, const float* __restrict__ pos,
    const int* __restrict__ cell_start, const uint32_t* __restrict__ rec, uint16_t* __restrict__ labels,
    int* __restrict__ ovf_count, int* __restrict__ ovf_list) {
    __shared__ int s_n;
    __shared__ int s_k[FS_MAXC];
    __shared__ float s_cy[FS_MAXC], s_cx[FS_MAXC];
    __shared__ __align__(16) float s_mu[FS_CH * FS_MAXC];
    const int b = blockIdx.y, tile = blockIdx.x;
    const FsTile t = fs_tile(p, tile);
    const int rmin = p.r + t.m0 * p.s, rmax = p.r + t.m1 * p.s;
    const int cr0 = max(rmin - p.S, 0) / p.G, cr1 = min(rmax + p.S, p.H - 1) / p.G;
    const int cc0 = max(t.c0 - p.S, 0) / p.G, cc1 = min(t.c1 + p.S, p.W - 1) / p.G;
    const int* cs = cell_start + (size_t)b * (p.ncell + 1);
    const uint32_t* rc = rec + (size_t)b * p.K;
    const float* ps = pos + (size_t)b * p.K * 2;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int cr = cr0 + (int)(threadIdx.x >> 5); cr <= cr1; cr += FS_TILE_R) {
        const int hi = cs[cr * p.cellW + cc1 + 1];
        for (int e = cs[cr * p.cellW + cc0] + (int)(threadIdx.x & 31); e < hi; e += 32) {
            const int k = (int)rc[e];
            const float2 c = *reinterpret_cast<const float2*>(ps + 2 * k);  // (y, x)
            const int iy = (int)c.x, ix = (int)c.y;
            if (iy >= rmin - p.S && iy <= rmax + p.S && ix >= t.c0 - p.S && ix <= t.c1 + p.S) {
                const int slot = atomicAdd(&s_n, 1);
                if (slot < FS_MAXC) {
                    s_k[slot] = k;
                    s_cy[slot] = c.x;
                    s_cx[slot] = c.y;
                }
            }
        }
    }
    __syncthreads();
    const int nc = s_n;
    if (nc > FS_MAXC) {
        if (threadIdx.x == 0) ovf_list[atomicAdd(ovf_count, 1)] = b * p.tiles + tile;
        return;
    }
    if (nc == 0) return;
    if (nc <= 8) fs_tile_body<8>(p, t, b, nc, features, feat, s_k, s_cy, s_cx, s_mu, labels);
    else if (nc <= 16) fs_tile_body<16>(p, t, b, nc, features, feat, s_k, s_cy, s_cx, s_mu, labels);
    else fs_tile_body<32>(p, t, b, nc, features, feat, s_k, s_cy, s_cx, s_mu, labels);
}

// The overflow path: the tiles k_fs_assign_tiles listed, one thread per pixel, each walking the cells its window
// touches and computing every candidate's distance with the same fs_acc / fs_key.  A grid-stride loop over the list,
// so a fixed grid covers any count.
__global__ void __launch_bounds__(FS_TILE_W * FS_TILE_R) k_fs_assign_fallback(
    FsParams p, const float* __restrict__ features, const float* __restrict__ feat, const float* __restrict__ pos,
    const int* __restrict__ cell_start, const uint32_t* __restrict__ rec, uint16_t* __restrict__ labels,
    const int* __restrict__ ovf_count, const int* __restrict__ ovf_list) {
    const long hw = (long)p.H * p.W;
    const int n = *ovf_count;
    for (int e = blockIdx.x; e < n; e += gridDim.x) {
        const int id = ovf_list[e];
        const int b = id / p.tiles;
        const FsTile t = fs_tile(p, id - b * p.tiles);
        if (!t.valid) continue;
        const int* cs = cell_start + (size_t)b * (p.ncell + 1);
        const uint32_t* rc = rec + (size_t)b * p.K;
        const float* ps = pos + (size_t)b * p.K * 2;
        const float* fp = features + (long)b * p.C * hw + (long)t.i * p.W + t.j;
        const int cr0 = max(t.i - p.S, 0) / p.G, cr1 = min(t.i + p.S, p.H - 1) / p.G;
        const int cc0 = max(t.j - p.S, 0) / p.G, cc1 = min(t.j + p.S, p.W - 1) / p.G;
        unsigned long long best = ~0ull;
        for (int cr = cr0; cr <= cr1; cr++) {
            const int hi = cs[cr * p.cellW + cc1 + 1];
            for (int q = cs[cr * p.cellW + cc0]; q < hi; q++) {
                const int k = (int)rc[q];
                const float cy = ps[2 * k], cx = ps[2 * k + 1];
                if (!fs_in_window(t.i, t.j, cy, cx, p.S)) continue;
                const float* mu = feat + ((long)b * p.K + k) * p.C;
                float fc = 0.f;
                for (int c = 0; c < p.C; c++) fc = fs_acc(fc, __ldg(fp + (long)c * hw), mu[c]);
                const unsigned long long key = fs_key(fc, t.i, t.j, cy, cx, p.w2, k);
                best = key < best ? key : best;
            }
        }
        if (best != ~0ull) labels[(long)b * hw + (long)t.i * p.W + t.j] = (uint16_t)(uint32_t)best;
    }
}

// The pool keys of a pass (pool_stage.h): keys[t] = image << 16 | label (0xffff outside [0, K)), vals[t] = the pixel
// index, over the pass rows of `batch` images in raster order (n = batch * npr * W)
__global__ void __launch_bounds__(256) k_fs_keys(FsParams p, const uint16_t* __restrict__ labels, long n,
                                                 uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const long per = (long)p.npr * p.W, hw = (long)p.H * p.W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const long b = t / per, rem = t - b * per;
        const long m = rem / p.W, j = rem - m * p.W;
        const long px = (p.r + m * p.s) * p.W + j;
        const uint32_t l = labels[b * hw + px];
        keys[t] = (uint32_t)b << 16 | (l < (uint32_t)p.K ? l : FS_NO_LABEL);
        vals[t] = (uint32_t)px;
    }
}

// The update after a pass, one warp per (image, cluster) over pool's sorted segments: the exact integer sums of the
// members' rows and columns give the centre, and the pooled means (means [B,C,K]) become feat [B,K,C].  A cluster
// without members keeps both.
__global__ void __launch_bounds__(256) k_fs_update(FsParams p, long nk, const uint32_t* __restrict__ seg_start,
                                                   const uint32_t* __restrict__ seg_end,
                                                   const uint32_t* __restrict__ members, const float* __restrict__ means,
                                                   float* __restrict__ pos, float* __restrict__ feat) {
    const long seg = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (seg >= nk) return;  // the whole warp leaves together
    const uint32_t s = seg_start[seg], e = seg_end[seg];
    if (e == s) return;
    unsigned long long si = 0, sj = 0;
    for (uint32_t q = s + lane; q < e; q += 32) {
        const uint32_t px = members[q];
        const uint32_t i = px / (uint32_t)p.W;
        si += i;
        sj += px - i * (uint32_t)p.W;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        si += __shfl_xor_sync(FSLIC_FULL, si, off);
        sj += __shfl_xor_sync(FSLIC_FULL, sj, off);
    }
    if (lane == 0) {
        const double n = (double)(e - s);
        pos[2 * seg] = __double2float_rn(__ddiv_rn((double)si, n));
        pos[2 * seg + 1] = __double2float_rn(__ddiv_rn((double)sj, n));
    }
    const long b = seg / p.K, k = seg - b * p.K;
    for (int c = lane; c < p.C; c += 32) feat[seg * p.C + c] = means[(b * p.C + c) * p.K + k];
}
