// fast_slic_b200/csrc/float_slic.cuh -- the SLIC engine over float32 data: feature maps [B,C,H,W] (DESIGN.md section
// 4.19) and volumes [B,C,D,H,W] (section 4.22).  No counterpart in the reference.  Every float operation is one
// separately rounded IEEE operation (no contraction) in the order the contracts give, so a numpy restatement
// reproduces every bit:
//   distance   fc = +0; for c = 0 .. C-1: fc = fs_acc(fc, f_c, mu_c);  t_a = (float)v_a - c_a,  d = fc + spatial(t)
//              with the spatial term of the geometry (MapSlic, VolumeSlic)
//   winner     the smallest dist_key(d, k) over the candidates |v_a - (int)c_a| <= R_a on every axis
//   update     c_a = (float)((double)sum v_a / (double)n) (exact integer sums), the feature means are pool's
//              (pool_stage.h) over the pass's pixels; a cluster without members keeps its centre and features.
//
// The kernels run over NA axes, outer to inner: (y, x) for feature maps, (z, y, x) for volumes.  A pass visits the
// rows r, r + s, .. of axis NA - 2 (of every slice).  Centre state: pos [B,K,NA], feat [B,K,C].  Before every pass
// k_float_slic_grid counting-sorts the centres into cells of pitch G_a >= R_a (at most FLOAT_SLIC_MAX_CELLS of them,
// capi_float_slic.cu), so a tile finds every centre whose window may reach it in a few ranges of cells.
#pragma once
#include "cellgrid.cuh"
#include "common.cuh"

#define FLOAT_SLIC_CH 32  // channels of the centroid features staged in shared memory at a time
#define FLOAT_SLIC_NO_LABEL 0xffffu

// What differs between the two geometries: the assign tile (TILE_W columns x TILE_R pass rows x TILE_D slices, 256
// threads), MAXC, the candidates a tile keeps in registers (more go to k_float_slic_assign_fallback; the tile kernel
// instantiates MAXC / 4, MAXC / 2 and MAXC accumulators), the unroll of its channel loop, and the spatial term.
struct MapSlic {
    static constexpr int NA = 2, TILE_W = 32, TILE_R = 8, TILE_D = 1, MAXC = 32, UNROLL = 4;
    // fs_key's term: w2 * (ty * ty + tx * tx), one weight w2[0] = (compactness / S)^2 for both axes
    static __device__ __forceinline__ float spatial(const float* t, const float* w2) {
        return __fmul_rn(w2[0], __fadd_rn(__fmul_rn(t[0], t[0]), __fmul_rn(t[1], t[1])));
    }
};

struct VolumeSlic {
    static constexpr int NA = 3, TILE_W = 16, TILE_R = 4, TILE_D = 4, MAXC = 64, UNROLL = 2;
    // sv_key's term: (w2z * (tz * tz) + w2y * (ty * ty)) + w2x * (tx * tx)
    static __device__ __forceinline__ float spatial(const float* t, const float* w2) {
        return __fadd_rn(__fadd_rn(__fmul_rn(w2[0], __fmul_rn(t[0], t[0])), __fmul_rn(w2[1], __fmul_rn(t[1], t[1]))),
                         __fmul_rn(w2[2], __fmul_rn(t[2], t[2])));
    }
};

template <class G>
constexpr int tile_threads = G::TILE_W * G::TILE_R * G::TILE_D;

// The tile's extent along axis a
template <class G>
__host__ __device__ constexpr int tile_extent(int a) {
    return a == G::NA - 1 ? G::TILE_W : a == G::NA - 2 ? G::TILE_R : G::TILE_D;
}

// One pass's parameters; the per-axis arrays use their first NA entries
struct FloatSlicParams {
    int L[3];             // extents
    int R[3];             // window radii
    int G[3], cells[3];   // cell pitches >= R_a and cells per axis
    float w2[3];          // spatial weights
    int C, K, ncell;
    int r, s, npr;        // the pass visits rows r, r + s, .. (npr of them) of axis NA - 2
    int ntiles[3], tiles; // tiles along each axis, and per image
};

template <int NA>
__host__ __device__ __forceinline__ long image_size(const FloatSlicParams& p) {
    long n = p.L[0];
#pragma unroll
    for (int a = 1; a < NA; a++) n *= p.L[a];
    return n;
}

// The raster index of the pixel v inside its image
template <int NA>
__device__ __forceinline__ long raster(const FloatSlicParams& p, const int* v) {
    long i = v[0];
#pragma unroll
    for (int a = 1; a < NA; a++) i = i * p.L[a] + v[a];
    return i;
}

template <int NA>
__device__ __forceinline__ int cell_of(const FloatSlicParams& p, const float* c) {
    int cell = (int)c[0] / p.G[0];
#pragma unroll
    for (int a = 1; a < NA; a++) cell = cell * p.cells[a] + (int)c[a] / p.G[a];
    return cell;
}

template <int NA>
__device__ __forceinline__ bool in_window(const FloatSlicParams& p, const int* v, const float* c) {
    bool in = true;
#pragma unroll
    for (int a = 0; a < NA; a++) in &= abs(v[a] - (int)c[a]) <= p.R[a];
    return in;
}

// The packed key of candidate k at centre c for pixel v from its feature distance fc
template <class G>
__device__ __forceinline__ unsigned long long slic_key(const FloatSlicParams& p, float fc, const int* v, const float* c,
                                                       int k) {
    float t[G::NA];
#pragma unroll
    for (int a = 0; a < G::NA; a++) t[a] = __fsub_rn((float)v[a], c[a]);
    return dist_key(__fadd_rn(fc, G::spatial(t, p.w2)), k);
}

// The cells [c0, c1] that the windows of the pixels of the box [lo, hi] reach, and the number of their rows (every
// axis but the last).  box_row gives the first cell of row q, whose cells run to c1[NA - 1] along the last axis.
template <int NA>
__device__ __forceinline__ int cell_box(const FloatSlicParams& p, const int* lo, const int* hi, int* c0, int* c1) {
    int rows = 1;
#pragma unroll
    for (int a = 0; a < NA; a++) {
        c0[a] = max(lo[a] - p.R[a], 0) / p.G[a];
        c1[a] = min(hi[a] + p.R[a], p.L[a] - 1) / p.G[a];
        if (a < NA - 1) rows *= c1[a] - c0[a] + 1;
    }
    return rows;
}

template <int NA>
__device__ __forceinline__ int box_row(const FloatSlicParams& p, const int* c0, const int* c1, int q) {
    int idx[NA - 1];
#pragma unroll
    for (int a = NA - 2; a > 0; a--) {
        const int n = c1[a] - c0[a] + 1;
        idx[a] = c0[a] + q % n;
        q /= n;
    }
    idx[0] = c0[0] + q;
    int row = idx[0];
#pragma unroll
    for (int a = 1; a < NA - 1; a++) row = row * p.cells[a] + idx[a];
    return row * p.cells[NA - 1];
}

// The seeds of feature maps, one thread per (image, cluster, channel): the grid centre of initialize_clusters and the
// features of its pixel, or the clamped init_pos (fminf / fmaxf send NaN to 0) and init_feat as given.  count = 0.
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

// The integer centre of cell i of n on an axis of length L: (lo + hi - 1) / 2 of [iL/n, (i+1)L/n)
__device__ __forceinline__ int sv_centre(int i, int L, int n) {
    return (int)(((long)i * L / n + (long)(i + 1) * L / n - 1) / 2);
}

// The seeds of volumes, one thread per (volume, cluster, channel): cluster k = (iz * nh + iy) * nw + ix sits at the
// centre of its cell with the features of that voxel.  count = 0.
__global__ void __launch_bounds__(256) k_sv_seed(const float* __restrict__ vol, long nkc, int D, int H, int W, int C,
                                                 int nd, int nh, int nw, float* __restrict__ pos,
                                                 float* __restrict__ feat, int32_t* __restrict__ count) {
    const long n = (long)D * H * W;
    const int K = nd * nh * nw;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nkc; t += (long)gridDim.x * blockDim.x) {
        const long bk = t / C;
        const int c = (int)(t - bk * C);
        const long b = bk / K;
        const int k = (int)(bk - b * K);
        const int ix = k % nw, iy = (k / nw) % nh, iz = k / (nw * nh);
        const int z = sv_centre(iz, D, nd), y = sv_centre(iy, H, nh), x = sv_centre(ix, W, nw);
        feat[t] = vol[(b * C + c) * n + ((long)z * H + y) * W + x];
        if (c == 0) {
            pos[3 * bk] = (float)z;
            pos[3 * bk + 1] = (float)y;
            pos[3 * bk + 2] = (float)x;
            count[bk] = 0;
        }
    }
}

// The cell grid of image blockIdx.x: rec [K] = the cluster indices sorted by cell, in any order inside one;
// cell_start [ncell + 1] = the first slot of each cell.  1024 threads, (ncell + 1) ints of dynamic shared memory.
template <class G>
__global__ void __launch_bounds__(1024) k_float_slic_grid(FloatSlicParams p, const float* __restrict__ pos,
                                                          int* __restrict__ cell_start, uint32_t* __restrict__ rec) {
    extern __shared__ int s_cnt[];
    __shared__ int s_warp[32];
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const float* ps = pos + (size_t)b * p.K * G::NA;
    int* cs = cell_start + (size_t)b * (p.ncell + 1);
    for (int c = tid; c <= p.ncell; c += nt) s_cnt[c] = 0;
    __syncthreads();
    for (int k = tid; k < p.K; k += nt) atomicAdd(&s_cnt[cell_of<G::NA>(p, ps + G::NA * k)], 1);
    scan_cells(s_cnt, s_warp, cs, p.ncell + 1, tid, nt);
    for (int k = tid; k < p.K; k += nt) {
        const int slot = atomicAdd(&s_cnt[cell_of<G::NA>(p, ps + G::NA * k)], 1);
        rec[(size_t)b * p.K + slot] = (uint32_t)k;
    }
}

// Tile `tile` of a pass: its box [lo, hi] (on axis NA - 2 the first and last of its pass rows) and the pixel v of this
// thread, the columns along the threads, then the pass rows, then the slices
template <int NA>
struct Tile {
    int lo[NA], hi[NA], v[NA];
    bool valid;
};

template <class G>
__device__ __forceinline__ Tile<G::NA> tile_of(const FloatSlicParams& p, int tile) {
    Tile<G::NA> t;
    unsigned thr = threadIdx.x;
    t.valid = true;
#pragma unroll
    for (int a = G::NA - 1; a >= 0; a--) {
        const int T = tile_extent<G>(a);
        const bool pass = a == G::NA - 2;
        const int i = a ? tile % p.ntiles[a] : tile;
        const int o = (int)(a ? thr % T : thr);
        if (a) {
            tile /= p.ntiles[a];
            thr /= T;
        }
        const int m0 = i * T, m1 = min(m0 + T - 1, (pass ? p.npr : p.L[a]) - 1), m = m0 + o;
        t.valid = t.valid && m <= m1;
        t.lo[a] = pass ? p.r + m0 * p.s : m0;
        t.hi[a] = pass ? p.r + m1 * p.s : m1;
        t.v[a] = pass ? p.r + m * p.s : m;
    }
    return t;
}

// The channel loop of a tile with nc <= NB candidates: every pixel reads f_c once per channel and adds it to one
// accumulator per candidate, so each (pixel, candidate) sum runs over the channels in order.  Then the window test,
// the spatial term and the smallest key.
template <class G, int NB>
__device__ __forceinline__ void tile_body(const FloatSlicParams& p, const Tile<G::NA>& t, int b, int nc,
                                          const float* __restrict__ features, const float* __restrict__ feat,
                                          const int* s_k, const float (*s_c)[G::NA], float* s_mu,
                                          uint16_t* __restrict__ labels) {
    const long n = image_size<G::NA>(p), v = raster<G::NA>(p, t.v);
    const float* fp = features + (long)b * p.C * n + v;
    float acc[NB];
#pragma unroll
    for (int q = 0; q < NB; q++) acc[q] = 0.f;
    for (int cb = 0; cb < p.C; cb += FLOAT_SLIC_CH) {
        const int cn = min(FLOAT_SLIC_CH, p.C - cb);
        __syncthreads();  // the previous chunk is consumed
        for (int e = threadIdx.x; e < nc * cn; e += blockDim.x) {
            const int q = e / cn, cc = e - q * cn;
            s_mu[cc * G::MAXC + q] = feat[((long)b * p.K + s_k[q]) * p.C + cb + cc];
        }
        __syncthreads();
#pragma unroll G::UNROLL
        for (int cc = 0; cc < cn; cc++) {
            const float x = t.valid ? __ldg(fp + (long)(cb + cc) * n) : 0.f;
            const float4* mu4 = reinterpret_cast<const float4*>(s_mu + cc * G::MAXC);
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
            float c[G::NA];
#pragma unroll
            for (int a = 0; a < G::NA; a++) c[a] = s_c[q][a];
            if (in_window<G::NA>(p, t.v, c)) {
                const unsigned long long key = slic_key<G>(p, acc[q], t.v, c, s_k[q]);
                best = key < best ? key : best;
            }
        }
    }
    if (best != ~0ull) labels[(long)b * n + v] = (uint16_t)(uint32_t)best;
}

// The assign kernel of a pass: one CTA per tile (grid: tiles of an image x images).  The CTA collects the centres
// whose window may reach the tile from the cells, one warp per row of cells; with more than MAXC it appends the tile
// to ovf_list (ovf_count counts them) and leaves it to k_float_slic_assign_fallback.  A pixel without a candidate
// keeps its label.
template <class G>
__global__ void __launch_bounds__(tile_threads<G>) k_float_slic_assign_tiles(
    FloatSlicParams p, const float* __restrict__ features, const float* __restrict__ feat,
    const float* __restrict__ pos, const int* __restrict__ cell_start, const uint32_t* __restrict__ rec,
    uint16_t* __restrict__ labels, int* __restrict__ ovf_count, int* __restrict__ ovf_list) {
    constexpr int NA = G::NA, MAXC = G::MAXC;
    __shared__ int s_n;
    __shared__ int s_k[MAXC];
    __shared__ float s_c[MAXC][NA];
    __shared__ __align__(16) float s_mu[FLOAT_SLIC_CH * MAXC];
    const int b = blockIdx.y, tile = blockIdx.x;
    const Tile<NA> t = tile_of<G>(p, tile);
    int c0[NA], c1[NA];
    const int nrows = cell_box<NA>(p, t.lo, t.hi, c0, c1);
    const int* cs = cell_start + (size_t)b * (p.ncell + 1);
    const uint32_t* rc = rec + (size_t)b * p.K;
    const float* ps = pos + (size_t)b * p.K * NA;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int q = (int)(threadIdx.x >> 5); q < nrows; q += tile_threads<G> / 32) {
        const int row = box_row<NA>(p, c0, c1, q);
        const int hi = cs[row + c1[NA - 1] + 1];
        for (int e = cs[row + c0[NA - 1]] + (int)(threadIdx.x & 31); e < hi; e += 32) {
            const int k = (int)rc[e];
            float c[NA];
            bool near = true;
#pragma unroll
            for (int a = 0; a < NA; a++) {
                c[a] = ps[NA * k + a];
                const int ic = (int)c[a];
                near = near && ic >= t.lo[a] - p.R[a] && ic <= t.hi[a] + p.R[a];
            }
            if (near) {
                const int slot = atomicAdd(&s_n, 1);
                if (slot < MAXC) {
                    s_k[slot] = k;
#pragma unroll
                    for (int a = 0; a < NA; a++) s_c[slot][a] = c[a];
                }
            }
        }
    }
    __syncthreads();
    const int nc = s_n;
    if (nc > MAXC) {
        if (threadIdx.x == 0) ovf_list[atomicAdd(ovf_count, 1)] = b * p.tiles + tile;
        return;
    }
    if (nc == 0) return;
    if (nc <= MAXC / 4) tile_body<G, MAXC / 4>(p, t, b, nc, features, feat, s_k, s_c, s_mu, labels);
    else if (nc <= MAXC / 2) tile_body<G, MAXC / 2>(p, t, b, nc, features, feat, s_k, s_c, s_mu, labels);
    else tile_body<G, MAXC>(p, t, b, nc, features, feat, s_k, s_c, s_mu, labels);
}

// The overflow path: the tiles k_float_slic_assign_tiles listed, one thread per pixel, each walking the cells its
// window touches and computing every candidate's distance with the same fs_acc / slic_key.  A grid-stride loop over
// the list, so a fixed grid covers any count.
template <class G>
__global__ void __launch_bounds__(tile_threads<G>) k_float_slic_assign_fallback(
    FloatSlicParams p, const float* __restrict__ features, const float* __restrict__ feat,
    const float* __restrict__ pos, const int* __restrict__ cell_start, const uint32_t* __restrict__ rec,
    uint16_t* __restrict__ labels, const int* __restrict__ ovf_count, const int* __restrict__ ovf_list) {
    constexpr int NA = G::NA;
    const long n = image_size<NA>(p);
    const int total = *ovf_count;
    for (int e = blockIdx.x; e < total; e += gridDim.x) {
        const int id = ovf_list[e];
        const int b = id / p.tiles;
        const Tile<NA> t = tile_of<G>(p, id - b * p.tiles);
        if (!t.valid) continue;
        const int* cs = cell_start + (size_t)b * (p.ncell + 1);
        const uint32_t* rc = rec + (size_t)b * p.K;
        const float* ps = pos + (size_t)b * p.K * NA;
        const long v = raster<NA>(p, t.v);
        const float* fp = features + (long)b * p.C * n + v;
        int c0[NA], c1[NA];
        const int nrows = cell_box<NA>(p, t.v, t.v, c0, c1);
        unsigned long long best = ~0ull;
        for (int q = 0; q < nrows; q++) {
            const int row = box_row<NA>(p, c0, c1, q);
            const int hi = cs[row + c1[NA - 1] + 1];
            for (int j = cs[row + c0[NA - 1]]; j < hi; j++) {
                const int k = (int)rc[j];
                float c[NA];
#pragma unroll
                for (int a = 0; a < NA; a++) c[a] = ps[NA * k + a];
                if (!in_window<NA>(p, t.v, c)) continue;
                const float* mu = feat + ((long)b * p.K + k) * p.C;
                float fc = 0.f;
                for (int ch = 0; ch < p.C; ch++) fc = fs_acc(fc, __ldg(fp + (long)ch * n), mu[ch]);
                const unsigned long long key = slic_key<G>(p, fc, t.v, c, k);
                best = key < best ? key : best;
            }
        }
        if (best != ~0ull) labels[(long)b * n + v] = (uint16_t)(uint32_t)best;
    }
}

// The pool keys of a pass (pool_stage.h): keys[t] = image << 16 | label (0xffff outside [0, K)), vals[t] = the pixel
// index, over the pass rows of every slice of `batch` images in raster order (total = batch * slices * npr * W; a
// feature map is one slice)
template <class G>
__global__ void __launch_bounds__(256) k_float_slic_keys(FloatSlicParams p, const uint16_t* __restrict__ labels,
                                                         long total, uint32_t* __restrict__ keys,
                                                         uint32_t* __restrict__ vals) {
    const uint32_t H = p.L[G::NA - 2], W = p.L[G::NA - 1];
    const long n = image_size<G::NA>(p), per = n / H * p.npr;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const long b = t / per;
        const uint32_t rem = (uint32_t)(t - b * per), row = rem / W, x = rem - row * W;
        const uint32_t z = row / (uint32_t)p.npr, m = row - z * (uint32_t)p.npr;
        const uint32_t v = (z * H + p.r + m * p.s) * W + x;
        const uint32_t l = labels[b * n + v];
        keys[t] = (uint32_t)b << 16 | (l < (uint32_t)p.K ? l : FLOAT_SLIC_NO_LABEL);
        vals[t] = v;
    }
}

// The update after a pass, one warp per (image, cluster) over pool's sorted segments: the exact integer sums of the
// members' coordinates give the centre, and the pooled means (means [B,C,K]) become feat [B,K,C].  A cluster without
// members keeps both.
template <class G>
__global__ void __launch_bounds__(256) k_float_slic_update(FloatSlicParams p, long nk,
                                                           const uint32_t* __restrict__ seg_start,
                                                           const uint32_t* __restrict__ seg_end,
                                                           const uint32_t* __restrict__ members,
                                                           const float* __restrict__ means, float* __restrict__ pos,
                                                           float* __restrict__ feat) {
    constexpr int NA = G::NA;
    const long seg = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (seg >= nk) return;  // the whole warp leaves together
    const uint32_t s = seg_start[seg], e = seg_end[seg];
    if (e == s) return;
    unsigned long long sum[NA];
#pragma unroll
    for (int a = 0; a < NA; a++) sum[a] = 0;
    for (uint32_t q = s + lane; q < e; q += 32) {
        uint32_t v = members[q];
#pragma unroll
        for (int a = NA - 1; a > 0; a--) {
            const uint32_t up = v / (uint32_t)p.L[a];
            sum[a] += v - up * (uint32_t)p.L[a];
            v = up;
        }
        sum[0] += v;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
#pragma unroll
        for (int a = 0; a < NA; a++) sum[a] += __shfl_xor_sync(FSLIC_FULL, sum[a], off);
    }
    if (lane == 0) {
        const double cnt = (double)(e - s);
#pragma unroll
        for (int a = 0; a < NA; a++) pos[NA * seg + a] = __double2float_rn(__ddiv_rn((double)sum[a], cnt));
    }
    const long b = seg / p.K, k = seg - b * p.K;
    for (int c = lane; c < p.C; c += 32) feat[seg * p.C + c] = means[(b * p.C + c) * p.K + k];
}
