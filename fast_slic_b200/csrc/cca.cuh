// fast_slic_b200/csrc/cca.cuh -- connectivity enforcement on the GPU.
//
// Replaces cca::ConnectivityEnforcer::execute with assign_disjoint_set / DisjointSet::merge /
// DisjointSet::flatten (fast-slic/src/cca.cpp:33-101, 103-173, 178-265; cca.h:36-57).
//
// Pipeline (all kernels batched over images with blockIdx.y):
//   k_ccl_tile     union-find of every 32 x 32 tile in shared memory; parent[p] = tile-local root
//   k_ccl_seams    lock-free union (atomicMin on roots) across the tile seams; the representative
//                  of a set is always its MINIMUM raster index == the reference's "leader"
//                  (cca.h:38-55 merges towards the smaller index)
//   k_ccl_flatten  parent[p] = root; per-root area (run-aggregated atomics); ordered root list per block,
//                  each root with its predecessor root (the root left of / above it)
//   k_scan_blocks  exclusive scan of the per-block counts (one CTA per image)
//   k_ccl_number   component number = rank of the root in raster order (cca.cpp:118-134);
//                  gathers the area by component number; counts candidates area >= thres
//   k_cca_select   only when candidates > K: libstdc++ std::partial_sort set semantics
//                  (cca.cpp:225-228), emulated step for step (make_heap / adjust_heap / push_heap)
//   k_kept_count / k_scan_blocks / k_kept_label   new label = rank among kept components, which
//                  are already in leader order (cca.cpp:229-237), else 0xFFFF
//   k_cca_absorb   unkept components take the label of the component left of (or above) their
//                  leader, transitively, by following predecessor roots (cca.cpp:238-255)
//   k_cca_output   out[p] = final label of root(p)  (cca.cpp:260-263)
#pragma once
#include "common.cuh"

#define CCA_BLOCK 1024
#define CCA_HIST 2052  // per-image histogram of candidate areas: [0..2047] exact, [2048] = larger

struct CcaParams {
    int H, W, N;       // N = H*W
    int K;             // max_label_size (cca.cpp:176)
    int thres;         // min_threshold
    int nblk;          // ceil(N / CCA_BLOCK)
    int heap_in_smem;  // k_cca_select keeps its heap in shared memory
    int which;         // post-selection kernels: -1 all images, 0 only images settled by k_cca_threshold, 1 only replayed ones
};

__device__ __forceinline__ bool cca_skip_image(const CcaParams& cp, const struct CcaCounters* ct);

// Per-image scalar scratch
struct CcaCounters {
    int ncomp;
    int ncand;
    int nkept;
    int sel_mode;  // 0: kept <=> area >= keep_thres; 1: selection ran, kept flag = top bit of carea
    int keep_thres;
    int need_sim;  // 1: the K-th largest area is tied ambiguously -> replay std::partial_sort step by step
    int dbg_ops;   // heap replacements performed by k_cca_select (diagnostics)
    int dbg_t;     // K-th largest candidate area found by k_cca_threshold (diagnostics)
};

__device__ __forceinline__ bool cca_skip_image(const CcaParams& cp, const CcaCounters* ct) {
    return cp.which >= 0 && (ct->need_sim != 0) != (cp.which != 0);
}

__device__ __forceinline__ int ccl_find(const int* par, int x) {
    int p = par[x];
    while (p != x) {
        x = p;
        p = par[x];
    }
    return x;
}

// lock-free union keeping the smaller index as root (Komura-style atomicMin reduction)
__device__ __forceinline__ void ccl_union(int* par, int a, int b) {
    a = ccl_find(par, a);
    b = ccl_find(par, b);
    while (a != b) {
        if (a < b) {
            int t = a;
            a = b;
            b = t;
        }  // a > b: hang a under b
        const int old = atomicMin(&par[a], b);
        if (old == a) break;  // a was still a root: done
        a = ccl_find(par, old);  // someone re-parented a meanwhile: continue from there
        b = ccl_find(par, b);
    }
}

// ---- level 1: union-find of one 32 x 32 pixel tile entirely in shared memory -----------------------
// One thread per pixel, one warp per tile row.  Runs inside a row come from a ballot; vertical links are
// united with shared-memory atomicMin (only where a run overlap starts); every pixel then points at the
// tile-local root (minimum raster index inside the tile), written as a GLOBAL raster index.
#define CCL_T 32

// One WARP per 32 x 32 tile, rows top-down, lane = column.  A run inherits the smallest root among the runs it
// touches in the row above (a segmented prefix-min by shuffles); shared-memory union-find is only needed
// when a run BRIDGES two components that were separate so far.  (The earlier one-thread-per-pixel version spent
// most of its instructions walking parent chains in divergent union loops, one or two lanes at a time.)
#define CCL_TW 4  // tiles (= warps) per CTA
__global__ void __launch_bounds__(32 * CCL_TW) k_ccl_tile(CcaParams cp, const uint16_t* __restrict__ labels,
                                                          int* __restrict__ par_all, uint32_t* __restrict__ area_all,
                                                          int tiles_x, int tiles_y, long ntiles_total) {
    __shared__ int s_par_all[CCL_TW][CCL_T * CCL_T];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long tile = (long)blockIdx.x * CCL_TW + warp;
    if (tile >= ntiles_total) return;  // no block-wide barrier below
    int* s_par = s_par_all[warp];
    const int per_img = tiles_x * tiles_y;
    const int b = (int)(tile / per_img);
    const int tl = (int)(tile - (long)b * per_img);
    const int tyb = tl / tiles_x, txb = tl - tyb * tiles_x;
    const int j = txb * CCL_T + lane;
    const bool colok = j < cp.W;
    const int nrows = min(CCL_T, cp.H - tyb * CCL_T);  // valid rows of this tile (>= 1)
    const uint16_t* lab = labels + (size_t)b * cp.N + (size_t)(tyb * CCL_T) * cp.W + j;
    // rows are consumed strictly in order, so the labels are prefetched one group of CCL_G rows ahead in
    // registers (the row loop is unrolled by CCL_G only: unrolled 32 times it no longer fits the instruction cache)
    constexpr int CCL_G = 8;
    uint32_t v[CCL_G], nv[CCL_G];
#pragma unroll
    for (int k = 0; k < CCL_G; k++) {
        // invalid pixels get labels that differ from everything
        v[k] = (colok && k < nrows) ? (uint32_t)lab[(size_t)k * cp.W] : (0x10000u + (uint32_t)(k * CCL_T + lane));
    }
    uint32_t up_v = 0xffffffffu, up_left = 0xffffffffu;
    int up_root = 0;
#pragma unroll 1
    for (int ty0 = 0; ty0 < CCL_T; ty0 += CCL_G) {
#pragma unroll
        for (int k = 0; k < CCL_G; k++) {
            const int ty = ty0 + CCL_G + k;
            nv[k] = (colok && ty < nrows) ? (uint32_t)lab[(size_t)ty * cp.W] : (0x10000u + (uint32_t)((ty & (CCL_T - 1)) * CCL_T + lane));
        }
#pragma unroll
        for (int k = 0; k < CCL_G; k++) {
            const int ty = ty0 + k;
            const uint32_t cur = v[k];
            const uint32_t left = __shfl_up_sync(FSLIC_FULL, cur, 1);
            const bool start = (lane == 0) || (cur != left);
            const unsigned m = __ballot_sync(FSLIC_FULL, start);
            const int sl = 31 - __clz(m & (0xffffffffu >> (31 - lane)));   // first lane of my run
            const unsigned above = (lane == 31) ? 0u : (m >> (lane + 1));
            const int end = above ? (lane + __ffs(above) - 1) : 31;        // last lane of my run
            // a vertical link matters only where a stretch of common columns of the two runs begins
            const bool conn = (ty > 0) && (up_v == cur);
            const bool need = conn && ((lane == 0) || (left != cur) || (up_left != up_v));
            unsigned cand = 0xffffffffu;
            if (need) cand = (unsigned)ccl_find(s_par, up_root);
            // min over the run: prefix min from the run start, then everyone reads the last lane of the run
            // (REDUX under per-run lane masks is executed one mask at a time -- WARPSYNC.EXCLUSIVE -- and was slower)
            unsigned pm = cand;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned y = __shfl_up_sync(FSLIC_FULL, pm, o);
                if (lane - o >= sl) pm = min(pm, y);
            }
            const unsigned rmin = __shfl_sync(FSLIC_FULL, pm, end);
            const unsigned own = (unsigned)(ty * CCL_T + sl);
            const int root = (int)(rmin < own ? rmin : own);
            if (need && cand != (unsigned)root) ccl_union(s_par, (int)cand, root);  // bridge
            s_par[ty * CCL_T + lane] = root;
            __syncwarp();
            up_left = left;
            up_v = cur;
            up_root = root;
        }
#pragma unroll
        for (int k = 0; k < CCL_G; k++) v[k] = nv[k];
    }
    if (!colok) return;
    int* pout = par_all + (size_t)b * cp.N + (size_t)(tyb * CCL_T) * cp.W + j;
    uint32_t* aout = area_all + (size_t)b * cp.N + (size_t)(tyb * CCL_T) * cp.W + j;
#pragma unroll 4
    for (int ty = 0; ty < nrows; ty++) {
        const int rt = ccl_find(s_par, ty * CCL_T + lane);
        const int ri = tyb * CCL_T + (rt >> 5), rj = txb * CCL_T + (rt & 31);
        pout[(size_t)ty * cp.W] = ri * cp.W + rj;
        aout[(size_t)ty * cp.W] = 0;
    }
}

// ---- level 2: unite tiles across their seams with the global lock-free union ------------------------
// index space per image: [0, nV) pixels on vertical seams (columns j = 32, 64, ..), then [nV, nV+nH)
// pixels on horizontal seams (rows i = 32, 64, ..).
__global__ void __launch_bounds__(256) k_ccl_seams(CcaParams cp, const uint16_t* __restrict__ labels,
                                                   int* __restrict__ par_all) {
    const int b = blockIdx.y;
    const int W = cp.W, H = cp.H;
    const int sv = (W - 1) / CCL_T, sh = (H - 1) / CCL_T;  // number of vertical / horizontal seams
    const int nV = sv * H, nH = sh * W;
    const uint16_t* lab = labels + (size_t)b * cp.N;
    int* par = par_all + (size_t)b * cp.N;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nV + nH; t += gridDim.x * blockDim.x) {
        if (t < nV) {
            const int i = t / sv, j = (t - i * sv + 1) * CCL_T;
            const int p = i * W + j;
            if (lab[p - 1] == lab[p]) ccl_union(par, p - 1, p);
        } else {
            const int u = t - nV;
            const int r = u / W, j = u - r * W;
            const int i = (r + 1) * CCL_T;
            const int p = i * W + j;
            const uint16_t v = lab[p], up = lab[p - W];
            if (up == v) {
                bool need = (j % CCL_T == 0) || (lab[p - 1] != v);
                if (!need) need = lab[p - W - 1] != up;
                if (need) ccl_union(par, p - W, p);
            }
        }
    }
}

// Block = 1024 consecutive pixels handled by 256 threads: warp w owns the four 32-pixel chunks 4w .. 4w+3
// (four independent root chases in flight per lane).  Besides flattening, the block emits its roots (= component
// leaders, cca.cpp:118-134) in raster order into rootbuf[blk * 1024 ...] and their count into blkcnt[blk], so that
// numbering the components afterwards touches the roots only, not every pixel again.  Beside every root it emits
// the root of the pixel left of it (above it in column 0) into predbuf: the component an unkept component is
// absorbed into (cca.cpp:243-246).  The left neighbour of a root at lane > 0 lies in the run of lane - 1 and at
// lane 0 of chunks 1..3 in the last run of the warp's previous chunk, both one shuffle away; only roots at lane 0
// of a warp's first chunk and roots in column 0 look their predecessor up with ccl_find.  chunkinfo gets the root
// mask of every 32-pixel chunk and the number of roots of the block in front of it: the root-list slot of any root.
__global__ void __launch_bounds__(256) k_ccl_flatten(CcaParams cp, const uint16_t* __restrict__ labels,
                                                     int* __restrict__ par_all, uint32_t* __restrict__ area_all,
                                                     int* __restrict__ blkcnt, int* __restrict__ rootbuf_all,
                                                     int* __restrict__ predbuf_all,
                                                     unsigned long long* __restrict__ chunkinfo_all) {
    __shared__ int s_chunk[32];  // roots per 32-pixel chunk
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint16_t* lab = labels + (size_t)b * cp.N;
    int* par = par_all + (size_t)b * cp.N;
    int p[4], sl[4], root[4];
    unsigned m[4], rmask[4];
    bool ok[4], start[4], col0[4];
    int jcol = (blockIdx.x * CCA_BLOCK + w * 128 + lane) % cp.W;  // column of chunk 0; the others by stepping
#pragma unroll
    for (int r = 0; r < 4; r++) {
        p[r] = blockIdx.x * CCA_BLOCK + (w * 4 + r) * 32 + lane;
        ok[r] = p[r] < cp.N;
        const uint32_t v = ok[r] ? lab[p[r]] : 0x10000u;
        const uint32_t left = __shfl_up_sync(FSLIC_FULL, v, 1);
        const int j = jcol;
        col0[r] = j == 0;
        jcol += 32;
        if (jcol >= cp.W) jcol = (cp.W >= 32) ? (jcol - cp.W) : (jcol % cp.W);
        start[r] = (lane == 0) || (j == 0) || (v != left);
        m[r] = __ballot_sync(FSLIC_FULL, start[r]);
        sl[r] = 31 - __clz(m[r] & (0xffffffffu >> (31 - lane)));
    }
    {   // the four root chases of a lane advance level by level, so up to four parent loads are in flight per lane
        // (four ccl_find() calls in a row would walk one chain after the other)
        int q[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            root[r] = p[r];
            q[r] = (ok[r] && start[r]) ? par[p[r]] : p[r];
        }
        for (;;) {
            bool mv[4], any = false;
#pragma unroll
            for (int r = 0; r < 4; r++) {
                mv[r] = q[r] != root[r];
                root[r] = q[r];
                any |= mv[r];
            }
            if (!any) break;
#pragma unroll
            for (int r = 0; r < 4; r++)
                if (mv[r]) q[r] = par[root[r]];
        }
    }
    int pred[4], findq[4];  // predecessor root of a root pixel, or the pixel whose root ccl_find still has to give it
    int prev_last = 0;      // root of the last pixel of the previous chunk
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int rt = __shfl_sync(FSLIC_FULL, root[r], sl[r]);
        const int left_rt = __shfl_up_sync(FSLIC_FULL, rt, 1);
        const int last_rt = __shfl_sync(FSLIC_FULL, rt, 31);
        bool isroot = false;
        pred[r] = -1;
        findq[r] = -1;
        if (ok[r]) {
            par[p[r]] = rt;
            if (start[r]) {
                // run length: distance to the next run start (or the end of the chunk / image)
                const unsigned above = (lane == 31) ? 0u : (m[r] >> (lane + 1));
                int len = above ? (__ffs(above)) : (32 - lane);
                if (p[r] + len > cp.N) len = cp.N - p[r];
                atomicAdd(&area_all[(size_t)b * cp.N + rt], (uint32_t)len);
                isroot = (rt == p[r]);
                // (pixel 0 is the leader of component 0, which has no predecessor)
                if (isroot && p[r] > 0) {
                    if (col0[r]) findq[r] = p[r] - cp.W;
                    else if (lane > 0) pred[r] = left_rt;
                    else if (r > 0) pred[r] = prev_last;
                    else findq[r] = p[r] - 1;
                }
            }
        }
        prev_last = last_rt;
        rmask[r] = __ballot_sync(FSLIC_FULL, isroot);
        if (lane == 0) s_chunk[w * 4 + r] = __popc(rmask[r]);
    }
#pragma unroll
    for (int r = 0; r < 4; r++)
        if (findq[r] >= 0) pred[r] = ccl_find(par, findq[r]);
    __syncthreads();
    // every warp scans the 32 chunk counts for itself (no second barrier)
    const int mine = s_chunk[lane];
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(FSLIC_FULL, incl, o);
        if (lane >= o) incl += y;
    }
    int* rootbuf = rootbuf_all + (size_t)b * cp.N + (size_t)blockIdx.x * CCA_BLOCK;
    int* predbuf = predbuf_all + (size_t)b * cp.N + (size_t)blockIdx.x * CCA_BLOCK;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int base = __shfl_sync(FSLIC_FULL, incl - mine, w * 4 + r);
        if ((rmask[r] >> lane) & 1u) {
            const int e = base + __popc(rmask[r] & ((1u << lane) - 1u));
            rootbuf[e] = p[r];
            predbuf[e] = pred[r];
        }
        if (lane == 0)
            chunkinfo_all[((size_t)b * cp.nblk + blockIdx.x) * (CCA_BLOCK / 32) + w * 4 + r] =
                ((unsigned long long)(unsigned)base << 32) | rmask[r];
    }
    if (threadIdx.x == 31) blkcnt[(size_t)b * cp.nblk + blockIdx.x] = incl;
}

// exclusive scan of cnt[0..n) (n = *n_dev if n_dev else n_static), total -> *total_out
__global__ void __launch_bounds__(1024) k_scan_blocks(const int* __restrict__ cnt_all, int* __restrict__ off_all,
                                                      int stride_per_image, int n_static,
                                                      const int* __restrict__ n_dev_base, int n_dev_stride_ints,
                                                      int n_div, int* __restrict__ total_base,
                                                      int total_stride_ints,
                                                      const CcaCounters* __restrict__ skip_counters, int which) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const int b = blockIdx.x;
    if (skip_counters && which >= 0 && (skip_counters[b].need_sim != 0) != (which != 0)) return;
    const int tid = threadIdx.x;
    const int* cnt = cnt_all + (size_t)b * stride_per_image;
    int* off = off_all + (size_t)b * stride_per_image;
    int n = n_static;
    if (n_dev_base) n = (n_dev_base[(size_t)b * n_dev_stride_ints] + n_div - 1) / n_div;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int c = base + tid;
        const int v = (c < n) ? cnt[c] : 0;
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(FSLIC_FULL, x, o);
            if ((tid & 31) >= o) x += y;
        }
        if ((tid & 31) == 31) s_warp[tid >> 5] = x;
        __syncthreads();
        if (tid < 32) {
            int w = s_warp[tid];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(FSLIC_FULL, w, o);
                if (tid >= o) w += y;
            }
            s_warp[tid] = w;
        }
        __syncthreads();
        const int woff = (tid >> 5) ? s_warp[(tid >> 5) - 1] : 0;
        const int excl = s_carry + woff + x - v;
        if (c < n) off[c] = excl;
        __syncthreads();
        if (tid == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) total_base[(size_t)b * total_stride_ints] = s_carry;
}

// Component numbers (= rank of the leader in raster order, cca.cpp:118-134) are implicit: the roots of block blk
// are components blkoff[blk] ..  One WARP per 1024-pixel block walks that block's ordered root list and gathers the
// area array by component number and the histogram of candidate areas for k_cca_threshold.
#define CCA_NUMBER_GRID 16
__global__ void __launch_bounds__(CCA_BLOCK) k_ccl_number(CcaParams cp, const int* __restrict__ rootbuf_all,
                                                          const uint32_t* __restrict__ aux_all,
                                                          const int* __restrict__ blkcnt,
                                                          const int* __restrict__ blkoff,
                                                          uint32_t* __restrict__ carea_all,
                                                          CcaCounters* __restrict__ counters,
                                                          unsigned int* __restrict__ ahist_all) {
    __shared__ int s_cand;
    // candidate areas 0..31 (the bulk: specks) are counted per warp and flushed once per block.  The lanes of a
    // warp are grouped by value first (MATCH.ANY): thirty lanes doing a shared-memory atomic on the SAME word are
    // serialised by the LSU at ~20 cycles each, which used to be this kernel's whole run time.
    __shared__ unsigned int s_hot[CCA_BLOCK / 32][32];
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    s_hot[warp][lane] = 0;
    if (threadIdx.x == 0) s_cand = 0;
    __syncthreads();
    const uint32_t* aux = aux_all + (size_t)b * cp.N;
    int ncand = 0;
    // a warp owns NB consecutive 1024-pixel blocks and walks their root lists as ONE flat sequence, NU x 32 roots
    // per step with all loads of a step in flight together (the kernel is a chain of dependent memory round trips)
    constexpr int NU = 8;
    const int wpi = gridDim.x * (CCA_BLOCK / 32);        // warps per image
    const int NB = (cp.nblk + wpi - 1) / wpi;            // blocks per warp (<= 32 for the images this grid is sized for)
    for (int blk0 = (blockIdx.x * (CCA_BLOCK / 32) + warp) * NB; blk0 < cp.nblk; blk0 += wpi * NB) {
        for (int sub = 0; sub < NB; sub += 32) {
            const int myblk = blk0 + sub + lane;
            const bool have = (sub + lane < NB) && (myblk < cp.nblk);
            const int mycnt = have ? blkcnt[(size_t)b * cp.nblk + myblk] : 0;
            const int myoff = have ? blkoff[(size_t)b * cp.nblk + myblk] : 0;
            int incl = mycnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(FSLIC_FULL, incl, o);
                if (lane >= o) incl += y;
            }
            const int total = __shfl_sync(FSLIC_FULL, incl, 31);
            const int nb_here = min(32, NB - sub);
            for (int r0 = 0; r0 < total; r0 += 32 * NU) {
                int pp[NU], cc[NU];  // root pixel (-1: none), component number
                uint32_t aa[NU];
#pragma unroll
                for (int u = 0; u < NU; u++) {
                    const int r = r0 + 32 * u + lane;
                    // block of flat index r: the first one whose inclusive prefix exceeds r
                    int bi = 0;
                    for (int q = 0; q < nb_here - 1; q++) bi += (r >= __shfl_sync(FSLIC_FULL, incl, q));
                    const int bincl = __shfl_sync(FSLIC_FULL, incl, bi), bcnt = __shfl_sync(FSLIC_FULL, mycnt, bi);
                    const int boff = __shfl_sync(FSLIC_FULL, myoff, bi);
                    const int t = r - (bincl - bcnt);
                    pp[u] = -1;  // (never a root entry)
                    if (r < total) {
                        pp[u] = rootbuf_all[(size_t)b * cp.N + (size_t)(blk0 + sub + bi) * CCA_BLOCK + t];
                        cc[u] = boff + t;
                    }
                }
#pragma unroll
                for (int u = 0; u < NU; u++) aa[u] = pp[u] != -1 ? aux[pp[u]] : 0u;
#pragma unroll
                for (int u = 0; u < NU; u++) {
                    uint32_t bin = 0xffffffffu;  // not a candidate
                    if (pp[u] != -1) {
                        carea_all[(size_t)b * cp.N + cc[u]] = aa[u];
                        // histogram of candidate areas: bins 0..2047 exact, bin 2048 = "2048 or more" (k_cca_threshold)
                        if ((int)aa[u] >= cp.thres) bin = aa[u] < 2048u ? aa[u] : 2048u;
                    }
                    const unsigned peers = __match_any_sync(FSLIC_FULL, bin);
                    if (bin != 0xffffffffu && lane == __ffs(peers) - 1) {
                        const unsigned n = __popc(peers);
                        ncand += (int)n;
                        if (bin < 32u) s_hot[warp][bin] += n;  // group leaders hold distinct bins: no atomic needed
                        else atomicAdd(&ahist_all[(size_t)b * CCA_HIST + bin], n);
                    }
                    __syncwarp();
                }
            }
        }
    }
    ncand = __reduce_add_sync(FSLIC_FULL, ncand);
    if (lane == 0 && ncand) atomicAdd(&s_cand, ncand);
    __syncthreads();
    if (threadIdx.x == 0 && s_cand) atomicAdd(&counters[b].ncand, s_cand);
    if (threadIdx.x < 32) {
        unsigned int tot = 0;
        for (int w = 0; w < CCA_BLOCK / 32; w++) tot += s_hot[w][threadIdx.x];
        if (tot) atomicAdd(&ahist_all[(size_t)b * CCA_HIST + threadIdx.x], tot);
    }
}

// ---------------------------------------------------------------------------------------------
// k_cca_threshold: decides, per image, what "the K largest candidates" are without replaying the
// heap whenever that is unambiguous.  Candidates are components with area >= thres (cca.cpp:213-219).
//   * ncand <= K: every candidate is kept (cca.cpp:225 is not taken)           -> keep_thres = thres
//   * else: t = K-th largest candidate area (exact 3 x 11-bit radix select), G = #(area > t),
//     E = #(area == t).  std::partial_sort keeps all G and K-G of the E tied ones; when E == K-G the
//     kept SET is simply {area >= t}                                             -> keep_thres = t
//   * otherwise the choice among the tied components depends on libstdc++'s heap dynamics
//                                                                                -> need_sim = 1
// One CTA per image, streaming the area array three times (4 B x ncomp, L2 resident).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_cca_threshold(CcaParams cp, const uint32_t* __restrict__ carea_all,
                                                        CcaCounters* __restrict__ counters,
                                                        const unsigned int* __restrict__ ahist_all) {
    __shared__ unsigned int s_hist[2048];
    __shared__ int s_warp[32];
    __shared__ unsigned int s_prefix, s_rank, s_found_bin, s_found_cnt;
    const int b = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    CcaCounters* ct = &counters[b];
    const int ncomp = ct->ncomp, ncand = ct->ncand;
    if (ncand <= cp.K) {
        if (tid == 0) {
            ct->keep_thres = cp.thres;
            ct->sel_mode = 0;
            ct->need_sim = 0;
        }
        return;
    }
    const uint32_t* area = carea_all + (size_t)b * cp.N;
    if (tid == 0) {
        s_prefix = 0;
        s_rank = (unsigned)cp.K;  // rank (1-based, from the top) still to locate inside the current prefix bucket
    }
    unsigned last_E = 0;
    // k_ccl_number already histogrammed the candidate areas below 2048; unless K or more candidates are
    // larger than that (then: the general 3-digit radix select below) the K-th largest is found in it directly
    const unsigned int* ahist = ahist_all + (size_t)b * CCA_HIST;
    const unsigned n_big = ahist[2048];
    const bool from_hist = n_big < (unsigned)cp.K;
    int first_pass = (cp.N < (1 << 22)) ? 1 : 0;  // areas <= N: the top digit is zero for everything
    if (from_hist) {
        first_pass = 2;
        if (tid == 0) s_rank = (unsigned)cp.K - n_big;
        __syncthreads();
    }
    for (int pass = first_pass; pass < 3; pass++) {
        const int shift = 22 - 11 * pass;
        for (int t = tid; t < 2048; t += 1024) s_hist[t] = from_hist ? ahist[t] : 0;
        __syncthreads();
        const unsigned prefix = s_prefix;
        for (int base = 0; base < (from_hist ? 0 : ncomp); base += 4096) {
            uint32_t av[4];
#pragma unroll
            for (int u = 0; u < 4; u++) {  // four independent loads in flight per thread
                const int c = base + u * 1024 + tid;
                av[u] = (c < ncomp) ? area[c] : 0xffffffffu;
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const uint32_t a = av[u];
                const bool valid = a != 0xffffffffu;
                const bool act = valid && ((int)a >= cp.thres) && ((pass == first_pass) || ((a >> (shift + 11)) == prefix));
                const unsigned bin = (a >> shift) & 2047u;
                // skew-aware histogram: the lanes that share the first active lane's bin add once
                const unsigned am = __ballot_sync(FSLIC_FULL, act);
                if (am) {
                    const int src = __ffs(am) - 1;
                    const unsigned b0 = __shfl_sync(FSLIC_FULL, bin, src);
                    const unsigned same = __ballot_sync(FSLIC_FULL, act && bin == b0);
                    if (lane == src) atomicAdd(&s_hist[b0], __popc(same));
                    if (act && bin != b0) atomicAdd(&s_hist[bin], 1u);
                }
            }
        }
        __syncthreads();
        // locate the bin holding the s_rank-th largest: inclusive scan from the top bin downwards
        const unsigned rank = s_rank;
        const int r0 = 2 * tid;  // reversed bins r0, r0+1  <->  bins 2047-r0, 2046-r0
        const unsigned h0 = s_hist[2047 - r0], h1 = s_hist[2046 - r0];
        unsigned x = h0 + h1;
        const unsigned mine = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            unsigned y = __shfl_up_sync(FSLIC_FULL, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = (int)x;
        __syncthreads();
        if (warp == 0) {
            unsigned w = (unsigned)s_warp[lane];
            unsigned z = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                unsigned y = __shfl_up_sync(FSLIC_FULL, z, o);
                if (lane >= o) z += y;
            }
            s_warp[lane] = (int)(z - w);
        }
        __syncthreads();
        const unsigned before = (unsigned)s_warp[warp] + x - mine;  // candidates in bins above this thread's pair
        if (before < rank && before + h0 >= rank) {
            s_found_bin = 2047 - r0;
            s_found_cnt = before;
        } else if (before + h0 < rank && before + h0 + h1 >= rank) {
            s_found_bin = 2046 - r0;
            s_found_cnt = before + h0;
        }
        __syncthreads();
        if (tid == 0) {
            s_prefix = (prefix << 11) | s_found_bin;
            s_rank = rank - s_found_cnt;
        }
        last_E = s_hist[s_found_bin];
        __syncthreads();
    }
    if (tid == 0) {
        const unsigned t = s_prefix;           // K-th largest candidate area
        const unsigned need = s_rank;          // how many of the tied (== t) components are kept: K - G
        if (last_E == need) {
            ct->keep_thres = (int)t;
            ct->sel_mode = 0;
            ct->need_sim = 0;
        } else {
            ct->need_sim = 1;
        }
        ct->dbg_t = (int)t;
    }
}

// ---------------------------------------------------------------------------------------------
// std::partial_sort(comps.begin(), comps.begin()+K, comps.end(), area-descending) -- the SET it leaves
// in the first K slots (cca.cpp:225-228), libstdc++ bits/stl_heap.h semantics.  The heap holds
// (area << 32 | component) words; only the area takes part in comparisons, like the reference's
// comparator (cca.cpp:179-185).  One CTA per image:
//   * all threads stream the components in ascending order in chunks, keeping only candidates
//     (area >= thres) that could still enter (area > current heap minimum, which never decreases);
//     survivors are compacted IN ORDER into a shared queue;
//   * thread 0 replays the queue sequentially through __pop_heap / __adjust_heap / __push_heap.
// ---------------------------------------------------------------------------------------------
#define SEL_CHUNK 8192  // components examined per round (8 per thread); the queue lives in dynamic shared memory
#define SEL_PER 8

__device__ __forceinline__ uint32_t hs_area(unsigned long long e) { return (uint32_t)(e >> 32); }

// The heap array is stored with a +1 slot offset (element i at h[i + 1]) so that the two children of a
// node (2i+1, 2i+2 -> slots 2i+2, 2i+3) form one aligned 16-byte pair: one LDS.128 / LDG.128 per level.
// h must hold len + 2 slots and be 16-byte aligned.
//
// __adjust_heap(first, hole, len, value) of bits/stl_heap.h walks the hole down to a leaf (child with the
// smaller area; on equal areas the RIGHT child), then __push_heap walks the value back up while
// area[parent] > area[value].  Along a root-to-leaf path of a valid heap the areas never decrease, so the
// value ends directly above the first path element whose area exceeds it: the same final arrangement is
// produced by this top-down walk that stops early -- it visits the same children in the same order.
// Heap storage accessors: SMEM = explicit shared-window addresses (LDS.128 / STS.64, no generic-address
// arithmetic on the critical path), otherwise plain global pointers.
template <bool SMEM>
struct HeapMem {
    unsigned long long* g;  // global base (slot 0)
    uint32_t s;             // shared-window byte address of slot 0
    __device__ __forceinline__ void pair(int slot, uint32_t& lo0, uint32_t& hi0, uint32_t& lo1, uint32_t& hi1) const {
        if (SMEM) {
            asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(lo0), "=r"(hi0), "=r"(lo1), "=r"(hi1) : "r"(s + 8u * (uint32_t)slot));
        } else {
            const uint4 v = *reinterpret_cast<const uint4*>(g + slot);
            lo0 = v.x; hi0 = v.y; lo1 = v.z; hi1 = v.w;
        }
    }
    __device__ __forceinline__ unsigned long long get(int slot) const {
        if (SMEM) {
            unsigned long long v;
            asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(s + 8u * (uint32_t)slot));
            return v;
        }
        return g[slot];
    }
    __device__ __forceinline__ void put(int slot, uint32_t lo, uint32_t hi) const {
        if (SMEM) asm volatile("st.shared.v2.u32 [%0], {%1,%2};" :: "r"(s + 8u * (uint32_t)slot), "r"(lo), "r"(hi) : "memory");
        else g[slot] = ((unsigned long long)hi << 32) | lo;
    }
    __device__ __forceinline__ void put(int slot, unsigned long long v) const { put(slot, (uint32_t)v, (uint32_t)(v >> 32)); }
};

template <bool SMEM>
__device__ __forceinline__ void hs_adjust_heap(const HeapMem<SMEM>& h, int hole, int len, unsigned long long value) {
    const uint32_t va = hs_area(value);
    for (;;) {
        const int l = 2 * hole + 1;
        if (l >= len) break;
        uint32_t lo0, hi0, lo1, hi1;  // children l (slot l+1) and l+1 (slot l+2): one aligned 16-byte pair
        h.pair(l + 1, lo0, hi0, lo1, hi1);
        const bool take_left = (l + 1 >= len) || (hi1 > hi0);  // right unless area[right] > area[left]
        const uint32_t clo = take_left ? lo0 : lo1, chi = take_left ? hi0 : hi1;
        if (chi > va) break;
        h.put(hole + 1, clo, chi);
        hole = take_left ? l : l + 1;
    }
    h.put(hole + 1, value);
}

// The __heap_select loop over the queued candidates (cca.cpp:226) on ONE warp with the heap in shared memory, padded
// with +infinity slots up to 2K+3 so that a node's children can always be loaded: missing children compare as
// +infinity, which reproduces libstdc++'s one-child and leaf cases without any bounds test.
//
// It is a PIPELINE of sift-downs.  Each __pop_heap only ever writes the node it currently stands on and moves down one
// level per half-step, so the next one may start at the root as soon as its predecessor stands on level >= 2: it then
// reads / writes strictly above everything the predecessor can still touch.  One trip of the loop = two half-steps of
// every sift-down in flight (a lane holds at most one: shared address of its hole and of the hole's children, its
// value) + at most one new sift-down.
//
// The loop is a single dependent chain on an in-order warp, i.e. its speed is the sum of the issue stalls of its
// instructions (first version: 85 instructions, 298 clocks per trip).  Hence PTX, and a selection step without
// cross-lane traffic other than one vote: the next 32 queue elements sit in registers, one per lane (`alive` = not yet
// consumed); elements in front of the first one that beats the root can be dropped for good (the root only grows); the
// lane HOLDING the first hit starts its sift-down itself (no find-first-set, no shuffles).  If that lane is still busy
// with an earlier sift-down (possible right after a window reload) the hit simply stays where it is and is retried in
// the next trip -- the root has not changed, and a sift-down ends within `depth` half-steps.
#define SEL_CHILDREN "ld.volatile.shared.v4.u32 {a0, a1, b0, b1}, [c];\n\t"
// The lanes exchange data through shared memory from one half-step to the next: a lane's store lands in the slot
// another lane's sift-down loads its children from.  The CUDA memory model orders those accesses only across a warp
// barrier, hence the bar.warp.sync behind the store.
#define SEL_HALF_STEP                                                                                       \
    "setp.gt.u32 tl, b1, a1;\n\t"            /* right child unless area[right] > area[left] */             \
    "min.u32 chi, a1, b1;\n\t"                                                                            \
    "selp.b32 clo, a0, b0, tl;\n\t"                                                                       \
    "setp.le.and.u32 mv, chi, vhi, act;\n\t" /* the child moves up, the hole moves down */                 \
    "min.u32 ohi, chi, vhi;\n\t"                                                                          \
    "selp.b32 olo, clo, vlo, mv;\n\t"                                                                     \
    "@act st.volatile.shared.v2.u32 [hole], {olo, ohi};\n\t" /* ... or the value lands here */             \
    "bar.warp.sync 0xffffffff;\n\t"                                                                      \
    "add.u32 c8, c, 8;\n\t"                                                                               \
    "selp.b32 nh, c, c8, tl;\n\t"                                                                         \
    "selp.b32 hole, nh, rooth, mv;\n\t"      /* idle lanes rest on the root: their loads are one broadcast */ \
    "add.u32 t0, hole, hole;\n\t"                                                                         \
    "sub.u32 c, t0, base;\n\t"               /* slot(h) = h + 1; children at slots 2h+2, 2h+3 */           \
    "mov.pred act, mv;\n\t"

#define SEL_LOOP_ASM                                                                                                        \
    "{\n\t"                                                                                                                 \
    ".reg .pred act, mv, tl, p, some, first, nact, take, kill, inq;\n\t"                                                    \
    ".reg .b32 base, c, hole, vlo, vhi, a0, a1, b0, b1, chi, clo, ohi, olo, c8, nh, t0, t1, t2, root, hit, elo, ehi;\n\t"    \
    ".reg .b32 lt, le, wpos, idx, qaddr, rooth, drain;\n\t"                                                                 \
    "mov.u32 base, %1;\n\t"                                                                                                 \
    "mov.u32 lt, %%lanemask_lt;\n\t"                                                                                        \
    "mov.u32 le, %%lanemask_le;\n\t"                                                                                        \
    "add.u32 rooth, base, 8;\n\t"     /* root = slot 1, its children = slots 2, 3 */                                        \
    "mov.u32 hole, rooth;\n\t"                                                                                              \
    "add.u32 c, base, 16;\n\t"                                                                                              \
    "mov.u32 vlo, 0;\n\t"                                                                                                   \
    "mov.u32 vhi, 0;\n\t"                                                                                                   \
    "setp.ne.u32 act, 0, 0;\n\t"                                                                                            \
    "mov.u32 wpos, %4;\n\t"                                                                                                 \
    SEL_CHILDREN                                                                                                            \
    "SEL_LOAD:\n\t"                    /* the window [wpos, wpos + 32) of the queue, one element per lane */                \
    "add.u32 idx, wpos, %5;\n\t"                                                                                            \
    "setp.lt.s32 inq, idx, %3;\n\t"                                                                                         \
    "mov.u32 elo, 0;\n\t"                                                                                                   \
    "mov.u32 ehi, 0;\n\t"              /* area 0 never beats the root: consumed / missing elements */                       \
    "shl.b32 qaddr, idx, 3;\n\t"                                                                                            \
    "add.u32 qaddr, qaddr, %2;\n\t"                                                                                         \
    "@inq ld.shared.v2.u32 {elo, ehi}, [qaddr];\n\t"                                                                        \
    "SEL_TRIP:\n\t"                                                                                                         \
    SEL_HALF_STEP                      /* (its children were loaded at the end of the previous trip) */                     \
    "ld.volatile.shared.u32 root, [base+12];\n\t"  /* final: the newest sift-down has left level 0 */                       \
    SEL_CHILDREN                                                                                                            \
    SEL_HALF_STEP                                                                                                           \
    "setp.gt.u32 p, ehi, root;\n\t"    /* comp(i, first) of __heap_select */                                                \
    "vote.sync.ballot.b32 hit, p, 0xffffffff;\n\t"                                                                          \
    "vote.sync.any.pred some, p, 0xffffffff;\n\t"                                                                           \
    SEL_CHILDREN                       /* of the next trip's first half-step: a lane that starts a sift-down now was */     \
                                       /* resting on the root, so the addresses do not depend on the decision below */      \
    "@!some bra.uni SEL_NEXT;\n\t"                                                                                          \
    "and.b32 t1, hit, lt;\n\t"                                                                                              \
    "setp.eq.and.u32 first, t1, 0, p;\n\t"                                                                                  \
    "not.pred nact, act;\n\t"                                                                                               \
    "and.pred take, first, nact;\n\t"                                                                                       \
    "and.b32 t2, hit, le;\n\t"                                                                                              \
    "setp.eq.or.u32 kill, t2, 0, take;\n\t"  /* elements in front of the first hit are gone for good */                     \
    "@take mov.u32 vlo, elo;\n\t"                                                                                           \
    "@take mov.u32 vhi, ehi;\n\t"                                                                                           \
    "@take add.u32 %0, %0, 1;\n\t"                                                                                          \
    "@kill mov.u32 ehi, 0;\n\t"                                                                                             \
    "or.pred act, act, take;\n\t"                                                                                           \
    "bra.uni SEL_TRIP;\n\t"                                                                                                 \
    "SEL_NEXT:\n\t"                    /* nothing left in the window beats the root, and the root only grows */             \
    "add.u32 wpos, wpos, 32;\n\t"                                                                                           \
    "setp.lt.s32 inq, wpos, %3;\n\t"                                                                                        \
    "@inq bra.uni SEL_LOAD;\n\t"                                                                                            \
    "mov.u32 drain, %6;\n\t"           /* no sift-down takes more than `depth` half-steps */                                \
    "SEL_DRAIN:\n\t"                                                                                                        \
    SEL_HALF_STEP                                                                                                           \
    SEL_CHILDREN                                                                                                            \
    "sub.u32 drain, drain, 1;\n\t"                                                                                          \
    "setp.gt.s32 inq, drain, 0;\n\t"                                                                                        \
    "@inq bra.uni SEL_DRAIN;\n\t"                                                                                           \
    "}\n\t"

__device__ __forceinline__ int sel_replay_smem(uint32_t heap_saddr, uint32_t queue_saddr, int qn, int consumed, int depth, int lane) {
    uint32_t cnt = 0;
    if (consumed < qn) {
        asm volatile(SEL_LOOP_ASM
                     : "+r"(cnt)
                     : "r"(heap_saddr), "r"(queue_saddr), "r"(qn), "r"(consumed), "r"(lane), "r"(depth)
                     : "memory");
        __syncwarp();
    }
    return (int)__reduce_add_sync(FSLIC_FULL, cnt);
}

// generic body shared by the pipeline kernel and the debug entry point
template <bool SMEM>
__device__ __forceinline__ void heap_select_body(const uint32_t* __restrict__ area, int ncomp, int K, int thres,
                                                  const HeapMem<SMEM> heap, uint32_t* __restrict__ mark_out /* |= 1<<31 */,
                                                  uint8_t* __restrict__ kept_bytes /* or nullptr */,
                                                  unsigned long long* s_queue /* shared, SEL_CHUNK entries */,
                                                  int* dbg_ops = nullptr) {
    __shared__ int s_warp[32];
    __shared__ int s_qn, s_filled;
    __shared__ uint32_t s_min;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nt = blockDim.x;
    if (tid == 0) {
        s_filled = 0;
        s_min = 0;
    }
    if (SMEM)  // +infinity padding behind the K live slots (see the replay loop)
        for (int u = K + 1 + tid; u < 2 * K + 4; u += nt) heap.put(u, 0u, 0xffffffffu);
    __syncthreads();
    // thread t owns components base + t*SEL_PER .. +SEL_PER-1 (ascending order inside the thread); the next
    // chunk is prefetched into registers while warp 0 replays the current one
    uint32_t cur[SEL_PER], nxt[SEL_PER];
#pragma unroll
    for (int u = 0; u < SEL_PER; u++) {
        const int c = tid * SEL_PER + u;
        cur[u] = (c < ncomp) ? area[c] : 0u;
    }
    for (int base = 0; base < ncomp; base += SEL_CHUNK) {
#pragma unroll
        for (int u = 0; u < SEL_PER; u++) {
            const int c = base + SEL_CHUNK + tid * SEL_PER + u;
            nxt[u] = (c < ncomp) ? area[c] : 0u;
        }
        const int filled = s_filled;
        const bool filling = filled < K;
        const uint32_t curmin = s_min;
        int cnt = 0;
#pragma unroll
        for (int u = 0; u < SEL_PER; u++) {
            const int c = base + tid * SEL_PER + u;
            cnt += (c < ncomp) && ((int)cur[u] >= thres) && (filling || cur[u] > curmin);
        }
        // ordered compaction: exclusive scan of cnt over the CTA
        int x = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(FSLIC_FULL, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int w = (lane < (nt >> 5)) ? s_warp[lane] : 0;
            int z = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(FSLIC_FULL, z, o);
                if (lane >= o) z += y;
            }
            s_warp[lane] = z - w;
            if (lane == 31) s_qn = z;
        }
        __syncthreads();
        int pos = s_warp[warp] + x - cnt;
#pragma unroll
        for (int u = 0; u < SEL_PER; u++) {
            const int c = base + tid * SEL_PER + u;
            if ((c < ncomp) && ((int)cur[u] >= thres) && (filling || cur[u] > curmin))
                s_queue[pos++] = ((unsigned long long)cur[u] << 32) | (uint32_t)c;
        }
        __syncthreads();
        const int qn = s_qn;
        // phase 1: the first K candidates fill the heap array in order
        int consumed = 0;
        if (filling) {
            consumed = min(qn, K - filled);
            for (int u = tid; u < consumed; u += nt) heap.put(filled + u + 1, s_queue[u]);
            __syncthreads();
        }
        const int f = filled + consumed;
        if (filling && f == K && K >= 2) {
            // __make_heap(first, middle): __adjust_heap on parents (K-2)/2 .. 0.  Nodes of one tree level
            // have disjoint subtrees, so a level can be processed in any order (here: in parallel); levels
            // go bottom-up exactly like the descending parent loop of bits/stl_heap.h.
            const int last_parent = (K - 2) / 2;
            int lvl = 31 - __clz(last_parent + 1);  // level of the last parent (root = level 0)
            for (; lvl >= 0; lvl--) {
                const int lo = (1 << lvl) - 1, hi = min((2 << lvl) - 2, last_parent);
                for (int node = lo + tid; node <= hi; node += nt) hs_adjust_heap(heap, node, K, heap.get(node + 1));
                __syncthreads();
            }
        }
        if (f == K && warp == 0) {
            // phase 2: the rest of the queue in order (cca.cpp:226 -> __heap_select loop), as a PIPELINE of
            // sift-downs inside one warp.  Each __pop_heap only ever writes the node it currently stands on
            // and moves down one level per step, so the next one may start at the root as soon as its
            // predecessor stands on level >= 2 (node index >= 3): it then reads / writes strictly above
            // everything the predecessor can still touch.  Lanes are pipeline slots; all advance in lockstep.
            // Timing is deterministic, so no cross-lane queries are needed: a sift-down moves exactly one
            // level per half-step (or has finished), one new sift-down may be issued per full step (two
            // levels behind its predecessor), and `depth` half-steps after the last issue everything is done.
            int nops = 0;
            if (SMEM) {
                nops = sel_replay_smem(heap.s, (uint32_t)__cvta_generic_to_shared(s_queue), qn, consumed, 32 - __clz(K), lane);
            } else {
            bool act = false;
            int hole = 0;
            uint32_t vlo = 0, vhi = 0;
            int qpos = consumed, next_lane = 0;
            const int depth = 32 - __clz(K);  // levels of the heap: no sift-down takes more half-steps
            int idle = depth;                 // half-steps since the last issue (start: pipeline empty)
            const uint32_t q_saddr = (uint32_t)__cvta_generic_to_shared(s_queue);
            // branch-free: idle lanes read a harmless slot and store nothing
            auto level_step = [&]() {
                const int l = 2 * hole + 1;
                const bool inb = act && (l < K);
                uint32_t lo0, hi0, lo1, hi1;
                heap.pair(inb ? l + 1 : 2, lo0, hi0, lo1, hi1);
                const bool take_left = (l + 1 >= K) || (hi1 > hi0);  // right unless area[right] > area[left]
                const uint32_t clo = take_left ? lo0 : lo1, chi = take_left ? hi0 : hi1;
                const bool move = inb && !(chi > vhi);  // the child moves up, the hole moves down
                if (act) heap.put(hole + 1, move ? clo : vlo, move ? chi : vhi);  // else: the value lands here
                hole = move ? (take_left ? l : l + 1) : hole;
                act = move;
                __syncwarp();
            };
            // Software pipelined: the root and the next queue element are fetched right after the first half-step
            // (by then the sift-down issued at the end of the previous iteration has rewritten the root for good)
            // and their latency hides behind the second half-step; the issue decision comes last.
            while (qpos < qn || idle < depth) {
                level_step();
                uint32_t elo = 0, ehi = 0, root_area = 0xffffffffu;
                const bool have = qpos < qn;
                if (have) {
                    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(elo), "=r"(ehi) : "r"(q_saddr + 8u * (uint32_t)qpos));
                    root_area = hs_area(heap.get(1));
                }
                level_step();
                idle += 2;
                if (have) {
                    qpos++;
                    if (ehi > root_area) {  // comp(i, first): __pop_heap(first, middle, i)
                        if (lane == next_lane) {
                            act = true;
                            hole = 0;
                            vlo = elo;
                            vhi = ehi;
                        }
                        next_lane = (next_lane + 1) & 31;
                        nops++;
                        idle = 0;
                    }
                }
            }
            }
            if (lane == 0) {
                s_min = hs_area(heap.get(1));
                if (dbg_ops) *dbg_ops += nops;
            }
        }
        if (tid == 0) s_filled = f;
        __syncthreads();
#pragma unroll
        for (int u = 0; u < SEL_PER; u++) cur[u] = nxt[u];
    }
    // publish the selected set
    const int filled = s_filled;
    for (int u = tid; u < filled; u += nt) {
        const uint32_t c = (uint32_t)(heap.get(u + 1) & 0xffffffffu);
        if (mark_out) mark_out[c] |= 0x80000000u;
        if (kept_bytes) kept_bytes[c] = 1;
    }
}

__global__ void __launch_bounds__(1024) k_cca_select(CcaParams cp, uint32_t* __restrict__ carea_all,
                                                     CcaCounters* __restrict__ counters,
                                                     unsigned long long* __restrict__ heap_global) {
    extern __shared__ __align__(16) unsigned char sel_smem[];  // [queue: SEL_CHUNK x u64][heap: (2K+4) x u64 if it fits]
    unsigned long long* s_queue = reinterpret_cast<unsigned long long*>(sel_smem);
    const int b = blockIdx.x;
    CcaCounters* ct = &counters[b];
    if (!ct->need_sim) return;  // k_cca_threshold settled it (or cca.cpp:225 is not taken)
    uint32_t* area = carea_all + (size_t)b * cp.N;
    if (cp.heap_in_smem) {
        HeapMem<true> hm;
        hm.g = nullptr;
        hm.s = (uint32_t)__cvta_generic_to_shared(sel_smem + SEL_CHUNK * 8);
        heap_select_body<true>(area, ct->ncomp, cp.K, cp.thres, hm, area, nullptr, s_queue, &ct->dbg_ops);
    } else {
        HeapMem<false> hm;
        hm.g = heap_global + (size_t)b * ((cp.K + 3) & ~1);
        hm.s = 0;
        heap_select_body<false>(area, ct->ncomp, cp.K, cp.thres, hm, area, nullptr, s_queue, &ct->dbg_ops);
    }
    if (threadIdx.x == 0) ct->sel_mode = 1;
}

__global__ void __launch_bounds__(1024) k_debug_heap_select(const uint32_t* __restrict__ area, int n, int middle,
                                                            uint8_t* __restrict__ kept,
                                                            unsigned long long* __restrict__ heap_global, int use_smem) {
    extern __shared__ __align__(16) unsigned char sel_smem[];
    unsigned long long* s_queue = reinterpret_cast<unsigned long long*>(sel_smem);
    if (use_smem) {
        HeapMem<true> hm;
        hm.g = nullptr;
        hm.s = (uint32_t)__cvta_generic_to_shared(sel_smem + SEL_CHUNK * 8);
        heap_select_body<true>(area, n, middle, 0, hm, nullptr, kept, s_queue);
    } else {
        HeapMem<false> hm;
        hm.g = heap_global;
        hm.s = 0;
        heap_select_body<false>(area, n, middle, 0, hm, nullptr, kept, s_queue);
    }
}

__device__ __forceinline__ bool cca_is_kept(uint32_t a, int sel_mode, int keep_thres) {
    return sel_mode ? (a >> 31) : ((int)a >= keep_thres);
}

// (both kernels walk the ncomp components of an image in chunks of 1024 with a small grid: ncomp is a few
//  thousand for real images, and it is only known on the device)
#define CCA_KEPT_GRID 16
// (four 1024-component chunks per trip: the loads of a trip are in flight together and the block-wide bookkeeping is
//  paid once per trip -- with one chunk per trip both kernels were a chain of load -> barrier round trips)
#define CCA_KEPT_U 4
__global__ void __launch_bounds__(CCA_BLOCK) k_kept_count(CcaParams cp, const uint32_t* __restrict__ carea_all,
                                                          const CcaCounters* __restrict__ counters,
                                                          int* __restrict__ blkcnt) {
    __shared__ int s_cnt[CCA_KEPT_U];
    const int b = blockIdx.y;
    if (cca_skip_image(cp, &counters[b])) return;
    const int ncomp = counters[b].ncomp;
    const int sel_mode = counters[b].sel_mode, keep_thres = counters[b].keep_thres;
    const uint32_t* carea = carea_all + (size_t)b * cp.N;
    for (int blk0 = blockIdx.x * CCA_KEPT_U; blk0 * CCA_BLOCK < ncomp; blk0 += gridDim.x * CCA_KEPT_U) {
        if (threadIdx.x < CCA_KEPT_U) s_cnt[threadIdx.x] = 0;
        uint32_t a[CCA_KEPT_U];
#pragma unroll
        for (int u = 0; u < CCA_KEPT_U; u++) {
            const int c = (blk0 + u) * CCA_BLOCK + threadIdx.x;
            a[u] = (c < ncomp) ? carea[c] : 0u;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < CCA_KEPT_U; u++) {
            const int c = (blk0 + u) * CCA_BLOCK + threadIdx.x;
            const bool kept = (c < ncomp) && cca_is_kept(a[u], sel_mode, keep_thres);
            const unsigned m = __ballot_sync(FSLIC_FULL, kept);
            if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s_cnt[u], __popc(m));
        }
        __syncthreads();
        if (threadIdx.x < CCA_KEPT_U && (blk0 + threadIdx.x) * CCA_BLOCK < ncomp)
            blkcnt[(size_t)b * cp.nblk + blk0 + threadIdx.x] = s_cnt[threadIdx.x];
        __syncthreads();  // s_cnt is zeroed again at the top of the next trip
    }
}

// newlabel[c] = rank among kept (cca.cpp:234-236); 0 for component 0 when it is not kept (cca.cpp:238); 0xFFFF for the
// components k_cca_absorb resolves.  blkoff here: kept components in front of each 1024-component chunk.
__global__ void __launch_bounds__(CCA_BLOCK) k_kept_label(CcaParams cp, const uint32_t* __restrict__ carea_all,
                                                          const CcaCounters* __restrict__ counters,
                                                          const int* __restrict__ blkoff,
                                                          uint16_t* __restrict__ cnew_all) {
    __shared__ int s_warp[CCA_KEPT_U][32];
    const int b = blockIdx.y;
    if (cca_skip_image(cp, &counters[b])) return;
    const int ncomp = counters[b].ncomp;
    const int sel_mode = counters[b].sel_mode, keep_thres = counters[b].keep_thres;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t* carea = carea_all + (size_t)b * cp.N;
    for (int blk0 = blockIdx.x * CCA_KEPT_U; blk0 * CCA_BLOCK < ncomp; blk0 += gridDim.x * CCA_KEPT_U) {
        uint32_t a[CCA_KEPT_U];
        int off[CCA_KEPT_U];
#pragma unroll
        for (int u = 0; u < CCA_KEPT_U; u++) {
            const int c = (blk0 + u) * CCA_BLOCK + tid;
            a[u] = (c < ncomp) ? carea[c] : 0u;
            off[u] = ((blk0 + u) * CCA_BLOCK < ncomp) ? blkoff[(size_t)b * cp.nblk + blk0 + u] : 0;
        }
        unsigned m[CCA_KEPT_U];
        bool kept[CCA_KEPT_U];
        __syncthreads();  // s_warp of the previous trip has been read
#pragma unroll
        for (int u = 0; u < CCA_KEPT_U; u++) {
            const int c = (blk0 + u) * CCA_BLOCK + tid;
            kept[u] = (c < ncomp) && cca_is_kept(a[u], sel_mode, keep_thres);
            m[u] = __ballot_sync(FSLIC_FULL, kept[u]);
            if (lane == 0) s_warp[u][warp] = __popc(m[u]);
        }
        __syncthreads();
        if (warp < CCA_KEPT_U) {  // warp u scans the 32 warp counts of chunk u
            const int w = s_warp[warp][lane];
            int x = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(FSLIC_FULL, x, o);
                if (lane >= o) x += y;
            }
            s_warp[warp][lane] = x - w;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < CCA_KEPT_U; u++) {
            const int c = (blk0 + u) * CCA_BLOCK + tid;
            if (c < ncomp) {
                uint16_t v = (c == 0) ? 0 : 0xFFFF;
                if (kept[u]) v = (uint16_t)(off[u] + s_warp[u][warp] + __popc(m[u] & ((1u << lane) - 1)));
                cnew_all[(size_t)b * cp.N + c] = v;
            }
        }
    }
}

// k_cca_absorb walks the ordered root lists of k_ccl_flatten, one WARP per 1024-pixel block: the roots of block blk
// are the components blkoff[blk] .. blkoff[blk + 1] - 1, in leader order.
#define CCA_TAIL_WARPS 8

// Component number and root-list slot of root pixel x, from the root mask of x's 32-pixel chunk (chunkinfo: mask in
// the low word, roots of the block in front of the chunk in the high word) -- two loads from compact tables.
__device__ __forceinline__ int cca_comp_of_root(const unsigned long long* chunkinfo, const int* blkoff, int x,
                                                int& slot) {
    const unsigned long long ci = chunkinfo[x >> 5];
    const int local = (int)(ci >> 32) + __popc((uint32_t)ci & ((1u << (x & 31)) - 1u));
    slot = (x >> 10) * CCA_BLOCK + local;
    return blkoff[x >> 10] + local;
}

// newlabel accesses that may meet a concurrent writer in k_cca_absorb: relaxed at GPU scope (morally strong, and not
// system scope like `volatile`, whose STRONG.SYS accesses made the kernel slower than the loads it saved)
__device__ __forceinline__ unsigned cca_ld_label(const uint16_t* p) {
    unsigned short v;
    asm volatile("ld.relaxed.gpu.global.u16 %0, [%1];" : "=h"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void cca_st_label(uint16_t* p, unsigned v) {
    asm volatile("st.relaxed.gpu.global.u16 [%0], %1;" ::"l"(p), "h"((unsigned short)v));
}

// Final label of every component, written at its root pixel (cca.cpp:238-255): unkept components take the label of
// the component left of their leader (above it in column 0), transitively.  An unkept component follows predecessor
// components until it meets one with a label: the first predecessor root comes with the root list (predbuf,
// coalesced), and the component number of a predecessor root comes from chunkinfo and blkoff; a later predecessor is
// the predbuf entry of that component's slot.  The labels live in the component-indexed newlabel array (2 B per
// component, cache resident), not at the scattered root pixels.  Usually the first predecessor is kept.
//
// Race-freedom: k_kept_label (an earlier launch) left every newlabel[c] either final (kept components, component 0)
// or 0xFFFF.  Here each unkept component's slot is written once, by the one thread that owns that component, with its
// final label; no slot is written twice or with anything else.  A concurrent reader of an unkept component's slot
// therefore sees 0xFFFF or that component's final label -- both accesses are aligned 16-bit relaxed GPU-scope (morally
// strong) operations, so there is no data race and no other value can be observed.  (A thread reads its own slot with
// a plain load: nobody else writes it.)  0xFFFF sends the reader on to the predecessor, whose final label is
// the same (cca.cpp:241-254 copies it); a final label is the answer.  Predecessors have strictly smaller component
// numbers and component 0 is always labelled, so every walk ends, with the same result under any interleaving.
__global__ void __launch_bounds__(32 * CCA_TAIL_WARPS) k_cca_absorb(CcaParams cp, const int* __restrict__ rootbuf_all,
                                                                   const int* __restrict__ predbuf_all,
                                                                   const unsigned long long* __restrict__ chunkinfo_all,
                                                                   const int* __restrict__ blkoff_all,
                                                                   const CcaCounters* __restrict__ counters,
                                                                   uint16_t* cnew_all, uint16_t* __restrict__ final_all,
                                                                   int nsplit) {
    const int b = blockIdx.y;
    if (cca_skip_image(cp, &counters[b])) return;
    // nsplit warps share a block's root list (small batches: more warps in flight per image)
    const int lane = threadIdx.x & 31, gw = blockIdx.x * CCA_TAIL_WARPS + (threadIdx.x >> 5);
    const int blk = gw / nsplit, part = gw - blk * nsplit;
    if (blk >= cp.nblk) return;  // (warp-uniform)
    const int* blkoff = blkoff_all + (size_t)b * cp.nblk;
    const int off = blkoff[blk];
    const int n = ((blk + 1 < cp.nblk) ? blkoff[blk + 1] : counters[b].ncomp) - off;
    const int* roots = rootbuf_all + (size_t)b * cp.N + (size_t)blk * CCA_BLOCK;
    const int* preds = predbuf_all + (size_t)b * cp.N;
    const unsigned long long* chunkinfo = chunkinfo_all + (size_t)b * cp.nblk * (CCA_BLOCK / 32);
    uint16_t* cnew = cnew_all + (size_t)b * cp.N;
    uint16_t* fin = final_all + (size_t)b * cp.N;
    // NU x 32 roots per trip, their loads in flight together (a block holds ~180 roots on 720p SLIC output)
    constexpr int NU = 8;
    for (int t0 = 32 * part; t0 < n; t0 += 32 * nsplit * NU) {
        int rt[NU], x[NU];
        unsigned lab[NU];
#pragma unroll
        for (int u = 0; u < NU; u++) {
            const int t = t0 + 32 * nsplit * u + lane;
            rt[u] = -1;  // no root here
            x[u] = 0;
            lab[u] = 0;
            if (t < n) {
                rt[u] = roots[t];
                x[u] = preds[(size_t)blk * CCA_BLOCK + t];
                lab[u] = cnew[off + t];
            }
        }
        // the walks of the NU roots of a lane advance hop by hop together, so that their loads are in flight at the
        // same time (walked one after the other, a warp paid the sum of the longest walks of its NU groups)
        int cx[NU], slot[NU];
        unsigned pl[NU];
        bool act[NU];
#pragma unroll
        for (int u = 0; u < NU; u++) {
            act[u] = rt[u] >= 0 && lab[u] == 0xFFFFu;
            pl[u] = 0;
            if (act[u]) cx[u] = cca_comp_of_root(chunkinfo, blkoff, x[u], slot[u]);
        }
        for (;;) {
            bool any = false;
#pragma unroll
            for (int u = 0; u < NU; u++) pl[u] = act[u] ? cca_ld_label(cnew + cx[u]) : pl[u];
#pragma unroll
            for (int u = 0; u < NU; u++) {
                if (act[u] && pl[u] != 0xFFFFu) {
                    act[u] = false;
                    lab[u] = pl[u];
                    cca_st_label(cnew + off + t0 + 32 * nsplit * u + lane, pl[u]);
                }
                any |= act[u];
            }
            if (!any) break;
            // not resolved yet: on to the predecessors
            int q[NU];
#pragma unroll
            for (int u = 0; u < NU; u++) q[u] = act[u] ? preds[slot[u]] : 0;
#pragma unroll
            for (int u = 0; u < NU; u++)
                if (act[u]) cx[u] = cca_comp_of_root(chunkinfo, blkoff, q[u], slot[u]);
        }
#pragma unroll
        for (int u = 0; u < NU; u++) {
            if (rt[u] < 0) continue;
            fin[rt[u]] = (uint16_t)lab[u];
        }
    }
}

__global__ void __launch_bounds__(256) k_cca_output(CcaParams cp, const int* __restrict__ par_all,
                                                    const uint16_t* __restrict__ final_all,
                                                    uint16_t* __restrict__ out_all,
                                                    const CcaCounters* __restrict__ counters) {
    const int b = blockIdx.y;
    if (cca_skip_image(cp, &counters[b])) return;
    const int* par = par_all + (size_t)b * cp.N;
    const uint16_t* fin = final_all + (size_t)b * cp.N;
    uint16_t* out = out_all + (size_t)b * cp.N;
    if ((cp.N & 7) == 0 && (reinterpret_cast<uintptr_t>(out_all) & 15) == 0 && (reinterpret_cast<uintptr_t>(par_all) & 15) == 0) {
        // 8 pixels per thread: two 16-byte root loads, eight gathers in flight, one 16-byte store
        for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < cp.N / 8; t += gridDim.x * blockDim.x) {
            const int4 r0 = reinterpret_cast<const int4*>(par)[2 * t], r1 = reinterpret_cast<const int4*>(par)[2 * t + 1];
            // neighbours mostly share their root: gather only where the root changes (predicated loads; the
            // kernel is bound by the one-sector-per-clock rate of scattered L1 accesses, not by bytes)
            const uint32_t a0 = fin[r0.x];
            uint32_t a1 = a0, a2, a3, a4, a5, a6, a7;
            if (r0.y != r0.x) a1 = fin[r0.y];
            a2 = a1; if (r0.z != r0.y) a2 = fin[r0.z];
            a3 = a2; if (r0.w != r0.z) a3 = fin[r0.w];
            a4 = a3; if (r1.x != r0.w) a4 = fin[r1.x];
            a5 = a4; if (r1.y != r1.x) a5 = fin[r1.y];
            a6 = a5; if (r1.z != r1.y) a6 = fin[r1.z];
            a7 = a6; if (r1.w != r1.z) a7 = fin[r1.w];
            reinterpret_cast<uint4*>(out)[t] = make_uint4(a0 | (a1 << 16), a2 | (a3 << 16), a4 | (a5 << 16), a6 | (a7 << 16));
        }
        return;
    }
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < cp.N; p += gridDim.x * blockDim.x) out[p] = fin[par[p]];
}
