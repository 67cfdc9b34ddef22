// fast_slic_b200/csrc/assign.cuh -- the assign + update hot loop.
//
// Replaces BaseContext::assign / assign_clusters / update of the reference
// (fast-slic/src/context.cpp:200-243, 259-298, 302-387; AVX2 form arch/x64/avx2.h:11-185).
//
// The reference is cluster-centric: every cluster scatters into its (2S+1)^2 window with a strict
// `<` against a per-pixel running minimum; ties are therefore won by the cluster visited first,
// i.e. by the smaller (phase, k) where phase = 2*((cy/T)&1) + ((cx/T)&1), T = 2S+32
// (context.cpp:214-242).  On the GPU the loop is turned inside out: every pixel gathers over the
// clusters whose window covers it and minimises the packed key  d << 16 | rank,  rank being the
// candidate's position in the (phase, k)-sorted candidate list of its CTA tile.  Pixels no window
// covers keep their previous label (context.cpp:289-294 never fires for them).
#pragma once
#include "common.cuh"
#include "prepare.cuh"

// ---------------------------------------------------------------------------------------------
// Spatial patch (BaseContext::set_spatial_patch, context.cpp:23-40), laid out for LINEAR addressing:
//   tbl[(di + OY) * TS + (dj + OX)] = spatial_u16(coef, di, dj)  inside the (2S+1)^2 window,
//                                   = FSLIC_BIGSP                outside it,
// for di in [-OY, OY], dj in [-OX, OX].  A pixel's entry for candidate c is then at
//   (i*TS + j) + ((OY - cy)*TS + (OX - cx)):  a per-thread constant plus a per-candidate constant,
// so the window predicate and both abs() disappear from the inner loop.
// ---------------------------------------------------------------------------------------------
// The spatial term of the u16 contexts: (u16)(coef * (|di| + |dj|)) with manhattan_spatial_dist (the default),
// (u16)(coef * hypotf(di, dj)) without it (context.cpp:27-38).  The reference's hypotf is glibc's, which returns the
// correctly rounded sqrtf(di^2 + dj^2) for every offset a context produces (|di|, |dj| <= 32767; checked exhaustively
// by tests/test_euclidean_cpu.py).  CUDA's hypotf is not correctly rounded, so euclid_dist rounds the exact integer
// square sum itself: a float square root is exact while the sum fits 24 bits, a double one (rounded once more to
// float: harmless for a square root of a 31-bit integer) beyond.
__device__ __forceinline__ float euclid_dist(int di, int dj) {
    const int n = di * di + dj * dj;  // <= 2 * 32767^2 < 2^31
    return n <= (1 << 24) ? __fsqrt_rn((float)n) : __double2float_rn(__dsqrt_rn((double)n));
}

__device__ __forceinline__ uint32_t spatial_u16(float coef, int di, int dj, int manhattan) {
    const float m = manhattan ? (float)(abs(di) + abs(dj)) : euclid_dist(di, dj);
    return (uint16_t)__float2uint_rz(__fmul_rn(coef, m));
}

__global__ void k_build_sptable(uint16_t* __restrict__ tbl, int S, int OY, int OX, int TS, float coef, int manhattan) {
    const int n = (2 * OY + 1) * TS;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const int r = t / TS, c = t - r * TS;
        const int di = abs(r - OY), dj = abs(c - OX);
        uint16_t v = (uint16_t)FSLIC_BIGSP;
        if (di <= S && dj <= S && c <= 2 * OX) v = (uint16_t)spatial_u16(coef, di, dj, manhattan);
        tbl[t] = v;
    }
}

struct AssignParams {
    int H, W, K, S, B;
    int stride, rem;   // rows i with i % stride == rem are processed; sub-row sr <-> i = rem + sr*stride
    int nsub;          // number of such rows
    int cfg_stride;    // the configured subsample stride (freshness test)
    int fresh_from;    // rows with (i % cfg_stride) >= fresh_from were never assigned before
    int G, cellW, cellH, ncell;
    uint32_t Ginv;     // ceil(2^32 / G): x / G == __umulhi(x, Ginv) for 0 <= x < 65536 (x * G < 2^32)
    int OY, OX, TS, tbl_elems;
    int tiles_x, tiles_y, ntiles;  // warp tiles (32 columns x R sub-rows) per image
    int tps;           // warp tiles per super tile: AS_T, or 1 when the launch is too small to fill the GPU otherwise
    float coef;        // generic path only
    int manhattan;     // manhattan_spatial_dist: 1 = |di| + |dj|, 0 = Euclidean (read where the term is computed inline)
    // k_assign5 only: everything warp uniform that the host can precompute lives in the constant bank, so the kernel
    // neither keeps it in registers nor re-derives it (the compiler rematerialised the divisions per super tile)
    int stx, per_img, total;        // super tiles per tile row / per image / in all
    int wstride, db, dty, dsx;      // a warp's step through the super tiles, decomposed into (image, tile row, column) carries
    uint32_t tbl_bytes;             // patch size in shared memory, padded to 128 bytes
    uint32_t cinfo_img_bytes, cells_img_bytes, acc_img_bytes;  // per-image pitches of cinfo / cell_start / acc
    int fuse_prepare;               // 1: the last CTA to finish runs prepare_in_tail for the next pass (small batches)
};

#define AS_WARPS 16
#define AS_THREADS (AS_WARPS * 32)
#define AS_LIST 32  // candidate capacity of one warp tile; beyond it the tile takes the brute-force path

__device__ __forceinline__ int div_g(int x, uint32_t ginv) { return (int)__umulhi((uint32_t)x, ginv); }

// Packed per-cluster accumulators, 3 x u64 (+1 pad) so one update is 3 RED.64 instead of 6 RED.32:
//   [0] = n | sum_y << 32      [1] = sum_x | sum_L << 32      [2] = sum_a | sum_b << 32
// Every half stays far below 2^32 (sum_y <= n*H), so the halves never carry into each other.
__device__ __forceinline__ void acc_add_pixel(unsigned long long* ac, uint32_t label, int i, int j, uint32_t q) {
    atomicAdd(&ac[label * 4 + 0], 1ull | ((unsigned long long)(uint32_t)i << 32));
    atomicAdd(&ac[label * 4 + 1], (unsigned long long)(uint32_t)j | ((unsigned long long)(q & 0xff) << 32));
    atomicAdd(&ac[label * 4 + 2], (unsigned long long)((q >> 8) & 0xff) | ((unsigned long long)((q >> 16) & 0xff) << 32));
}

// ---------------------------------------------------------------------------------------------
// The per-pixel paths (k_assign_generic, k_assign_preempt, k_assign_real, k_assign_lsc, the warp tiles' overflow and
// k_trace_pass) share one gather, one store rule and, per path, one distance function.
// ---------------------------------------------------------------------------------------------
// Pixel t (0 <= t < nsub * W * B) of a grid-stride loop over the rows of the pass: image b, row i, column j.
__device__ __forceinline__ void pass_pixel(const AssignParams& ap, long t, int& b, int& i, int& j) {
    const long per_img = (long)ap.nsub * ap.W;
    b = (int)(t / per_img);
    const long r = t - (long)b * per_img;
    const int sr = (int)(r / ap.W);
    j = (int)(r - (long)sr * ap.W);
    i = ap.rem + sr * ap.stride;
}

// Minimum of  distance bits << 32 | sortkey  over the records of the cells within m rows / columns of pixel (i, j):
// the lexicographic minimum of (d, phase, k), the reference's visiting order breaking ties.  dist(r, d) sets d to the
// distance bits of candidate r and returns false when r is no candidate for the pixel.  ~0 when there is none.
// Callers name the lambda before the call: nvcc 12.9's front end asserts (il.c, i_copy_expr_tree) on one written inline
// in this call's argument list inside a function template.
template <class Dist>
__device__ __forceinline__ unsigned long long gather_min(const AssignParams& ap, int i, int j, int m,
                                                         const CInfo* __restrict__ ci, const int* __restrict__ cs,
                                                         Dist dist) {
    unsigned long long best = ~0ull;
    const int cr0 = max(i - m, 0) / ap.G, cr1 = min(i + m, ap.H - 1) / ap.G;
    const int cc0 = max(j - m, 0) / ap.G, cc1 = min(j + m, ap.W - 1) / ap.G;
    for (int cr = cr0; cr <= cr1; cr++) {
        const int s = cs[cr * ap.cellW + cc0], e = cs[cr * ap.cellW + cc1 + 1];
        for (int u = s; u < e; u++) {
            const CInfo r = ci[u];
            uint32_t d;
            if (!dist(r, d)) continue;
            const unsigned long long key = ((unsigned long long)d << 32) | r.sortkey;
            best = key < best ? key : best;
        }
    }
    return best;
}

// The label of pixel (i, j) at *lp after its gather, stored and returned.  A hit stores the winner's k: any candidate on
// the float paths, one below 0xFFFF on the u16 paths (U16), since the reference stores a candidate only when it is
// strictly below the running minimum, which starts at the type's maximum.  Where nothing hits, 0xFFFF on a row no pass
// has assigned yet, else the label of an earlier pass, which stays (context.cpp:289-294 never fires).
template <bool U16>
__device__ __forceinline__ uint32_t store_label(const AssignParams& ap, unsigned long long best, int i,
                                                uint16_t* __restrict__ lp) {
    uint32_t label;
    if (best != ~0ull && (!U16 || (uint32_t)(best >> 32) < 0xFFFFu)) {
        label = (uint32_t)(best & 0xffff);
        *lp = (uint16_t)label;
    } else if ((i % ap.cfg_stride) >= ap.fresh_from) {
        *lp = 0xFFFF;
        label = 0xFFFF;
    } else {
        label = *lp;
    }
    return label;
}

// The u16 distance of the default contexts from pixel (i, j) with colour q to candidate r: false outside r's
// (2S+1)^2 window and, with active_only, for a cluster whose record in cl is not active (context.cpp:218).  The warp
// tiles pass their spatial patch in shared memory (TS > 0: its row pitch) and read the term from it, like their main
// loop; the other callers compute it.
template <int TS>
__device__ __forceinline__ bool u16_dist(const AssignParams& ap, int i, int j, uint32_t q, const CInfo& r,
                                         bool active_only, const fslic_cluster* __restrict__ cl,
                                         const uint16_t* s_tbl, uint32_t& d) {
    const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
    const int di = i - cy, dj = j - cx;
    if (abs(di) > ap.S || abs(dj) > ap.S) return false;
    if (active_only && !cl[r.sortkey & 0xffffu].is_active) return false;
    const uint32_t sp = TS ? (uint32_t)s_tbl[(di + ap.OY) * TS + (dj + ap.OX)]
                           : spatial_u16(ap.coef, di, dj, ap.manhattan);
    d = sad4_acc(q, r.color, sp) & 0xffffu;  // u16 arithmetic like the scalar reference
    return true;
}

// Brute-force assignment of one pixel straight from the cell grid over every cluster whose window covers it.  Returns
// the new label (or the kept one) and stores it.  Used by the generic kernel and by warp tiles whose candidate list
// overflowed.
template <int TS = 0>
__device__ __forceinline__ uint32_t assign_pixel_generic(const AssignParams& ap, int i, int j, uint32_t q,
                                                          const CInfo* __restrict__ ci, const int* __restrict__ cs,
                                                          uint16_t* __restrict__ lb, const uint16_t* s_tbl) {
    const auto dist = [&](const CInfo& r, uint32_t& d) { return u16_dist<TS>(ap, i, j, q, r, false, nullptr, s_tbl, d); };
    const unsigned long long best = gather_min(ap, i, j, ap.S, ci, cs, dist);
    return store_label<true>(ap, best, i, &lb[(size_t)i * ap.W + j]);
}

__device__ __forceinline__ uint32_t lds_u16(uint32_t saddr) {
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

// exact per-byte equality -> 0x80 in every byte of w that equals the corresponding byte of m
__device__ __forceinline__ uint32_t eq80(uint32_t w, uint32_t m) {
    const uint32_t t = w ^ m;
    const uint32_t a = (t & 0x7f7f7f7fu) + 0x7f7f7f7fu;
    return ~(a | t) & 0x80808080u;
}

__device__ __forceinline__ void mma_u8_16x8x32(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------------------------------------
// k_assign_warp<TS, STRIDE, UPDATE>: the hot kernel.  Persistent CTAs (the spatial patch is loaded
// into shared memory once per CTA); inside a CTA every WARP is autonomous -- no block barrier
// after the patch load.  A warp walks "super tiles" of 4 horizontally adjacent warp tiles
// (each 32 columns x 4 sub-rows):
//   L. candidate lists for the 4 tiles at once, 8 lanes per tile: the clusters whose (2S+1)^2
//      window can touch the tile are collected from the cell grid (exact filter, ballot
//      compaction, <= 32 per tile), ranked by (phase, k) -- the reference's visiting order
//      (context.cpp:214-242) -- and staged {colour, patch offset} by rank in per-warp shared memory;
//   then per tile:
//   1. 4 quad loads per lane (LDG.32, 128 B per warp row);
//   2. per candidate and pixel:  LDS.U16 patch entry [immediate row offsets: TS and STRIDE are
//      compile-time] -> VABSDIFF4.U8.ACC (colour SAD + spatial) -> IMAD (d << 16 | rank) -> VIMNMX;
//   3. labels out (STG.U16, 64 B per warp row);
//   4. update sums (context.cpp:316-327) as an exact int8 tensor-core product
//        one-hot(rank)^T (candidates x pixels)  x  [1, row, lane, L, a, b] (pixels x features)
//      (mma.sync m16n8k32 u8 x u8 -> s32, 4 MMAs per 128 pixels and 16 candidates); the D fragment of lane
//      (g, tig) is accumulator word tig of candidates g and g+8, flushed as RED.64 if they received pixels.
//      Integer sums are order independent => exact.
// HBM per processed pixel: 4 B quad read + 2 B label written.
// ---------------------------------------------------------------------------------------------
#define AS_RG 1    // row groups of 4 sub-rows per lane (R = 4 * AS_RG rows per warp tile)
#define AS_MINB 2  // resident CTAs per SM the register budget is sized for
#define AS_R (4 * AS_RG)
#define AS_T 4   // warp tiles per super tile
#define AS_STAGE_BYTES (AS_WARPS * AS_T * AS_LIST * 22)

template <int TS, int STRIDE, bool UPDATE>
__global__ void __launch_bounds__(AS_THREADS, AS_MINB) k_assign_warp(AssignParams ap, const uint32_t* __restrict__ quad,
                                                               uint16_t* __restrict__ labels,
                                                               const CInfo* __restrict__ cinfo,
                                                               const int* __restrict__ cell_start,
                                                               unsigned long long* __restrict__ acc,
                                                               const uint16_t* __restrict__ g_tbl) {
    constexpr int R = AS_R;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint16_t* s_tbl = reinterpret_cast<uint16_t*>(smem_raw);
    // per-warp private staging block behind the patch in dynamic shared memory (AS_STAGE_BYTES in total):
    //   [ent: AS_T x 32 x uint2][ukey: AS_T x 32 x u32][ucol: same][ucyx: same][k: AS_T x 32 x u16]
    // the MMA A staging [32 pixel lanes][8 features] x u32 aliases ukey+ucol of the SAME warp (dead once ranked)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned char* wst = smem_raw + ((ap.tbl_elems * 2 + 15) & ~15) + warp * (AS_T * AS_LIST * 22);
    uint2 (*s_ent)[AS_LIST] = reinterpret_cast<uint2 (*)[AS_LIST]>(wst);
    uint32_t (*s_ukey)[AS_LIST] = reinterpret_cast<uint32_t (*)[AS_LIST]>(wst + AS_T * AS_LIST * 8);
    uint32_t (*s_ucol)[AS_LIST] = reinterpret_cast<uint32_t (*)[AS_LIST]>(wst + AS_T * AS_LIST * 12);
    int32_t (*s_ucyx)[AS_LIST] = reinterpret_cast<int32_t (*)[AS_LIST]>(wst + AS_T * AS_LIST * 16);
    uint16_t (*s_k)[AS_LIST] = reinterpret_cast<uint16_t (*)[AS_LIST]>(wst + AS_T * AS_LIST * 20);
    uint32_t (*s_feat)[8] = reinterpret_cast<uint32_t (*)[8]>(wst + AS_T * AS_LIST * 8);
    static_assert(32 * 8 * 4 <= AS_T * AS_LIST * 8, "the MMA staging must fit in ukey + ucol");
    static_assert(AS_R <= 16, "row index feature is a byte and the sums are scaled by 128 in s32");

    for (int t = tid; t < (ap.tbl_elems + 1) / 2; t += AS_THREADS)
        reinterpret_cast<uint32_t*>(s_tbl)[t] = reinterpret_cast<const uint32_t*>(g_tbl)[t];
    __syncthreads();

    const int S = ap.S, W = ap.W, H = ap.H;
    const int stride = STRIDE ? STRIDE : ap.stride;
    const int g = lane >> 2, tig = lane & 3;   // MMA fragment coordinates
    const int grp = lane >> 3, gl = lane & 7;  // list building: 8 lanes per tile
    const int rowpix = stride * W;

    // super-tile walk without divisions: (b, ty, sx) advance by a fixed (db, dty, dsx) with carries
    const int tps = ap.tps;
    const int stx = (ap.tiles_x + tps - 1) / tps;  // super tiles per tile row
    const long per_img = (long)stx * ap.tiles_y;
    const long total = per_img * ap.B;
    const long wstride = (long)gridDim.x * AS_WARPS;
    const long first = (long)blockIdx.x * AS_WARPS + warp;
    int b = (int)(first / per_img);
    const int tl0 = (int)(first - (long)b * per_img);
    int ty = tl0 / stx, sx = tl0 - ty * stx;
    const int db = (int)(wstride / per_img);
    const int dtl = (int)(wstride - (long)db * per_img);
    const int dty = dtl / stx, dsx = dtl - dty * stx;
    for (long st = first; st < total; st += wstride, b += db, ty += dty, sx += dsx) {
        if (sx >= stx) { sx -= stx; ty += 1; }
        if (ty >= ap.tiles_y) { ty -= ap.tiles_y; b += 1; }
        const int wsr0 = ty * R;
        const int nrow = min(R, ap.nsub - wsr0);  // valid sub-rows of this tile row (>= 1)
        const int wi0 = ap.rem + wsr0 * stride, wi1 = wi0 + (nrow - 1) * stride;
        const size_t img_off = (size_t)b * H * W;
        const CInfo* ci = cinfo + (size_t)b * ap.K;
        const int* cs = cell_start + (size_t)b * (ap.ncell + 1);
        unsigned long long* ac = acc + (size_t)b * ap.K * 4;

        // ---- L. candidate lists of the 4 tiles, 8 lanes each ----
        // tile of this lane group: columns [gj0, gj0+31]; wanted clusters: cy in [wi0-S, wi1+S], cx in [gj0-S, gj0+31+S]
        const int gtx = sx * tps + grp;
        const bool gvalid = grp < tps && gtx < ap.tiles_x;
        const int gj0 = gtx * 32;
        int n_g = 0;  // candidates found for this group's tile (same value in its 8 lanes)
        {
            const int cr0 = div_g(max(wi0 - S, 0), ap.Ginv), cr1 = div_g(min(wi1 + S, H - 1), ap.Ginv);
            const int cc0 = div_g(max(gj0 - S, 0), ap.Ginv), cc1 = div_g(min(gj0 + 31 + S, W - 1), ap.Ginv);
            for (int crb = cr0; crb <= cr1; crb += 8) {
                const int cr = crb + gl;
                int rs = 0, cnt = 0;
                if (gvalid && cr <= cr1) {
                    rs = cs[cr * ap.cellW + cc0];
                    cnt = cs[cr * ap.cellW + cc1 + 1] - rs;
                }
                int incl = cnt;  // inclusive scan inside the 8-lane group
#pragma unroll
                for (int o = 1; o < 8; o <<= 1) {
                    const int y = __shfl_up_sync(FSLIC_FULL, incl, o, 8);
                    if (gl >= o) incl += y;
                }
                const int T = __shfl_sync(FSLIC_FULL, incl, 7, 8);
                const int Tmax = __reduce_max_sync(FSLIC_FULL, T);
                const int nr = min(8, cr1 - crb + 1);  // cell rows in this chunk (same for every lane group)
                for (int t0 = 0; t0 < Tmax; t0 += 8) {
                    const int t = t0 + gl;
                    int row = 0;
                    for (int r = 0; r < nr - 1; r++) row += (t >= __shfl_sync(FSLIC_FULL, incl, r, 8));
                    const int rincl = __shfl_sync(FSLIC_FULL, incl, row, 8);
                    const int rcnt = __shfl_sync(FSLIC_FULL, cnt, row, 8);
                    const int rstart = __shfl_sync(FSLIC_FULL, rs, row, 8);
                    bool hit = false;
                    CInfo r;
                    if (t < T) {
                        r = ci[rstart + (t - (rincl - rcnt))];
                        const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
                        hit = (cy >= wi0 - S) && (cy <= wi1 + S) && (cx >= gj0 - S) && (cx <= gj0 + 31 + S);
                    }
                    const unsigned gb = (__ballot_sync(FSLIC_FULL, hit) >> (grp * 8)) & 0xffu;
                    const int slot = n_g + __popc(gb & ((1u << gl) - 1));
                    if (hit && slot < AS_LIST) {
                        s_ukey[grp][slot] = r.sortkey;
                        s_ucol[grp][slot] = r.color;
                        s_ucyx[grp][slot] = r.cyx;
                    }
                    n_g += __popc(gb);
                }
            }
        }
        __syncwarp();
        {   // rank by (phase, k) (keys are unique) and stage by rank
            const int nmax = __reduce_max_sync(FSLIC_FULL, min(n_g, AS_LIST));
            for (int a0 = 0; a0 < nmax; a0 += 8) {
                const int a = a0 + gl;
                const bool mine = a < n_g && n_g <= AS_LIST;
                const uint32_t key = mine ? s_ukey[grp][a] : 0u;
                int rank = 0;
                for (int u = 0; u < nmax; u++) rank += (u < n_g) && (s_ukey[grp][u] < key);
                if (mine) {
                    const int32_t cyx = s_ucyx[grp][a];
                    const int cy = (int16_t)(cyx & 0xffff), cx = cyx >> 16;
                    s_ent[grp][rank] =
                        make_uint2(s_ucol[grp][a], (uint32_t)(2 * ((ap.OY - cy) * TS + (ap.OX - cx))));
                    s_k[grp][rank] = (uint16_t)(key & 0xffff);
                }
            }
        }
        __syncwarp();
        // ---- the 4 tiles, one after the other ----
#pragma unroll 1
        for (int tq = 0; tq < tps; tq++) {
            const int tx = sx * tps + tq;
            if (tx >= ap.tiles_x) break;  // warp uniform
            const int n = __shfl_sync(FSLIC_FULL, n_g, tq * 8);
            const int wj0 = tx * 32;
            const int j = wj0 + lane;
            const bool colok = j < W;
            const uint32_t* qrow = quad + img_off + (size_t)wi0 * W + j;  // this lane's pixel in row 0 of the tile
            uint16_t* lrow = labels + img_off + (size_t)wi0 * W + j;

            // ---- 1. pixels ----
            uint32_t q[R];
#pragma unroll
            for (int rr = 0; rr < R; rr++) {
                const bool ok = colok && rr < nrow;
                q[rr] = ok ? ld_nc_u32(qrow + rr * rowpix) : 0u;
            }

            if (n > AS_LIST) {
                // ---- overflow (clusters piled on one spot): brute force, direct atomics ----
#pragma unroll
                for (int rr = 0; rr < R; rr++) {
                    if (colok && rr < nrow) {
                        const int i = wi0 + rr * stride;
                        const uint32_t label = assign_pixel_generic<TS>(ap, i, j, q[rr], ci, cs, labels + img_off, s_tbl);
                        if (UPDATE && label != 0xFFFF) acc_add_pixel(ac, label, i, j, q[rr]);
                    }
                }
                continue;
            }

            // ---- 2. distances ----
            // every (row, column) of the footprint is inside the patch for every listed candidate, valid or not.
            // patch entry of (row rr, candidate c) at shared byte address row0 + c.offset + rr * 2*stride*TS
            const unsigned char* rowp = smem_raw + 2 * (wi0 * TS + j);
            uint32_t best[R];
#pragma unroll
            for (int rr = 0; rr < R; rr++) best[rr] = 0xffffffffu;
            for (int c = 0; c < n; c++) {
                const uint2 e = s_ent[tq][c];
                const unsigned char* pc = rowp + (int)e.y;
#pragma unroll
                for (int rr = 0; rr < R; rr++) {
                    const uint32_t sp = *reinterpret_cast<const uint16_t*>(pc + rr * (2 * stride * TS));
                    const uint32_t d = sad4_acc(q[rr], e.x, sp);
                    best[rr] = min(best[rr], d * 65536u + (uint32_t)c);
                }
            }

            // ---- 3. labels (context.cpp:316-327) ----
            uint32_t rw[AS_RG];  // local rank bytes, 4 rows per word (0xFF = contributes to no candidate)
#pragma unroll
            for (int gq = 0; gq < AS_RG; gq++) rw[gq] = 0;
#pragma unroll
            for (int rr = 0; rr < R; rr++) {
                const bool ok = colok && rr < nrow;
                const bool covered = ok && ((best[rr] >> 16) < FSLIC_BIGSP);
                uint32_t rb = 0xff;
                if (covered) {
                    rb = best[rr] & 0xff;
                    lrow[rr * rowpix] = s_k[tq][rb];
                } else if (ok) {
                    const int i = wi0 + rr * stride;
                    if ((i % ap.cfg_stride) >= ap.fresh_from) {
                        lrow[rr * rowpix] = 0xFFFF;
                    } else if (UPDATE) {  // a stale label from an earlier pass still counts (context.cpp:318-319)
                        const uint16_t old = lrow[rr * rowpix];
                        if (old != 0xFFFF) acc_add_pixel(ac, old, i, j, q[rr]);
                    }
                }
                rw[rr >> 2] |= rb << (8 * (rr & 3));
            }

            // ---- 4. update sums on the tensor cores ----
            if (UPDATE) {
                // D[candidate][feature] += OneHot[candidate][pixel] * F[pixel][feature]   (m16n8k32, u8 x u8 -> s32)
                //   A = one-hot of the winning rank, built in registers (16 candidates per pass: one pass unless
                //       the list is longer than 16);  B = [1, row, lane, L, a, b, 0, 0] per pixel, staged in smem.
                // Lane (g, tig) ends up with features (2 tig, 2 tig + 1) of candidates g and g + 8: exactly the two
                // halves of packed accumulator word tig -- no compaction of the winners, no shuffles of D.
                const int n16 = (n + 15) >> 4;
                for (int nt = 0; nt < n16; nt++) {
                    int d[4] = {0, 0, 0, 0};
                    const uint32_t mg0 = (uint32_t)(nt * 16 + g) * 0x01010101u, mg1 = mg0 + 0x08080808u;
#pragma unroll
                    for (int gq = 0; gq < AS_RG; gq++) {
                        // stage this row group's features: [count 1, row index, lane index, L, a, b, 0, 0] per pixel lane
                        const uint32_t q0 = q[4 * gq], q1 = q[4 * gq + 1], q2 = q[4 * gq + 2], q3 = q[4 * gq + 3];
                        const uint32_t lo01 = __byte_perm(q0, q1, 0x5140), lo23 = __byte_perm(q2, q3, 0x5140);
                        const uint32_t hi01 = __byte_perm(q0, q1, 0x0062), hi23 = __byte_perm(q2, q3, 0x0062);
                        __syncwarp();  // the previous group's fragments have been read
                        *reinterpret_cast<uint4*>(&s_feat[lane][0]) =
                            make_uint4(0x01010101u, 0x03020100u + 0x04040404u * gq, (uint32_t)lane * 0x01010101u,
                                       __byte_perm(lo01, lo23, 0x5410));
                        *reinterpret_cast<uint4*>(&s_feat[lane][4]) =
                            make_uint4(__byte_perm(lo01, lo23, 0x7632), __byte_perm(hi01, hi23, 0x5410), 0u, 0u);
                        __syncwarp();
#pragma unroll
                        for (int s4 = 0; s4 < 4; s4++) {
                            const uint32_t w0 = __shfl_sync(FSLIC_FULL, rw[gq], 8 * s4 + tig);
                            const uint32_t w1 = __shfl_sync(FSLIC_FULL, rw[gq], 8 * s4 + 4 + tig);
                            mma_u8_16x8x32(d, eq80(w0, mg0), eq80(w0, mg1), eq80(w1, mg0), eq80(w1, mg1),
                                           s_feat[8 * s4 + tig][g], s_feat[8 * s4 + 4 + tig][g]);
                        }
                    }
                    // sums are scaled by 128 (the one-hot byte is 0x80)
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) {
                        const int c = nt * 16 + g + 8 * hh;
                        const uint32_t v0 = (uint32_t)d[2 * hh] >> 7, v1 = (uint32_t)d[2 * hh + 1] >> 7;
                        const uint32_t cnt = __shfl_sync(FSLIC_FULL, v0, lane & ~3);  // feature 0 lives in the tig = 0 lane
                        if (c < n && tig < 3 && cnt != 0) {
                            unsigned long long word;
                            if (tig == 0)
                                word = (unsigned long long)cnt |
                                       ((unsigned long long)(cnt * (uint32_t)wi0 + (uint32_t)stride * v1) << 32);
                            else if (tig == 1)
                                word = (unsigned long long)(cnt * (uint32_t)wj0 + v0) | ((unsigned long long)v1 << 32);
                            else
                                word = (unsigned long long)v0 | ((unsigned long long)v1 << 32);
                            atomicAdd(&ac[(uint32_t)s_k[tq][c] * 4 + tig], word);
                        }
                    }
                }
                __syncwarp();  // s_feat is rewritten by the next tile
            }
        }
        __syncwarp();  // the list staging is rewritten by the next super tile
    }
}

// ---------------------------------------------------------------------------------------------
// k_assign_generic<UPDATE>: correctness-first path without the shared-memory patch, for S so large
// that the linear patch does not fit in shared memory.  One thread per pixel.
// ---------------------------------------------------------------------------------------------
template <bool UPDATE>
__global__ void __launch_bounds__(256) k_assign_generic(AssignParams ap, const uint32_t* __restrict__ quad,
                                                         uint16_t* __restrict__ labels,
                                                         const CInfo* __restrict__ cinfo,
                                                         const int* __restrict__ cell_start,
                                                         unsigned long long* __restrict__ acc) {
    const long total = (long)ap.nsub * ap.W * ap.B;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        int b, i, j;
        pass_pixel(ap, t, b, i, j);
        const uint32_t q = quad[(size_t)b * ap.H * ap.W + (size_t)i * ap.W + j];
        const uint32_t label = assign_pixel_generic(ap, i, j, q, cinfo + (size_t)b * ap.K,
                                                    cell_start + (size_t)b * (ap.ncell + 1),
                                                    labels + (size_t)b * ap.H * ap.W, nullptr);
        if (UPDATE && label != 0xFFFF) acc_add_pixel(acc + (size_t)b * ap.K * 4, label, i, j, q);
    }
}
