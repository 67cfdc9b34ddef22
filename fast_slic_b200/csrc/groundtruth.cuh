// fast_slic_b200/csrc/groundtruth.cuh -- superpixels scored against a ground-truth map (DESIGN.md section 4.14):
// per-superpixel class histograms, the overlap table behind achievable segmentation accuracy (ASA) and
// undersegmentation error (UE), and boundary recall / precision within a Chebyshev tolerance.  No counterpart in the
// reference.  Integer only: every result is exact and independent of the launch order.
//
//   k_gt_histogram    one thread per pixel: lanes of a warp with the same (image, label, class) add once (MATCH.ANY),
//                     the leader with one int32 atomicAdd;
//   k_gt_keys         one 64-bit key per pixel, image << (16 + gbits) | label << gbits | gt, all ones in the bits in use
//                     for a pixel that is not counted;
//   (radix sort of the keys over the bits in use, run-length encoding: one run per (image, label, gt) with its count)
//   k_gt_run_totals   n_k and max_g n_kg per (image, label) from the runs;
//   k_gt_run_ue       min(n_kg, n_k - n_kg) per run, added per (image, label);
//   k_gt_reduce       one block per image: the pixel, ASA and UE sums over its labels;
//   k_gt_bitmaps      one warp per 32 columns of a row: superpixel boundary, gt boundary and gt valid bits (BALLOT);
//   k_gt_boundary_counts  one thread per bitmap word: the bitmaps ORed over the (2r+1)^2 window, four popc counts,
//                     one warp reduction and one int64 atomicAdd per warp and term.
#pragma once
#include <limits.h>

#include "common.cuh"

// The eight fields of one image's scores in d_out [batch][GT_FIELDS] (int64)
#define GT_PIXELS 0
#define GT_ASA 1
#define GT_UE 2
#define GT_BOUNDARY 3
#define GT_BOUNDARY_HITS 4
#define GT_SP_BOUNDARY 5
#define GT_SP_BOUNDARY_HITS 6
#define GT_FIELDS 7

// A gt value is valid when it is in [0, 2^31 - 1] and is not the ignore index
template <typename T>
__device__ __forceinline__ bool gt_valid(T v, int has_ignore, long long ignore) {
    const long long g = (long long)v;
    return g >= 0 && g <= INT_MAX && !(has_ignore && g == ignore);
}

// Pixel (i, j) of a map is a superpixel boundary pixel when its right or lower neighbour exists and carries another
// raw label.  p is the pixel's offset in the map.
__device__ __forceinline__ bool gt_sp_boundary(const uint16_t* __restrict__ lab, long p, int i, int j, int H, int W) {
    const uint16_t s = lab[p];
    return (j + 1 < W && lab[p + 1] != s) || (i + 1 < H && lab[p + W] != s);
}

// Image index and in-image offset of pixel t of a call: 32-bit divisions where they suffice
__device__ __forceinline__ long gt_image(long t, long hw, long n) {
    return n <= (long)UINT32_MAX ? (long)((uint32_t)t / (uint32_t)hw) : t / hw;
}

// out [batch*K*C] (zeroed before): out[(b*K + k)*C + c] += 1 for each pixel of image b with label k < K and class
// c in [0, C)
template <typename T>
__global__ void __launch_bounds__(256) k_gt_histogram(const uint16_t* __restrict__ lab, const T* __restrict__ cls, long hw,
                                                       long n, int K, int C, int32_t* __restrict__ out) {
    const long step = (long)gridDim.x * blockDim.x;
    const long nround = (n + step - 1) / step * step;  // whole warps stay in the loop: the warp intrinsics need all lanes
    const int lane = threadIdx.x & 31;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < nround; t += step) {
        unsigned long long key = ~0ull;
        if (t < n) {
            const uint32_t k = lab[t];
            const long long c = (long long)cls[t];
            if (k < (uint32_t)K && c >= 0 && c < C)
                key = ((unsigned long long)gt_image(t, hw, n) * K + k) * (unsigned long long)C + (unsigned long long)c;
        }
        const unsigned peers = __match_any_sync(FSLIC_FULL, key);
        if (key != ~0ull && lane == __ffs(peers) - 1) atomicAdd(&out[key], __popc(peers));
    }
}

// key[t] = image << (16 + gbits) | label << gbits | gt of a counted pixel (valid gt, label < K), else `none` (all ones
// in the bits in use: no counted key reaches it, since label <= 65533)
template <typename T>
__global__ void __launch_bounds__(256) k_gt_keys(const uint16_t* __restrict__ lab, const T* __restrict__ gt, long hw, long n,
                                                  int K, int gbits, int has_ignore, long long ignore, unsigned long long none,
                                                  unsigned long long* __restrict__ key) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const uint32_t k = lab[t];
        const T g = gt[t];
        unsigned long long v = none;
        if (k < (uint32_t)K && gt_valid(g, has_ignore, ignore))
            v = (unsigned long long)gt_image(t, hw, n) << (16 + gbits) | (unsigned long long)k << gbits |
                (unsigned long long)(long long)g;
        key[t] = v;
    }
}

// Over the *nruns runs (unique key, count): nk[image*K + label] += count, mx[image*K + label] = max of the counts
__global__ void __launch_bounds__(256) k_gt_run_totals(const unsigned long long* __restrict__ ukey,
                                                        const int* __restrict__ cnt, const int* __restrict__ nruns,
                                                        unsigned long long none, int gbits, int K,
                                                        uint32_t* __restrict__ nk, uint32_t* __restrict__ mx) {
    const long runs = *nruns;
    for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < runs; r += (long)gridDim.x * blockDim.x) {
        const unsigned long long key = ukey[r];
        if (key == none) continue;
        const long node = (long)(key >> (16 + gbits)) * K + (long)((key >> gbits) & 0xffffu);
        atomicAdd(&nk[node], (uint32_t)cnt[r]);
        atomicMax(&mx[node], (uint32_t)cnt[r]);
    }
}

// ue[image*K + label] += min(n_kg, n_k - n_kg) over the runs, after k_gt_run_totals
__global__ void __launch_bounds__(256) k_gt_run_ue(const unsigned long long* __restrict__ ukey, const int* __restrict__ cnt,
                                                    const int* __restrict__ nruns, unsigned long long none, int gbits, int K,
                                                    const uint32_t* __restrict__ nk, unsigned long long* __restrict__ ue) {
    const long runs = *nruns;
    for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < runs; r += (long)gridDim.x * blockDim.x) {
        const unsigned long long key = ukey[r];
        if (key == none) continue;
        const long node = (long)(key >> (16 + gbits)) * K + (long)((key >> gbits) & 0xffffu);
        const uint32_t c = (uint32_t)cnt[r], rest = nk[node] - c;
        atomicAdd(&ue[node], (unsigned long long)(c < rest ? c : rest));
    }
}

__device__ __forceinline__ unsigned long long gt_warp_sum(unsigned long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FSLIC_FULL, v, o);
    return v;
}

// One block of 256 per image b: out[b][GT_PIXELS / GT_ASA / GT_UE] = the sums of nk, mx and ue over its K labels
__global__ void __launch_bounds__(256) k_gt_reduce(const uint32_t* __restrict__ nk, const uint32_t* __restrict__ mx,
                                                    const unsigned long long* __restrict__ ue, int K,
                                                    long long* __restrict__ out) {
    __shared__ unsigned long long part[3][8];
    const long base = (long)blockIdx.x * K;
    unsigned long long s[3] = {0, 0, 0};
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
        s[0] += nk[base + k];
        s[1] += mx[base + k];
        s[2] += ue[base + k];
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int f = 0; f < 3; f++) {
        s[f] = gt_warp_sum(s[f]);
        if (lane == 0) part[f][warp] = s[f];
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        unsigned long long t = 0;
        for (int w = 0; w < 8; w++) t += part[threadIdx.x][w];
        out[(long)blockIdx.x * GT_FIELDS + (threadIdx.x == 0 ? GT_PIXELS : threadIdx.x == 1 ? GT_ASA : GT_UE)] = (long long)t;
    }
}

// Bitmaps [batch][H][Wd] of u32 words, bit l of word w = column 32 w + l (0 past the last column): sp = superpixel
// boundary, gb = gt boundary, gv = gt valid.  Grid: y over images, x over the H * Wd * 32 columns of an image, one warp
// per word.
template <typename T>
__global__ void __launch_bounds__(256) k_gt_bitmaps(const uint16_t* __restrict__ lab, const T* __restrict__ gt, int batch,
                                                     int H, int W, int Wd, int has_ignore, long long ignore,
                                                     uint32_t* __restrict__ sp, uint32_t* __restrict__ gb,
                                                     uint32_t* __restrict__ gv) {
    // H * Wd < 2^32 for H * W <= 2^29: 32-bit word indices
    const uint32_t words = (uint32_t)H * (uint32_t)Wd;
    const uint32_t warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, wstep = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const uint16_t* l = lab + b * ((long)H * W);
        const T* g = gt + b * ((long)H * W);
        // a warp's lanes are the 32 columns of one word and leave the loop together
        for (uint32_t q = warp0; q < words; q += wstep) {
            const int i = (int)(q / (uint32_t)Wd), w = (int)(q - (uint32_t)i * (uint32_t)Wd), j = w * 32 + lane;
            bool s = false, e = false, ok = false;
            if (j < W) {
                const long p = (long)i * W + j;
                s = gt_sp_boundary(l, p, i, j, H, W);
                const T x = g[p];
                ok = gt_valid(x, has_ignore, ignore);
                if (ok) {
                    if (j + 1 < W) {
                        const T y = g[p + 1];
                        e = gt_valid(y, has_ignore, ignore) && y != x;
                    }
                    if (!e && i + 1 < H) {
                        const T y = g[p + W];
                        e = gt_valid(y, has_ignore, ignore) && y != x;
                    }
                }
            }
            const uint32_t ws = __ballot_sync(FSLIC_FULL, s), we = __ballot_sync(FSLIC_FULL, e),
                           wv = __ballot_sync(FSLIC_FULL, ok);
            if (lane == 0) {
                const long o = b * (long)words + q;
                sp[o] = ws;
                gb[o] = we;
                gv[o] = wv;
            }
        }
    }
}

// Bit c of the result: any of bits c - r .. c + r of the 96 columns (left, mid, right), 0 <= r <= 32
__device__ __forceinline__ uint32_t gt_hdilate(uint32_t left, uint32_t mid, uint32_t right, int r) {
    unsigned long long v = (unsigned long long)right << 32 | mid;  // bit c: columns c .. c + r
    unsigned long long u = (unsigned long long)mid << 32 | left;   // bit 32 + c: columns c - r .. c
    int cover = 1;                                                  // shifts 0 .. cover - 1 are ORed in
    while (cover * 2 <= r + 1) {
        v |= v >> cover;
        u |= u << cover;
        cover *= 2;
    }
    if (r + 1 > cover) {
        const int s = r + 1 - cover;
        v |= v >> s;
        u |= u << s;
    }
    return (uint32_t)v | (uint32_t)(u >> 32);
}

// out[b][GT_BOUNDARY .. GT_SP_BOUNDARY_HITS] += the gt boundary pixels, those with a superpixel boundary pixel in their
// window, the superpixel boundary pixels valid in gt, and those with a gt boundary pixel in their window.  Grid: y over
// images, x over the H * Wd words of an image, one thread per word.
__global__ void __launch_bounds__(256) k_gt_boundary_counts(const uint32_t* __restrict__ sp, const uint32_t* __restrict__ gb,
                                                             const uint32_t* __restrict__ gv, int batch, int H, int Wd,
                                                             int r, long long* __restrict__ out) {
    const uint32_t words = (uint32_t)H * (uint32_t)Wd;  // < 2^32 for H * W <= 2^29
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const uint32_t* s = sp + b * (long)words;
        const uint32_t* e = gb + b * (long)words;
        uint32_t c[4] = {0, 0, 0, 0};
        for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < words; q += gridDim.x * blockDim.x) {
            const int i = (int)(q / (uint32_t)Wd), w = (int)(q - (uint32_t)i * (uint32_t)Wd);
            const int i0 = i - r < 0 ? 0 : i - r, i1 = i + r >= H ? H - 1 : i + r;
            uint32_t vs[3] = {0, 0, 0}, ve[3] = {0, 0, 0};
            for (int ii = i0; ii <= i1; ii++) {
                const long row = (long)ii * Wd;
                if (w > 0) {
                    vs[0] |= s[row + w - 1];
                    ve[0] |= e[row + w - 1];
                }
                vs[1] |= s[row + w];
                ve[1] |= e[row + w];
                if (w + 1 < Wd) {
                    vs[2] |= s[row + w + 1];
                    ve[2] |= e[row + w + 1];
                }
            }
            const uint32_t ds = gt_hdilate(vs[0], vs[1], vs[2], r), de = gt_hdilate(ve[0], ve[1], ve[2], r);
            const uint32_t own_s = s[q] & gv[b * (long)words + q], own_e = e[q];
            c[0] += __popc(own_e);
            c[1] += __popc(own_e & ds);
            c[2] += __popc(own_s);
            c[3] += __popc(own_s & de);
        }
        // at most H * W <= 2^29 per image and term: the warp sums fit u32
#pragma unroll
        for (int f = 0; f < 4; f++) {
            const uint32_t t = __reduce_add_sync(FSLIC_FULL, c[f]);
            if ((threadIdx.x & 31) == 0 && t)
                atomicAdd(reinterpret_cast<unsigned long long*>(&out[b * GT_FIELDS + GT_BOUNDARY + f]),
                          (unsigned long long)t);
        }
    }
}

// out[t] = 1 where pixel t is a superpixel boundary pixel, else 0
__global__ void __launch_bounds__(256) k_gt_boundaries(const uint16_t* __restrict__ lab, long hw, int H, int W, long n,
                                                        uint8_t* __restrict__ out) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const uint32_t p = (uint32_t)(t - gt_image(t, hw, n) * hw);  // hw <= 2^29: 32-bit divisions
        const int i = (int)(p / (uint32_t)W), j = (int)(p - (uint32_t)i * (uint32_t)W);
        out[t] = gt_sp_boundary(lab, t, i, j, H, W) ? 1 : 0;
    }
}

// ---- Volumes (DESIGN.md section 4.24): label volumes u16 [batch, D, H, W] and gt of the same shape.  The overlap keys
// are k_gt_keys' over D * H * W voxels per volume; the boundary terms use 3-D one-sided boundaries and a box window
// |dz| <= rz, |dy| <= ry, |dx| <= rx, dilated separably:
//   k_gt_bitmaps3d        k_gt_bitmaps with the +z neighbour too, over the D * H rows of each volume;
//   k_gt_dilate_yx        one thread per word: the superpixel and gt boundary bitmaps ORed over rows i - ry .. i + ry
//                         of the word's slice and three words, dilated by rx within them;
//   k_gt_boundary_counts3d  one thread per word: those ORed over slices z - rz .. z + rz, then k_gt_boundary_counts'
//                         four popc counts, warp sums and int64 atomicAdds.

// Voxel (z, i, j) of a volume is a supervoxel boundary voxel when its +x, +y or +z neighbour exists and carries another
// raw label.  p is the voxel's offset in the volume, hw = H * W.
__device__ __forceinline__ bool gt_sp_boundary3d(const uint16_t* __restrict__ lab, long p, int z, int i, int j, int D,
                                                 int H, int W, long hw) {
    const uint16_t s = lab[p];
    return (j + 1 < W && lab[p + 1] != s) || (i + 1 < H && lab[p + W] != s) || (z + 1 < D && lab[p + hw] != s);
}

// Bitmaps [batch][D][H][Wd] as k_gt_bitmaps' (sp, gb, gv), with 3-D boundaries.  Grid: y over volumes, x over the
// D * H * Wd * 32 columns of a volume, one warp per word.
template <typename T>
__global__ void __launch_bounds__(256) k_gt_bitmaps3d(const uint16_t* __restrict__ lab, const T* __restrict__ gt,
                                                       int batch, int D, int H, int W, int Wd, int has_ignore,
                                                       long long ignore, uint32_t* __restrict__ sp,
                                                       uint32_t* __restrict__ gb, uint32_t* __restrict__ gv) {
    // D * H * Wd < 2^32 for D * H * W <= 2^29: 32-bit word indices
    const uint32_t words = (uint32_t)D * (uint32_t)H * (uint32_t)Wd;
    const long hw = (long)H * W, dhw = (long)D * hw;
    const uint32_t warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, wstep = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const uint16_t* l = lab + b * dhw;
        const T* g = gt + b * dhw;
        for (uint32_t q = warp0; q < words; q += wstep) {
            const uint32_t row = q / (uint32_t)Wd, w = q - row * (uint32_t)Wd;
            const int z = (int)(row / (uint32_t)H), i = (int)(row - (uint32_t)z * (uint32_t)H), j = (int)w * 32 + lane;
            bool s = false, e = false, ok = false;
            if (j < W) {
                const long p = (long)row * W + j;
                s = gt_sp_boundary3d(l, p, z, i, j, D, H, W, hw);
                const T x = g[p];
                ok = gt_valid(x, has_ignore, ignore);
                if (ok) {
                    if (j + 1 < W) {
                        const T y = g[p + 1];
                        e = gt_valid(y, has_ignore, ignore) && y != x;
                    }
                    if (!e && i + 1 < H) {
                        const T y = g[p + W];
                        e = gt_valid(y, has_ignore, ignore) && y != x;
                    }
                    if (!e && z + 1 < D) {
                        const T y = g[p + hw];
                        e = gt_valid(y, has_ignore, ignore) && y != x;
                    }
                }
            }
            const uint32_t ws = __ballot_sync(FSLIC_FULL, s), we = __ballot_sync(FSLIC_FULL, e),
                           wv = __ballot_sync(FSLIC_FULL, ok);
            if (lane == 0) {
                const long o = b * (long)words + q;
                sp[o] = ws;
                gb[o] = we;
                gv[o] = wv;
            }
        }
    }
}

// ds / de = sp / gb dilated within each slice: bit c of word (z, i, w) is set when a bit of rows i - ry .. i + ry
// (clipped to the slice) and columns c - rx .. c + rx is.  Grid: y over volumes, x over the D * H * Wd words.
__global__ void __launch_bounds__(256) k_gt_dilate_yx(const uint32_t* __restrict__ sp, const uint32_t* __restrict__ gb,
                                                       int batch, int D, int H, int Wd, int ry, int rx,
                                                       uint32_t* __restrict__ ds, uint32_t* __restrict__ de) {
    const uint32_t words = (uint32_t)D * (uint32_t)H * (uint32_t)Wd;
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const uint32_t* s = sp + b * (long)words;
        const uint32_t* e = gb + b * (long)words;
        for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < words; q += gridDim.x * blockDim.x) {
            const uint32_t row = q / (uint32_t)Wd, w = q - row * (uint32_t)Wd;
            const uint32_t z = row / (uint32_t)H;
            const int i = (int)(row - z * (uint32_t)H);
            const int i0 = i - ry < 0 ? 0 : i - ry, i1 = i + ry >= H ? H - 1 : i + ry;
            const uint32_t slice = z * (uint32_t)H * (uint32_t)Wd;
            uint32_t vs[3] = {0, 0, 0}, ve[3] = {0, 0, 0};
            for (int ii = i0; ii <= i1; ii++) {
                const uint32_t r0 = slice + (uint32_t)ii * (uint32_t)Wd + w;
                if (w > 0) {
                    vs[0] |= s[r0 - 1];
                    ve[0] |= e[r0 - 1];
                }
                vs[1] |= s[r0];
                ve[1] |= e[r0];
                if (w + 1 < (uint32_t)Wd) {
                    vs[2] |= s[r0 + 1];
                    ve[2] |= e[r0 + 1];
                }
            }
            ds[b * (long)words + q] = gt_hdilate(vs[0], vs[1], vs[2], rx);
            de[b * (long)words + q] = gt_hdilate(ve[0], ve[1], ve[2], rx);
        }
    }
}

// out[b][GT_BOUNDARY .. GT_SP_BOUNDARY_HITS] += k_gt_boundary_counts' four terms, the windows being ds / de ORed over
// slices z - rz .. z + rz (clipped to the volume).  Grid: y over volumes, x over the D * H * Wd words.
__global__ void __launch_bounds__(256) k_gt_boundary_counts3d(const uint32_t* __restrict__ sp,
                                                               const uint32_t* __restrict__ gb,
                                                               const uint32_t* __restrict__ gv,
                                                               const uint32_t* __restrict__ ds,
                                                               const uint32_t* __restrict__ de, int batch, int D,
                                                               int H, int Wd, int rz, long long* __restrict__ out) {
    const uint32_t plane = (uint32_t)H * (uint32_t)Wd, words = (uint32_t)D * plane;
    for (long b = blockIdx.y; b < batch; b += gridDim.y) {
        const long o = b * (long)words;
        uint32_t c[4] = {0, 0, 0, 0};
        for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < words; q += gridDim.x * blockDim.x) {
            const int z = (int)(q / plane);
            const uint32_t r = q - (uint32_t)z * plane;
            const int z0 = z - rz < 0 ? 0 : z - rz, z1 = z + rz >= D ? D - 1 : z + rz;
            uint32_t ws = 0, we = 0;
            for (int zz = z0; zz <= z1; zz++) {
                ws |= ds[o + (uint32_t)zz * plane + r];
                we |= de[o + (uint32_t)zz * plane + r];
            }
            const uint32_t own_s = sp[o + q] & gv[o + q], own_e = gb[o + q];
            c[0] += __popc(own_e);
            c[1] += __popc(own_e & ws);
            c[2] += __popc(own_s);
            c[3] += __popc(own_s & we);
        }
        // at most D * H * W <= 2^29 per volume and term: the warp sums fit u32
#pragma unroll
        for (int f = 0; f < 4; f++) {
            const uint32_t t = __reduce_add_sync(FSLIC_FULL, c[f]);
            if ((threadIdx.x & 31) == 0 && t)
                atomicAdd(reinterpret_cast<unsigned long long*>(&out[b * GT_FIELDS + GT_BOUNDARY + f]),
                          (unsigned long long)t);
        }
    }
}

// out[t] = 1 where voxel t is a supervoxel boundary voxel, else 0
__global__ void __launch_bounds__(256) k_gt_boundaries3d(const uint16_t* __restrict__ lab, uint32_t dhw, int D, int H,
                                                          int W, long n, uint8_t* __restrict__ out) {
    const uint32_t hw = (uint32_t)H * (uint32_t)W;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long)gridDim.x * blockDim.x) {
        const uint32_t p = (uint32_t)(t - gt_image(t, dhw, n) * (long)dhw);  // dhw <= 2^29: 32-bit divisions
        const uint32_t z = p / hw, r = p - z * hw, i = r / (uint32_t)W, j = r - i * (uint32_t)W;
        out[t] = gt_sp_boundary3d(lab, t, (int)z, (int)i, (int)j, D, H, W, (long)hw) ? 1 : 0;
    }
}
