// fast_slic_b200/csrc/trace.cuh -- per-pass snapshots of the engine state for debug_mode (fslic_b200_set_trace).
//
// The reference's Recorder (recorder.h; pushed at context.cpp:157,173) copies, after seeding and after every
// assign + update of the subsampled loop: the pre-CCA assignment, the per-pixel minimum distance and the K cluster
// records.  The assign kernels here keep no per-pixel minimum, so k_trace_pass recomputes it from the records the pass
// read, with the pass's own distance functions, one thread per pixel over the cell grid (the structure of
// k_assign_preempt / k_assign_real).  It also recomputes the argmin and counts the pixels whose label the pass set
// differently.  For the u16 default path that is an independent check of the tile kernels (TMA, LDG), whose candidate
// lists, shared-memory patch and packed keys share no code with this gather; for the generic, `preemptive`, float and LSC
// kernels the trace restates the same per-pixel gather and distance, so there it only catches races and launch errors.
//
// What a snapshot holds (context.cpp:200-206, 289-294):
//   * min_dists is reset to the type's maximum on EVERY pixel at the start of an assign, so rows outside the pass,
//     pixels no window covers and (preemptive) pixels covered by inactive clusters only read 65535 / FLT_MAX;
//   * the assignment starts at 0xFFFF and keeps earlier passes' labels where no window reaches.
#pragma once
#include <float.h>
#include "assign.cuh"
#include "lsc.cuh"

// The float distance of k_assign_real<VARIANT> (realdist.cuh: the same operations with the same rounding intrinsics, in
// the same order) of pixel (i, j), colour (qr, qg, qb), to candidate `r` (its record cl[k] for the NoQ variant); false
// when the candidate's window does not cover the pixel.  Kept apart so that the assign kernel's code stays as it is.
template <int VARIANT>
__device__ __forceinline__ bool trace_real_dist(const AssignParams& ap, int i, int j, int qr, int qg, int qb,
                                                const CInfo& r, const fslic_cluster* __restrict__ cl, float& d) {
    const int S = ap.S;
    const float coef = ap.coef, fS = (float)S;
    if (VARIANT == 2) {
        const fslic_cluster c = cl[r.sortkey & 0xffffu];
        // context.cpp:472-473: my_max<int>(cy - S, 0) .. my_min<int>(cy + S + 1, H), float arithmetic truncated
        const int i0 = max((int)__fsub_rn(c.y, fS), 0), i1 = min((int)__fadd_rn(__fadd_rn(c.y, fS), 1.0f), ap.H);
        const int j0 = max((int)__fsub_rn(c.x, fS), 0), j1 = min((int)__fadd_rn(__fadd_rn(c.x, fS), 1.0f), ap.W);
        if (i < i0 || i >= i1 || j < j0 || j >= j1) return false;
        const float dr = __fsub_rn((float)qr, c.r), dg = __fsub_rn((float)qg, c.g), db = __fsub_rn((float)qb, c.b);
        const float dy = __fmul_rn(coef, __fsub_rn((float)i, c.y)), dx = __fmul_rn(coef, __fsub_rn((float)j, c.x));
        if (ap.manhattan)
            d = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(fabsf(dr), fabsf(dg)), fabsf(db)), fabsf(dx)), fabsf(dy));
        else
            d = __fadd_rn(__fmaf_rn(dx, dx, __fmaf_rn(db, db, __fmaf_rn(dr, dr, __fmul_rn(dg, dg)))), __fmul_rn(dy, dy));
    } else {
        const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
        const int di = i - cy, dj = j - cx;
        if (abs(di) > S || abs(dj) > S) return false;
        const int cr_ = r.color & 0xff, cg_ = (r.color >> 8) & 0xff, cb_ = (r.color >> 16) & 0xff;
        if (VARIANT == 0) {
            const float patch = __fmul_rn(coef, ap.manhattan ? (float)(abs(di) + abs(dj)) : euclid_dist(di, dj));
            d = __fadd_rn(patch, (float)(abs(qr - cr_) + abs(qg - cg_) + abs(qb - cb_)));
        } else {
            const float fdi = __fmul_rn(coef, (float)di), fdj = __fmul_rn(coef, (float)dj);
            const float patch = __fmaf_rn(fdj, fdj, __fmul_rn(fdi, fdi));
            const int er = qr - cr_, eg = qg - cg_, eb = qb - cb_;
            d = __fadd_rn(patch, (float)(er * er + eg * eg + eb * eb));  // < 2^24: exact in float
        }
    }
    return true;
}

struct TraceParams {
    AssignParams ap;    // geometry of the pass (H, W, K, S, B, stride, rem, cell grid, coef, manhattan)
    int fresh_after;    // rows with (i % stride) >= fresh_after have not been assigned by any pass yet
    int preempt;        // 1: inactive clusters are not candidates (context.cpp:218)
    long long img_pitch;  // elements between two images' snapshots of the same slot: T * H * W
    const float* feat;  // LSC: normalised pixel features [B][10][N] and the centroid features [B][K][LSC_CF] the pass read
    const float* cf;
};

// KIND -1: u16 distance of the default contexts (spatial_u16 + sad4_acc, like assign_pixel_generic); 0 / 1 / 2: the
// float-distance variants (trace_real_dist); 4: LSC, the fused chain fma(diff, diff, d) over the ten features of
// k_assign_lsc (lsc.cpp:212-216), candidates with d >= FLT_MAX or NaN (an emptied cluster's 0/0 centroid) left out.
// out_assign / out_dist point at the pass's slot of image 0.
template <int KIND>
__global__ void __launch_bounds__(256) k_trace_pass(TraceParams tp, const uint32_t* __restrict__ quad,
                                                     const uint16_t* __restrict__ labels, const CInfo* __restrict__ cinfo,
                                                     const int* __restrict__ cell_start,
                                                     const fslic_cluster* __restrict__ clusters,
                                                     uint16_t* __restrict__ out_assign, void* __restrict__ out_dist,
                                                     unsigned int* __restrict__ mismatches) {
    const AssignParams& ap = tp.ap;
    const int S = ap.S, W = ap.W, H = ap.H;
    const long per_img = (long)H * W;
    const long total = per_img * ap.B;
    unsigned int bad = 0;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int b = (int)(t / per_img);
        const long p = t - (long)b * per_img;
        const int i = (int)(p / W), j = (int)(p - (long)i * W);
        const size_t img_off = (size_t)b * per_img;
        const uint16_t label = labels[img_off + p];
        const size_t o = (size_t)b * tp.img_pitch + p;
        out_assign[o] = (i % ap.stride) >= tp.fresh_after ? (uint16_t)0xFFFF : label;
        const bool in_pass = (i % ap.stride) == ap.rem;
        unsigned long long best = ~0ull;
        if (in_pass) {
            const uint32_t q = quad[img_off + p];
            const CInfo* ci = cinfo + (size_t)b * ap.K;
            const int* cs = cell_start + (size_t)b * (ap.ncell + 1);
            const fslic_cluster* cl = clusters + (size_t)b * ap.K;
            const int m = S + (KIND == 2 ? 1 : 0);
            const int cr0 = max(i - m, 0) / ap.G, cr1 = min(i + m, H - 1) / ap.G;
            const int cc0 = max(j - m, 0) / ap.G, cc1 = min(j + m, W - 1) / ap.G;
            for (int cr = cr0; cr <= cr1; cr++) {
                const int s = cs[cr * ap.cellW + cc0], e = cs[cr * ap.cellW + cc1 + 1];
                for (int u = s; u < e; u++) {
                    const CInfo r = ci[u];
                    uint32_t dk;
                    if (KIND < 0) {
                        const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
                        const int di = i - cy, dj = j - cx;
                        if (abs(di) > S || abs(dj) > S) continue;
                        if (tp.preempt && !cl[r.sortkey & 0xffffu].is_active) continue;
                        dk = sad4_acc(q, r.color, spatial_u16(ap.coef, di, dj, ap.manhattan)) & 0xffffu;
                    } else if (KIND == 4) {
                        const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
                        if (abs(i - cy) > S || abs(j - cx) > S) continue;
                        const float* c = tp.cf + ((size_t)b * ap.K + (r.sortkey & 0xffffu)) * LSC_CF;
                        const float* x = tp.feat + (size_t)b * LSC_NF * per_img + p;
                        float d = 0.f;
#pragma unroll
                        for (int f = 0; f < LSC_NF; f++) {
                            const float diff = __fsub_rn(x[(size_t)f * per_img], c[f]);
                            d = __fmaf_rn(diff, diff, d);
                        }
                        if (!(d < FLT_MAX)) continue;
                        dk = __float_as_uint(d);
                    } else {
                        float d;
                        if (!trace_real_dist<(KIND < 0 || KIND > 2 ? 0 : KIND)>(ap,i, j, q & 0xff, (q >> 8) & 0xff, (q >> 16) & 0xff, r, cl, d))
                            continue;
                        dk = __float_as_uint(d);
                    }
                    const unsigned long long key = ((unsigned long long)dk << 32) | r.sortkey;
                    best = key < best ? key : best;
                }
            }
        }
        // the reference stores a candidate only when it is strictly below the running minimum, which starts at the max
        const bool hit = best != ~0ull && (KIND >= 0 || (uint32_t)(best >> 32) < 0xFFFFu);
        if (hit && (best & 0xffffu) != label) bad++;
        if (KIND < 0)
            static_cast<uint16_t*>(out_dist)[o] = hit ? (uint16_t)(best >> 32) : (uint16_t)0xFFFF;
        else
            static_cast<float*>(out_dist)[o] = hit ? __uint_as_float((uint32_t)(best >> 32)) : FLT_MAX;
    }
    if (bad) atomicAdd(mismatches, bad);
}

// Snapshot -1 (context.cpp:157): the cluster records as iterate() found them, with the colour re-seeded from the quad
// image like the first prepare does (reseed_colour, prepare.cuh) and is_updatable = 2 (PreemptiveGrid::initialize,
// preemptive.h:59-67).  The centres themselves are not clamped yet: that is the first assign's (context.cpp:209-212).
__global__ void k_trace_seed(int H, int W, int K, int B, const uint32_t* __restrict__ quad,
                             const fslic_cluster* __restrict__ clusters, fslic_cluster* __restrict__ out, long long img_pitch) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * K) return;
    const int b = t / K, k = t - b * K;
    fslic_cluster c = clusters[t];
    reseed_colour(c, quad + (size_t)b * H * W, H, W);
    c.is_updatable = 2;
    out[(size_t)b * img_pitch + k] = c;
}

// PreemptiveGrid::finalize (preemptive.h:69-74) for a traced call, whose last prepare left the active set of the final
// update in place so that the last snapshot could record it.
__global__ void k_trace_activate(fslic_cluster* __restrict__ clusters, int n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) clusters[t].is_active = 1;
}
