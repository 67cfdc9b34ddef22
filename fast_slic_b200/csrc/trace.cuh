// fast_slic_b200/csrc/trace.cuh -- per-pass snapshots of the engine state for debug_mode (fslic_b200_set_trace).
//
// The reference's Recorder (recorder.h; pushed at context.cpp:157,173) copies, after seeding and after every
// assign + update of the subsampled loop: the pre-CCA assignment, the per-pixel minimum distance and the K cluster
// records.  The assign kernels here keep no per-pixel minimum, so k_trace_pass recomputes it from the records the pass
// read, one thread per pixel over the cell grid with the gather (gather_min) and distance functions of the per-pixel
// assign kernels.  It also recomputes the argmin and counts the pixels whose label the pass set differently.  For the u16
// default path that is an independent check of the tile kernels (TMA, LDG), whose candidate lists, shared-memory patch
// and packed keys share no code with the trace (it computes the spatial term inline and never reads the patch); for the
// generic, `preemptive`, float and LSC kernels the trace runs the same code, so there it only catches races and launch
// errors.
//
// What a snapshot holds (context.cpp:200-206, 289-294):
//   * min_dists is reset to the type's maximum on EVERY pixel at the start of an assign, so rows outside the pass,
//     pixels no window covers and (preemptive) pixels covered by inactive clusters only read 65535 / FLT_MAX;
//   * the assignment starts at 0xFFFF and keeps earlier passes' labels where no window reaches.
#pragma once
#include <float.h>
#include "assign.cuh"
#include "lsc.cuh"
#include "realdist.cuh"

struct TraceParams {
    AssignParams ap;    // geometry of the pass (H, W, K, S, B, stride, rem, cell grid, coef, manhattan)
    int fresh_after;    // rows with (i % stride) >= fresh_after have not been assigned by any pass yet
    int preempt;        // 1: inactive clusters are not candidates (context.cpp:218)
    long long img_pitch;  // elements between two images' snapshots of the same slot: T * H * W
    const float* feat;  // LSC: normalised pixel features [B][10][N] and the centroid features [B][K][LSC_CF] the pass read
    const float* cf;
};

// KIND -1: the u16 distance of the default contexts (u16_dist, its spatial term computed inline as in
// k_assign_generic); 0 / 1 / 2: the float-distance variants (real_dist); 4: LSC (lsc_dist over the centroid
// features the pass read).  out_assign / out_dist point at the pass's slot of image 0.
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
            const fslic_cluster* cl = clusters + (size_t)b * ap.K;
            const float* cf = tp.cf + (size_t)b * ap.K * LSC_CF;
            float x[LSC_NF];
            if constexpr (KIND == 4) {
#pragma unroll
                for (int f = 0; f < LSC_NF; f++) x[f] = tp.feat[((size_t)b * LSC_NF + f) * per_img + p];
            }
            const auto dist = [&](const CInfo& r, uint32_t& d) {
                if constexpr (KIND < 0) {
                    return u16_dist<0>(ap, i, j, q, r, tp.preempt != 0, cl, nullptr, d);
                } else if constexpr (KIND == 4) {
                    const int cy = (int16_t)(r.cyx & 0xffff), cx = r.cyx >> 16;
                    if (abs(i - cy) > S || abs(j - cx) > S) return false;
                    return lsc_dist(x, cf + (size_t)(r.sortkey & 0xffffu) * LSC_CF, d);
                } else {
                    return real_dist<KIND>(ap, i, j, q, r, cl, d);
                }
            };
            best = gather_min(ap, i, j, S + (KIND == 2 ? 1 : 0), cinfo + (size_t)b * ap.K,
                              cell_start + (size_t)b * (ap.ncell + 1), dist);
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
