// fast_slic_b200/csrc/realdist.cuh -- the float-distance variants of the assign step (SURVEY.md section 8(f) row 3).
//
// Replaces ContextRealDist (BaseContext<float>::assign_clusters, fast-slic/src/context.cpp:259-298 with the float
// patch of :23-33), ContextRealDistL2::assign_clusters / set_spatial_patch (:394-445) and
// ContextRealDistNoQ::assign_clusters_proto<true> (:462-499).  The scheduler (assign(), :200-243) and the update's integer
// sums (:302-357) are the default path's; only the distance, the window of the NoQ variant and its float centroids
// (:375-381) differ.  Correctness first: one thread per pixel gathers over the cell grid (gather_min, like
// assign_pixel_generic); every float operation is written with an explicit rounding intrinsic in the order of the
// reference's object code, so labels and clusters are bit-identical (tests/test_parity_gpu.py::test_real_dist_variants).
//   VARIANT 0  d = coef * (|di| + |dj|)  +  (|dr| + |dg| + |db|)                     one multiply, one add
//   VARIANT 1  d = fma(dj', dj', di' * di')  +  (dr^2 + dg^2 + db^2),  di' = coef * di   (GCC fuses the patch like this)
//   VARIANT 2  d = |r - cr| + |g - cg| + |b - cb| + |coef (j - cx)| + |coef (i - cy)|  on float centroids, left to right
// With manhattan_spatial_dist off (ap.manhattan == 0) variant 0 takes coef * hypotf(di, dj) (euclid_dist, one multiply)
// and variant 2 the squared form of assign_clusters_proto<false> (:462-496) as the reference's object code evaluates it:
//   d = fma(dx, dx, fma(db, db, fma(dr, dr, dg * dg))) + dy * dy       (dy * dy hoisted out of the row loop)
// Variant 1 ignores the flag (ContextRealDistL2::set_spatial_patch, :435-445).
// Ties: strict '>' against the running minimum in visiting order => minimum of (d, phase, k); non-negative floats
// order like their bit patterns, so the key is  float_bits(d) << 32 | phase << 16 | k.
#pragma once
#include "assign.cuh"

// The float distance of pixel (i, j) with colour q to candidate r (its record cl[k] for the NoQ variant); false when
// r's window does not cover the pixel.  Used by k_assign_real and k_trace_pass.
template <int VARIANT>
__device__ __forceinline__ bool real_dist(const AssignParams& ap, int i, int j, uint32_t q, const CInfo& r,
                                          const fslic_cluster* __restrict__ cl, uint32_t& bits) {
    const int S = ap.S;
    const float coef = ap.coef, fS = (float)S;
    const int qr = q & 0xff, qg = (q >> 8) & 0xff, qb = (q >> 16) & 0xff;
    float d;
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
    bits = __float_as_uint(d);
    return true;
}

template <int VARIANT, bool UPDATE>
__global__ void __launch_bounds__(256) k_assign_real(AssignParams ap, const uint32_t* __restrict__ quad,
                                                      uint16_t* __restrict__ labels, const CInfo* __restrict__ cinfo,
                                                      const int* __restrict__ cell_start,
                                                      const fslic_cluster* __restrict__ clusters,
                                                      unsigned long long* __restrict__ acc) {
    const long total = (long)ap.nsub * ap.W * ap.B;
    const int W = ap.W, H = ap.H;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        int b, i, j;
        pass_pixel(ap, t, b, i, j);
        const size_t img_off = (size_t)b * H * W;
        const uint32_t q = quad[img_off + (size_t)i * W + j];
        const fslic_cluster* cl = clusters + (size_t)b * ap.K;
        const auto dist = [&](const CInfo& r, uint32_t& d) { return real_dist<VARIANT>(ap, i, j, q, r, cl, d); };
        // the NoQ window is cut from float centres: one more row / column to look at
        const unsigned long long best = gather_min(ap, i, j, ap.S + (VARIANT == 2 ? 1 : 0), cinfo + (size_t)b * ap.K,
                                                   cell_start + (size_t)b * (ap.ncell + 1), dist);
        const uint32_t label = store_label<false>(ap, best, i, labels + img_off + (size_t)i * W + j);
        if (UPDATE && label != 0xFFFF) acc_add_pixel(acc + (size_t)b * ap.K * 4, label, i, j, q);
    }
}
