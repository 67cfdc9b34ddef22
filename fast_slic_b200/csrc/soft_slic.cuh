// fast_slic_b200/csrc/soft_slic.cuh -- differentiable soft SLIC (DESIGN.md section 4.20): SSN-style soft associations of
// every pixel with the 9 grid cells around it, the association-weighted cell means, the gather back to pixels, and the
// exact backward of each.  No counterpart in the reference.  Every float operation is one separately rounded IEEE
// operation (no contraction) in the order the contract gives, and no float atomics, so a numpy restatement reproduces
// every bit:
//   grid     pixel (i, j) is in cell (a, b) = (i*nh / H, j*nw / W), label a*nw + b
//   slots    slot n = (da+1)*3 + (db+1) of a pixel is cell (a+da, b+db); a slot outside the grid is invalid: its value
//            is +0.0 and it takes part in no sum; sums over slots run over the valid ones in n order from +0.0
//   block    the pixels whose own cell is within +-1 of cell k in both directions, a rectangle; a sum over it deals the
//            block's pixels in raster order to 32 lanes (lane l adds pixels l, l+32, .. from +0.0), then the butterfly
//            o = 16, 8, 4, 2, 1, as pool.cuh does
//   channels sums over c run in c order from +0.0
// Layouts: per-pixel maps [B,C,H,W], associations and slot gradients [B,9,H,W], per-cell maps [B,C,K], Z [B,K].
#pragma once
#include "cellgrid.cuh"
#include "common.cuh"
#include "glibc_expf.cuh"

#define SS_SLOTS 9
#define SS_CG 8  // channels one warp of k_ss_cell_sum sums per walk over the block

struct SsGrid {
    int H, W, C, nh, nw, K;
};

__device__ __forceinline__ int ss_cell_row(const SsGrid& g, int i) { return (int)((long long)i * g.nh / g.H); }
__device__ __forceinline__ int ss_cell_col(const SsGrid& g, int j) { return (int)((long long)j * g.nw / g.W); }
// the first row of cell row a (a = nh gives H): the least i with i*nh >= a*H; likewise for columns
__device__ __forceinline__ int ss_row0(const SsGrid& g, int a) { return (int)(((long long)a * g.H + g.nh - 1) / g.nh); }
__device__ __forceinline__ int ss_col0(const SsGrid& g, int b) { return (int)(((long long)b * g.W + g.nw - 1) / g.nw); }

// The 9 slot cells of pixel (i, j): k[n] is the cell of slot n, the pixel's own cell where the slot is invalid (so
// that every load stays in bounds), and bit n of the result is set iff slot n is valid
__device__ __forceinline__ unsigned ss_slots(const SsGrid& g, int i, int j, int (&k)[SS_SLOTS]) {
    const int a = ss_cell_row(g, i), b = ss_cell_col(g, j);
    unsigned valid = 0;
#pragma unroll
    for (int n = 0; n < SS_SLOTS; n++) {
        const int aa = a + n / 3 - 1, bb = b + n % 3 - 1;
        const bool ok = aa >= 0 && aa < g.nh && bb >= 0 && bb < g.nw;
        k[n] = ok ? aa * g.nw + bb : a * g.nw + b;
        valid |= (unsigned)ok << n;
    }
    return valid;
}

// Grid-stride loop over the items t of the call (pixels t = b*hw + p, or cells t = b*K + k)
#define SS_FOR(n)                                                                           \
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < (n); t += (long)gridDim.x * blockDim.x)

// Forward of soft_assign, one thread per pixel: d_n = sum_c (f_c - mu_{k(n)c})^2 (fs_acc), m = the fminf fold of the
// valid d_n in n order, e_n = expf(m - d_n) (glibc's, glibc_expf.cuh), s = sum_n e_n, q_n = e_n / s.  Every f_c is
// read once; the centroids [B,C,K] come through the read-only cache.
__global__ void __launch_bounds__(256) k_ss_assign(SsGrid g, long n, const float* __restrict__ feat,
                                                   const float* __restrict__ mu, float* __restrict__ q) {
    const long hw = (long)g.H * g.W;
    SS_FOR(n) {
        const long b = t / hw, p = t - b * hw;
        const int i = (int)(p / g.W), j = (int)(p - (long)i * g.W);
        int k[SS_SLOTS];
        const unsigned valid = ss_slots(g, i, j, k);
        const float* f = feat + b * g.C * hw + p;
        const float* m = mu + b * g.C * g.K;
        float d[SS_SLOTS];
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) d[s] = 0.f;
        for (int c = 0; c < g.C; c++) {
            const float x = __ldg(f + (long)c * hw);
            const float* mc = m + (long)c * g.K;
#pragma unroll
            for (int s = 0; s < SS_SLOTS; s++) d[s] = fs_acc(d[s], x, __ldg(mc + k[s]));
        }
        float lo = 0.f;
        bool any = false;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) {
            if (valid >> s & 1) {
                lo = any ? fminf(lo, d[s]) : d[s];
                any = true;
            }
        }
        float e[SS_SLOTS], sum = 0.f;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) {
            e[s] = gexpf::expf(__fsub_rn(lo, d[s]));
            if (valid >> s & 1) sum = __fadd_rn(sum, e[s]);
        }
        float* o = q + b * SS_SLOTS * hw + p;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) o[(long)s * hw] = valid >> s & 1 ? __fdiv_rn(e[s], sum) : 0.f;
    }
}

enum SsTerm {
    SS_POOL = 0,  // sum of w*v and of w: M = A / Z where Z != 0, else 0 (soft_pool forward)
    SS_SUM = 1,   // sum of w*v (soft_unpool backward: gM)
    SS_DIFF = 2,  // -2 * sum of w*(f - mu_k) (soft_assign backward: gmu, w = gd)
};

// One warp per (image, cell, group of SS_CG channels), grid-stride: walks the cell's block in the lane order above.
// w [B,9,H,W] is read at the slot through which each block pixel sees the cell; v [B,C,H,W].  SS_POOL: out = M [B,C,K]
// and z = Z [B,K] (written by the first group; every group sums Z itself, in the same order).  SS_SUM: out = the sums.
// SS_DIFF: out = -2 * the sums of w * (v - mu_k) (mu [B,C,K]).
template <int TERM>
__global__ void __maxnreg__(80) k_ss_cell_sum(SsGrid g, long nwarps, const float* __restrict__ w,
                                                     const float* __restrict__ v, const float* __restrict__ mu,
                                                     float* __restrict__ out, float* __restrict__ z) {
    const long hw = (long)g.H * g.W;
    const int lane = threadIdx.x & 31, groups = (g.C + SS_CG - 1) / SS_CG;
    for (long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; wid < nwarps;
         wid += ((long)gridDim.x * blockDim.x) >> 5) {
        const long bk = wid / groups;
        const int c0 = (int)(wid - bk * groups) * SS_CG, cn = min(SS_CG, g.C - c0);
        const long b = bk / g.K;
        const int k = (int)(bk - b * g.K), a = k / g.nw, bb = k - a * g.nw;
        const int r0 = ss_row0(g, max(a - 1, 0)), r1 = ss_row0(g, min(a + 2, g.nh));
        const int q0 = ss_col0(g, max(bb - 1, 0)), q1 = ss_col0(g, min(bb + 2, g.nw));
        const int bw = q1 - q0, nb = (r1 - r0) * bw;
        const float* wb = w + b * SS_SLOTS * hw;
        const float* vb = v + (b * g.C + c0) * hw;
        float acc[SS_CG], zs = 0.f, m[SS_CG];
#pragma unroll
        for (int u = 0; u < SS_CG; u++) {
            acc[u] = 0.f;
            m[u] = TERM == SS_DIFF && u < cn ? __ldg(mu + (b * g.C + c0 + u) * g.K + k) : 0.f;
        }
        for (int e = lane; e < nb; e += 32) {
            const int di = e / bw, i = r0 + di, j = q0 + (e - di * bw);
            const int s = (a - ss_cell_row(g, i) + 1) * 3 + (bb - ss_cell_col(g, j) + 1);
            const long p = (long)i * g.W + j;
            const float x = __ldg(wb + (long)s * hw + p);
            if (TERM == SS_POOL) zs = __fadd_rn(zs, x);
#pragma unroll
            for (int u = 0; u < SS_CG; u++) {
                if (u < cn) {
                    const float y = __ldg(vb + (long)u * hw + p);
                    acc[u] = __fadd_rn(acc[u], __fmul_rn(x, TERM == SS_DIFF ? __fsub_rn(y, m[u]) : y));
                }
            }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            if (TERM == SS_POOL) zs = __fadd_rn(zs, __shfl_xor_sync(FSLIC_FULL, zs, o));
#pragma unroll
            for (int u = 0; u < SS_CG; u++) acc[u] = __fadd_rn(acc[u], __shfl_xor_sync(FSLIC_FULL, acc[u], o));
        }
        if (lane == 0) {
            float* ob = out + (b * g.C + c0) * g.K + k;
#pragma unroll
            for (int u = 0; u < SS_CG; u++) {
                if (u < cn) {
                    float r = acc[u];
                    if (TERM == SS_POOL) r = zs != 0.f ? __fdiv_rn(acc[u], zs) : 0.f;
                    if (TERM == SS_DIFF) r = __fmul_rn(-2.f, acc[u]);
                    ob[(long)u * g.K] = r;
                }
            }
            if (TERM == SS_POOL && c0 == 0) z[bk] = zs;
        }
    }
}

// One thread per pixel and every channel: out_c = sum over the valid slots n of w_n * x_{k(n)c} (SS_SUM; the soft_unpool
// forward and soft_pool's gV), or 2 * sum_n w_n * (f_c - mu_{k(n)c}) (SS_DIFF; soft_assign's gF, w = gd, f = feat).
// x [B,C,K], w [B,9,H,W], feat and out [B,C,H,W].
template <int TERM>
__global__ void __launch_bounds__(256) k_ss_unpool(SsGrid g, long n, const float* __restrict__ x,
                                                   const float* __restrict__ w, const float* __restrict__ feat,
                                                   float* __restrict__ out) {
    const long hw = (long)g.H * g.W;
    SS_FOR(n) {
        const long b = t / hw, p = t - b * hw;
        const int i = (int)(p / g.W), j = (int)(p - (long)i * g.W);
        int k[SS_SLOTS];
        const unsigned valid = ss_slots(g, i, j, k);
        float ws[SS_SLOTS];
        const float* wp = w + b * SS_SLOTS * hw + p;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) ws[s] = __ldg(wp + (long)s * hw);
        const float* xb = x + b * g.C * g.K;
        const float* fp = feat + b * g.C * hw + p;
        float* op = out + b * g.C * hw + p;
        for (int c = 0; c < g.C; c++) {
            const float* xc = xb + (long)c * g.K;
            const float f = TERM == SS_DIFF ? __ldg(fp + (long)c * hw) : 0.f;
            float acc = 0.f;
#pragma unroll
            for (int s = 0; s < SS_SLOTS; s++) {
                if (valid >> s & 1) {
                    const float y = __ldg(xc + k[s]);
                    acc = __fadd_rn(acc, __fmul_rn(ws[s], TERM == SS_DIFF ? __fsub_rn(f, y) : y));
                }
            }
            op[(long)c * hw] = TERM == SS_DIFF ? __fmul_rn(2.f, acc) : acc;
        }
    }
}

// One thread per pixel: gq_n = sum_c x_{k(n)c} * y_c (+ add_{k(n)} when add is given) for the valid slots, +0.0 for the
// invalid ones.  x [B,C,K], y [B,C,H,W], add [B,K], gq [B,9,H,W].  Both soft_pool's and soft_unpool's gQ.
__global__ void __launch_bounds__(256) k_ss_slot_dot(SsGrid g, long n, const float* __restrict__ x,
                                                     const float* __restrict__ y, const float* __restrict__ add,
                                                     float* __restrict__ gq) {
    const long hw = (long)g.H * g.W;
    SS_FOR(n) {
        const long b = t / hw, p = t - b * hw;
        const int i = (int)(p / g.W), j = (int)(p - (long)i * g.W);
        int k[SS_SLOTS];
        const unsigned valid = ss_slots(g, i, j, k);
        const float* xb = x + b * g.C * g.K;
        const float* yp = y + b * g.C * hw + p;
        float acc[SS_SLOTS];
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) acc[s] = 0.f;
#pragma unroll 1
        for (int c = 0; c < g.C; c++) {
            const float yc = __ldg(yp + (long)c * hw);
            const float* xc = xb + (long)c * g.K;
#pragma unroll
            for (int s = 0; s < SS_SLOTS; s++) acc[s] = __fadd_rn(acc[s], __fmul_rn(__ldg(xc + k[s]), yc));
        }
        float* o = gq + b * SS_SLOTS * hw + p;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) {
            float r = add ? __fadd_rn(acc[s], __ldg(add + b * g.K + k[s])) : acc[s];
            o[(long)s * hw] = valid >> s & 1 ? r : 0.f;
        }
    }
}

// The softmax backward of one pixel per thread: t = sum_n q_n * g_n over the valid slots, gd_n = q_n * (t - g_n), +0.0
// on the invalid slots.  q, gq, gd [B,9,H,W].
__global__ void __launch_bounds__(256) k_ss_softmax_bwd(SsGrid g, long n, const float* __restrict__ q,
                                                        const float* __restrict__ gq, float* __restrict__ gd) {
    const long hw = (long)g.H * g.W;
    SS_FOR(n) {
        const long b = t / hw, p = t - b * hw;
        const int i = (int)(p / g.W), j = (int)(p - (long)i * g.W);
        int k[SS_SLOTS];
        const unsigned valid = ss_slots(g, i, j, k);
        const long base = b * SS_SLOTS * hw + p;
        float qs[SS_SLOTS], gs[SS_SLOTS], dot = 0.f;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) {
            qs[s] = __ldg(q + base + (long)s * hw);
            gs[s] = __ldg(gq + base + (long)s * hw);
            if (valid >> s & 1) dot = __fadd_rn(dot, __fmul_rn(qs[s], gs[s]));
        }
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++)
            gd[base + (long)s * hw] = valid >> s & 1 ? __fmul_rn(qs[s], __fsub_rn(dot, gs[s])) : 0.f;
    }
}

// soft_pool's backward through the division, one thread per (image, cell): where Z != 0, gA_c = gM_c / Z and
// gZ = -(sum_c gA_c * M_c); where Z == 0, gA = gZ = +0.0.  gm, m, ga [B,C,K]; z, gz [B,K].
__global__ void __launch_bounds__(256) k_ss_pool_grad(SsGrid g, long nk, const float* __restrict__ gm,
                                                      const float* __restrict__ m, const float* __restrict__ z,
                                                      float* __restrict__ ga, float* __restrict__ gz) {
    SS_FOR(nk) {
        const long b = t / g.K, k = t - b * g.K;
        const float zk = z[t];
        const long o = b * g.C * g.K + k;
        float acc = 0.f;
        for (int c = 0; c < g.C; c++) {
            const float a = zk != 0.f ? __fdiv_rn(gm[o + (long)c * g.K], zk) : 0.f;
            ga[o + (long)c * g.K] = a;
            if (zk != 0.f) acc = __fadd_rn(acc, __fmul_rn(a, m[o + (long)c * g.K]));
        }
        gz[t] = zk != 0.f ? -acc : 0.f;
    }
}

// labels [B,H,W] = the cell of each pixel's first largest q over its valid slots, a NaN counting as the maximum (as in
// paint_argmax)
__global__ void __launch_bounds__(256) k_ss_argmax(SsGrid g, long n, const float* __restrict__ q,
                                                   uint16_t* __restrict__ labels) {
    const long hw = (long)g.H * g.W;
    SS_FOR(n) {
        const long b = t / hw, p = t - b * hw;
        const int i = (int)(p / g.W), j = (int)(p - (long)i * g.W);
        int k[SS_SLOTS];
        const unsigned valid = ss_slots(g, i, j, k);
        const float* qp = q + b * SS_SLOTS * hw + p;
        bool any = false;
        int best = 0;
        float bv = 0.f;
#pragma unroll
        for (int s = 0; s < SS_SLOTS; s++) {
            if (!(valid >> s & 1) || (any && isnan(bv))) continue;
            const float v = __ldg(qp + (long)s * hw);
            if (!any || isnan(v) || v > bv) {
                bv = v;
                best = k[s];
            }
            any = true;
        }
        labels[t] = (uint16_t)best;
    }
}
