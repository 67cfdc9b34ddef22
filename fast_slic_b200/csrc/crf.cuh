// crf.cuh -- the reference's SimpleCRF (src/simple-crf.{h,hpp,cpp}): a mean-field CRF over superpixel nodes, linked
// in space by an adjacency list per frame and in time node-to-node between consecutive frames.
//
// Every float operation is the one the reference's object code (g++ -O3 -mavx2 -mfma) performs, in its order, with
// explicit __f*_rn / __fmaf_rn intrinsics so that nvcc contracts nothing on its own, and glibc's expf comes from
// glibc_expf.cuh.  What the object code fuses (simple-crf.hpp:135-174, simple-crf.cpp:62-151):
//   rgb   = -fma(db, db, fma(dr, dr, dg*dg))                 d* = (c1.* - c2.*) / srgb
//   xy    = -fma(dx, dx, dy*dy)                              d* = (c1.* - c2.*) / sxy      (same for smooth_sxy)
//   E_s   = fma(w, expf(fma(rgb, 0.5, xy*0.5)), smooth_w * expf(smooth_xy * 0.5))
//   E_t   = temporal_w * expf(rgb_t * 0.5)
//   msg   = fma(E * q_j, sqrtf((float)m_j / (float)max((int)m_i, 1)), msg)     neighbours in list order, then t-1, t+1
//   acc   = fma(compat[c'], msg[c'], acc)                                    c' != c in class order, compat = 1
//   e_c   = expf(-(unary_c + acc));  s = sum_c e_c;  s = (double)s < 1e-5 ? 1e-5f : s;  q_c = e_c / s
#pragma once
#include <stdint.h>
#include "glibc_expf.cuh"

struct CrfParams {  // == SimpleCRFParams (simple-crf.h:11-19)
    float spatial_w, temporal_w, spatial_srgb, temporal_srgb, spatial_sxy, spatial_smooth_w, spatial_smooth_sxy;
};

// Device view of one frame; the CRF keeps an array of these in time order (index 0 = first_time).
struct CrfFrameDev {
    const fslic_cluster* clusters;  // [N]
    const int32_t* offsets;         // [N + 1] CSR of the adjacency lists
    const int32_t* nbr;             // [E]
    const float* unary;             // [C][N]
    float* q[2];                    // [C][N] ping-pong
    float* msg;                     // [C][N] scratch of one iteration
    float* e_sp;                    // [E] spatial energy of each edge (neighbour -> node)
    float* r_sp;                    // [E] sqrtf((float)m_neighbour / m_node)
    float* tmp;                     // [4][N] energy and ratio to the previous frame, then to the next one
};

__device__ __forceinline__ float crf_sq_sum3(float a, float b, float c) {  // fma(c, c, fma(b, b, a*a))
    return __fmaf_rn(c, c, __fmaf_rn(b, b, __fmul_rn(a, a)));
}

// SimpleCRFFrame::calc_spatial_pairwise_energy(c1, c2) for c1 != c2 (simple-crf.hpp:149-174)
__device__ __forceinline__ float crf_spatial_energy(const fslic_cluster& c1, const fslic_cluster& c2, const CrfParams& p) {
    const float dr = __fdiv_rn(__fsub_rn(c1.r, c2.r), p.spatial_srgb);
    const float dg = __fdiv_rn(__fsub_rn(c1.g, c2.g), p.spatial_srgb);
    const float db = __fdiv_rn(__fsub_rn(c1.b, c2.b), p.spatial_srgb);
    const float rgb = -crf_sq_sum3(dg, dr, db);
    const float dx = __fdiv_rn(__fsub_rn(c1.x, c2.x), p.spatial_sxy);
    const float dy = __fdiv_rn(__fsub_rn(c1.y, c2.y), p.spatial_sxy);
    const float xy = -__fmaf_rn(dx, dx, __fmul_rn(dy, dy));
    const float exponent = __fmaf_rn(rgb, 0.5f, __fmul_rn(xy, 0.5f));
    const float sx = __fdiv_rn(__fsub_rn(c1.x, c2.x), p.spatial_smooth_sxy);
    const float sy = __fdiv_rn(__fsub_rn(c1.y, c2.y), p.spatial_smooth_sxy);
    const float smooth = -__fmaf_rn(sx, sx, __fmul_rn(sy, sy));
    const float e_smooth = gexpf::expf(__fmul_rn(smooth, 0.5f));
    return __fmaf_rn(p.spatial_w, gexpf::expf(exponent), __fmul_rn(e_smooth, p.spatial_smooth_w));
}

// SimpleCRFFrame::calc_temporal_pairwise_energy(node, other) for two different frames (simple-crf.hpp:135-147)
__device__ __forceinline__ float crf_temporal_energy(const fslic_cluster& c1, const fslic_cluster& c2, const CrfParams& p) {
    const float dr = __fdiv_rn(__fsub_rn(c1.r, c2.r), p.temporal_srgb);
    const float dg = __fdiv_rn(__fsub_rn(c1.g, c2.g), p.temporal_srgb);
    const float db = __fdiv_rn(__fsub_rn(c1.b, c2.b), p.temporal_srgb);
    const float rgb = -crf_sq_sum3(dg, dr, db);
    return __fmul_rn(gexpf::expf(__fmul_rn(rgb, 0.5f)), p.temporal_w);
}

// sqrtf((float)m_other / m_i) with m_i = max((int)num_members, 1) (simple-crf.cpp:76-79,87): the numerator converts the
// uint32 field, the denominator the clamped int.
__device__ __forceinline__ float crf_member_ratio(uint32_t m_other, float m_i) {
    return __fsqrt_rn(__fdiv_rn((float)m_other, m_i));
}
__device__ __forceinline__ float crf_own_members(uint32_t m) {
    const int mi = (int)m;
    return (float)(mi <= 0 ? 1 : mi);
}

// The kernels below run a set of independent time chains, one per CRF, in the same launches: blockIdx.y picks the
// chain, blockIdx.x covers that chain's frames, and threads past its range return.  Temporal links never leave a chain,
// so every chain computes what it would alone.  A chain is one CRF's frame table, its length, the ping-pong buffer its
// previous inference left q in, and its params.
struct CrfChain {
    const CrfFrameDev* frames;
    int T, cur;
    CrfParams p;
};

// Up to CRF_GROUP_MAX chains (or frames, for the per-frame kernels) per launch, passed by value as __grid_constant__
// so a launch uploads nothing and never waits on the host.  64 chains take 3 KB, inside the 4 KB classic
// kernel-parameter limit; larger groups take several launch sets.
#define CRF_GROUP_MAX 64
struct CrfChainSet {
    CrfChain ch[CRF_GROUP_MAX];
};
static_assert(sizeof(CrfChainSet) + 16 <= 4096, "chain set must fit the classic kernel-parameter space");

// Once per inference() call: everything that depends only on the clusters, the graph and the params.  One thread per
// (frame, node); bound by the clusters' gather, a few µs at the sizes the CRF is used at.
__global__ void k_crf_pairwise(const __grid_constant__ CrfChainSet set, int N) {
    const CrfChain& ch = set.ch[blockIdx.y];
    const CrfFrameDev* __restrict__ frames = ch.frames;
    const int T = ch.T;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)T * N) return;
    const int t = (int)(gid / N), i = (int)(gid % N);
    const CrfFrameDev f = frames[t];
    const fslic_cluster ci = f.clusters[i];
    const float mi = crf_own_members(ci.num_members);
    for (int k = f.offsets[i]; k < f.offsets[i + 1]; k++) {
        const int j = f.nbr[k];
        const fslic_cluster cj = f.clusters[j];
        f.e_sp[k] = j == i ? 0.0f : crf_spatial_energy(cj, ci, ch.p);  // calc_spatial_pairwise_energy(neighbor, i)
        f.r_sp[k] = crf_member_ratio(cj.num_members, mi);
    }
    if (t > 0) {
        const fslic_cluster co = frames[t - 1].clusters[i];
        f.tmp[i] = crf_temporal_energy(ci, co, ch.p);
        f.tmp[N + i] = crf_member_ratio(co.num_members, mi);
    }
    if (t < T - 1) {
        const fslic_cluster co = frames[t + 1].clusters[i];
        f.tmp[2 * N + i] = crf_temporal_energy(ci, co, ch.p);
        f.tmp[3 * N + i] = crf_member_ratio(co.num_members, mi);
    }
}

// One infer_once() (simple-crf.cpp:62-151) in two launches: new q of every frame from the old q of all frames
// (Jacobi), into the other ping-pong buffer.  Step `it` of an inference passes flip = it & 1: each chain reads
// q[cur ^ flip] and writes q[cur ^ flip ^ 1].
// k_crf_msg: one thread per (frame, class, node) sums the messages in list order, then t-1, then t+1.  Bound by the
// latency of its dependent q gathers (deg + 2 per thread).
__global__ void k_crf_msg(const __grid_constant__ CrfChainSet set, int N, int C, int flip) {
    const CrfChain& ch = set.ch[blockIdx.y];
    const CrfFrameDev* __restrict__ frames = ch.frames;
    const int T = ch.T, cur = ch.cur ^ flip;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long CN = (long long)C * N;
    if (gid >= (long long)T * CN) return;
    const int t = (int)(gid / CN);
    const long long ci = gid % CN;  // c * N + i
    const int i = (int)(ci % N);
    const CrfFrameDev f = frames[t];
    const float* qc = f.q[cur] + (ci - i);
    float m = 0.0f;
    for (int k = f.offsets[i], k1 = f.offsets[i + 1]; k < k1; k++)
        m = __fmaf_rn(__fmul_rn(f.e_sp[k], qc[f.nbr[k]]), f.r_sp[k], m);
    if (t > 0) m = __fmaf_rn(__fmul_rn(f.tmp[i], frames[t - 1].q[cur][ci]), f.tmp[N + i], m);
    if (t < T - 1) m = __fmaf_rn(__fmul_rn(f.tmp[2 * N + i], frames[t + 1].q[cur][ci]), f.tmp[3 * N + i], m);
    f.msg[ci] = m;
}

// k_crf_compat: one thread per (frame, node) does the O(C^2) compatibility sums in class order (not "total minus
// own", which rounds differently), the C expf and the normalisation.  Compute bound on the C^2 chain per thread.
__global__ void k_crf_compat(const __grid_constant__ CrfChainSet set, int N, int C, int flip) {
    const CrfChain& ch = set.ch[blockIdx.y];
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)ch.T * N) return;
    const int t = (int)(gid / N), i = (int)(gid % N);
    const CrfFrameDev f = ch.frames[t];
    float* qo = f.q[ch.cur ^ flip ^ 1];
    float s = 0.0f;
    for (int c = 0; c < C; c++) {
        float acc = 0.0f;
        for (int o = 0; o < C; o++) {
            if (o == c) continue;  // Potts model
            acc = __fmaf_rn(1.0f, f.msg[(size_t)o * N + i], acc);  // compat_by_class[o] == 1
        }
        const float e = gexpf::expf(-__fadd_rn(f.unary[(size_t)c * N + i], acc));
        qo[(size_t)c * N + i] = e;
        s = __fadd_rn(s, e);
    }
    s = (double)s < 1e-5 ? 1e-5f : s;
    for (int c = 0; c < C; c++) qo[(size_t)c * N + i] = __fdiv_rn(qo[(size_t)c * N + i], s);
}

// The unaries and current q buffer of up to CRF_GROUP_MAX frames, blockIdx.y = frame, for the per-frame kernels.
struct CrfFrameQ {
    float* unary;
    float* q;
};
struct CrfFrameQSet {
    CrfFrameQ f[CRF_GROUP_MAX];
};

// reset_inferred (simple-crf.cpp:57-59): q = expf(-unary) of frame blockIdx.y, n = C * N values each
__global__ void __launch_bounds__(256) k_crf_reset(const __grid_constant__ CrfFrameQSet set, long long n) {
    const CrfFrameQ& f = set.f[blockIdx.y];
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
        f.q[k] = gexpf::expf(-f.unary[k]);
}

// get_inferred into a packed buffer: out[y][k] = q of frame y
__global__ void __launch_bounds__(256) k_crf_get_q(const __grid_constant__ CrfFrameQSet set, float* __restrict__ out,
                                                   long long n) {
    const float* __restrict__ q = set.f[blockIdx.y].q;
    out += (long long)blockIdx.y * n;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x)
        out[k] = q[k];
}

// The two pairwise-energy queries of the Python frame object (csimple_crf.pyx:209-227), one value each.
__global__ void k_crf_energy(const fslic_cluster a, const fslic_cluster b, int spatial, CrfParams p, float* out) {
    *out = spatial ? crf_spatial_energy(a, b, p) : crf_temporal_energy(a, b, p);
}

__global__ void k_expf_debug(uint32_t first, long long n, float* out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = gexpf::expf(__uint_as_float(first + (uint32_t)i));
}
