// fast_slic_b200/csrc/message_passing.cuh -- message passing over superpixel graphs (DESIGN.md section 4.21): the
// gather of node rows to graph entries, the softmax over each node's entries, and the sum / mean / max aggregation of
// (weighted) neighbour rows, with the exact backward of each.  No counterpart in the reference.  Every float operation is
// one separately rounded IEEE operation (no contraction) in the order the contract gives, and no float atomics, so a
// numpy restatement reproduces every bit:
//   graph    indptr int64 [N+1] and targets int64 [E] (edge_index[1]); the row of entry e is the node n with
//            indptr[n] <= e < indptr[n+1], its target t = targets[e].  An entry whose target is outside [0, N) is no
//            edge: it takes part in no sum, maximum or softmax and receives no gradient.  Row bounds are clamped into
//            [0, E], so any indptr keeps every read in bounds.
//   rows     a row sum adds its valid entries' terms in increasing e from +0.0, one rounded add each
//   columns  a transposed sum over node t's in-entries (the valid entries with target t) adds them in increasing e from
//            +0.0; they come from one stable radix sort of the entries keyed by target (invalid targets keyed N)
//   heads    a weight [E,H] gives head h the channels [h*D, (h+1)*D), D = C / H
// Layouts: node maps [N,C], entry maps [E,C], weights and scores [E,H], arg-max tables int32 [N,C].
#pragma once
#include "common.cuh"
#include "glibc_expf.cuh"

#define MP_CPL 4  // channels per lane of one pass of the warp-per-node sums (128 channels per pass)

// Grid-stride loops over items (threads) and over warps
#define MP_FOR(n) for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < (n); t += (long)gridDim.x * blockDim.x)
#define MP_FOR_WARP(w, n)                                                                          \
    for (long w = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < (n); w += ((long)gridDim.x * blockDim.x) >> 5)

__device__ __forceinline__ bool mp_valid(long long t, long n) { return (unsigned long long)t < (unsigned long long)n; }

// Row n's entries [*s, *e), both clamped into [0, E]
__device__ __forceinline__ void mp_row(const long long* __restrict__ indptr, long n, long E, long* s, long* e) {
    long long a = __ldg(indptr + n), b = __ldg(indptr + n + 1);
    a = a < 0 ? 0 : (a > E ? E : a);
    b = b < a ? a : (b > E ? E : b);
    *s = (long)a;
    *e = (long)b;
}

// The total order of non-NaN floats, -0.0 < +0.0, as signed ints (boundary.cuh's)
__device__ __forceinline__ int mp_okey(float v) {
    const int i = __float_as_int(v);
    return i ^ ((i >> 31) & 0x7fffffff);
}

// Whether v replaces the current maximum `best` (which exists): the first NaN stays, a NaN replaces a number, otherwise
// only a strictly larger value in the total order (so the first attaining entry is the arg-max)
__device__ __forceinline__ bool mp_beats(float v, float best) {
    return !isnan(best) && (isnan(v) || mp_okey(v) > mp_okey(best));
}

// ---- edge_gather forward

// "target": out[e, c] = x[t_e, c], +0.0 for an invalid target.  One thread per (entry, channel).
__global__ void __launch_bounds__(256) k_mp_gather_target(const long long* __restrict__ tgt, const float* __restrict__ x,
                                                          long N, long E, int C, float* __restrict__ out) {
    MP_FOR(E * C) {
        const long e = t / C;
        const int c = (int)(t - e * C);
        const long long tt = __ldg(tgt + e);
        out[t] = mp_valid(tt, N) ? __ldg(x + tt * C + c) : 0.f;
    }
}

// "source": out[e, c] = x[row(e), c], +0.0 for an invalid target.  One warp per node, lanes over channels.
__global__ void __launch_bounds__(256) k_mp_gather_source(const long long* __restrict__ indptr,
                                                          const long long* __restrict__ tgt, const float* __restrict__ x,
                                                          long N, long E, int C, float* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    MP_FOR_WARP(n, N) {
        long s, e;
        mp_row(indptr, n, E, &s, &e);
        for (int c = lane; c < C; c += 32) {
            const float v = __ldg(x + n * C + c);
            for (long i = s; i < e; i++) out[i * C + c] = mp_valid(__ldg(tgt + i), N) ? v : 0.f;
        }
    }
}

// ---- the warp-per-node sums: one warp per node, lanes over channels (MP_CPL per lane per pass), the node's entries
// fetched 32 at a time by the lanes and broadcast with shuffles, so every read of a source row is one coalesced load.

enum MpSum {
    MP_AGG = 0,      // row n, term w[e,h] * x[t_e, c] (forward of aggregate sum / mean)
    MP_AGG_MAX = 1,  // row n, the maximum of the same terms and its entry (forward of aggregate max)
    MP_ROWS = 2,     // row n, term x[e, c] (edge_gather "source" backward: x = grad_out [E,C])
    MP_COLS = 3,     // in-entries of n, term x[e, c] (edge_gather "target" backward: x = grad_out [E,C])
    MP_COLS_AGG = 4, // in-entries of n, term w[e,h] * x[row(e), c], and with amax only where amax[row(e), c] == e
                     // (aggregate backward to x: x = grad_out or grad_out / deg [N,C])
};

// Row mode (MP_AGG, MP_AGG_MAX, MP_ROWS): the node's entries are [indptr[n], indptr[n+1]) with a valid target.
// Column mode (MP_COLS, MP_COLS_AGG): sorted positions [tptr[n], tptr[n+1]) of the transposed order; sval gives the
// entry, rowof the entry's row.  w [E,H] or null; D = C / H.  out [N,C]; MP_AGG with deg: mean (deg [N] receives the
// valid entry count, out the sum / (float)count, +0.0 for none); MP_AGG_MAX: amax [N,C] the arg-max entry (-1 for none)
// and out its term (+0.0 for none).
template <int MODE>
__global__ void __launch_bounds__(256) k_mp_sum(const long long* __restrict__ indptr, const long long* __restrict__ tgt,
                                                const uint32_t* __restrict__ tptr, const uint32_t* __restrict__ sval,
                                                const uint32_t* __restrict__ rowof, const float* __restrict__ x,
                                                const float* __restrict__ w, const int32_t* __restrict__ amax_in,
                                                long N, long E, int C, int H, float* __restrict__ out,
                                                int32_t* __restrict__ deg, int32_t* __restrict__ amax_out) {
    constexpr bool COLS = MODE == MP_COLS || MODE == MP_COLS_AGG;
    const int lane = threadIdx.x & 31;
    const int D = C / H;
    MP_FOR_WARP(n, N) {
        long s, e;
        if (COLS) {
            s = (long)__ldg(tptr + n);
            e = (long)__ldg(tptr + n + 1);
        } else {
            mp_row(indptr, n, E, &s, &e);
        }
        int count = 0;
        for (int c0 = 0; c0 < C; c0 += 32 * MP_CPL) {
            float acc[MP_CPL];
            int arg[MP_CPL];
#pragma unroll
            for (int u = 0; u < MP_CPL; u++) {
                acc[u] = 0.f;
                arg[u] = -1;
            }
            count = 0;
            for (long i0 = s; i0 < e; i0 += 32) {
                // lane j fetches entry i0 + j: its index, its source row (-1: no edge)
                long my_e = -1, my_src = -1;
                if (i0 + lane < e) {
                    const long i = i0 + lane;
                    if (COLS) {
                        my_e = (long)__ldg(sval + i);
                        my_src = MODE == MP_COLS ? my_e : (long)__ldg(rowof + my_e);
                    } else {
                        my_e = i;
                        const long long tt = __ldg(tgt + i);
                        my_src = mp_valid(tt, N) ? (MODE == MP_ROWS ? i : (long)tt) : -1;
                    }
                }
                const int m = (int)min(32L, e - i0);
                for (int j = 0; j < m; j++) {
                    const long src = __shfl_sync(FSLIC_FULL, my_src, j);
                    if (src < 0) continue;  // the whole warp skips an entry that is no edge
                    const long ent = __shfl_sync(FSLIC_FULL, my_e, j);
                    count++;
#pragma unroll
                    for (int u = 0; u < MP_CPL; u++) {
                        const int c = c0 + lane + 32 * u;
                        if (c < C) {
                            if (MODE == MP_COLS_AGG && amax_in && __ldg(amax_in + src * C + c) != (int32_t)ent) continue;
                            float v = __ldg(x + src * C + c);
                            if (w && (MODE == MP_AGG || MODE == MP_AGG_MAX || MODE == MP_COLS_AGG))
                                v = __fmul_rn(__ldg(w + ent * H + c / D), v);
                            if (MODE == MP_AGG_MAX) {
                                if (arg[u] < 0 || mp_beats(v, acc[u])) {
                                    acc[u] = v;
                                    arg[u] = (int)ent;
                                }
                            } else {
                                acc[u] = __fadd_rn(acc[u], v);
                            }
                        }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < MP_CPL; u++) {
                const int c = c0 + lane + 32 * u;
                if (c < C) {
                    float r = acc[u];
                    if (MODE == MP_AGG && deg) r = count ? __fdiv_rn(r, __int2float_rn(count)) : 0.f;
                    out[n * C + c] = r;
                    if (MODE == MP_AGG_MAX) amax_out[n * C + c] = arg[u];
                }
            }
        }
        if (MODE == MP_AGG && deg && lane == 0) {
            // C >= 1, so the count of the last pass is the row's
            deg[n] = count;
        }
    }
}

// ---- aggregate backward to the weights: one warp per entry.  grad_w[e,h] = the sum over head h's channels c of
// g[row(e), c] * x[t_e, c] (with amax, only the channels where amax[row(e), c] == e), in pool's lane order: channel j of
// the head goes to lane j mod 32, each lane adds left to right from +0.0, then the butterfly o = 16, 8, 4, 2, 1.  A head
// of D <= 16 channels is summed in a segment of P = the power of two >= D lanes with the butterfly o = P/2 .. 1 only,
// 32 / P heads per pass: each lane holds at most one term, lanes past D would hold +0.0, and a lane sum is never -0.0,
// so the full butterfly's steps o >= P add +0.0 to lane 0's value and change no bit.  +0.0 for an invalid target.
__global__ void __launch_bounds__(256) k_mp_grad_weight(const long long* __restrict__ tgt,
                                                        const uint32_t* __restrict__ rowof, const float* __restrict__ g,
                                                        const float* __restrict__ x, const int32_t* __restrict__ amax,
                                                        long N, long E, int C, int H, float* __restrict__ gw) {
    const int lane = threadIdx.x & 31;
    const int D = C / H;
    int P = 32;
    if (D <= 16) {
        P = 1;
        while (P < D) P <<= 1;
    }
    const int G = 32 / P, j = lane & (P - 1), hl = lane / P;
    MP_FOR_WARP(e, E) {
        const long long tt = __ldg(tgt + e);
        const bool ok = mp_valid(tt, N);
        const long r = ok ? (long)__ldg(rowof + e) : 0;
        for (int h0 = 0; h0 < H; h0 += G) {
            const int h = h0 + hl;
            float acc = 0.f;
            if (ok && h < H) {
                for (int c = j; c < D; c += P) {
                    const int cc = h * D + c;
                    if (amax && __ldg(amax + r * C + cc) != (int32_t)e) continue;
                    acc = __fadd_rn(acc, __fmul_rn(__ldg(g + r * C + cc), __ldg(x + tt * C + cc)));
                }
            }
            for (int o = P >> 1; o; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(FSLIC_FULL, acc, o));
            if (j == 0 && h < H) gw[e * H + h] = acc;
        }
    }
}

// gs[n, c] = g[n, c] / (float)deg[n] (one rounded division), +0.0 where deg is 0: the gradient of the mean, rounded once
__global__ void __launch_bounds__(256) k_mp_scale(const float* __restrict__ g, const int32_t* __restrict__ deg, long N,
                                                  int C, float* __restrict__ gs) {
    MP_FOR(N * C) {
        const int d = __ldg(deg + t / C);
        gs[t] = d ? __fdiv_rn(__ldg(g + t), __int2float_rn(d)) : 0.f;
    }
}

// ---- edge_softmax: one thread per (node, head), heads fastest.  Over the row's valid entries in increasing e:
// m = the maximum (a NaN wins, else the total order with -0.0 < +0.0), y_e = expf(s_e - m) (glibc's), Z = sum y_e from
// +0.0, out_e = y_e / Z; out_e = +0.0 for an entry that is no edge.
__global__ void __launch_bounds__(256) k_mp_softmax(const long long* __restrict__ indptr,
                                                    const long long* __restrict__ tgt, const float* __restrict__ sc,
                                                    long N, long E, int H, float* __restrict__ out) {
    MP_FOR(N * H) {
        const long n = t / H;
        const int h = (int)(t - n * H);
        long s, e;
        mp_row(indptr, n, E, &s, &e);
        float m = 0.f;
        bool any = false;
        for (long i = s; i < e; i++) {
            if (!mp_valid(__ldg(tgt + i), N)) continue;
            const float v = __ldg(sc + i * H + h);
            if (!any || mp_beats(v, m)) m = v;
            any = true;
        }
        float z = 0.f;
        for (long i = s; i < e; i++) {
            float y = 0.f;
            if (mp_valid(__ldg(tgt + i), N)) {
                y = gexpf::expf(__fsub_rn(__ldg(sc + i * H + h), m));
                z = __fadd_rn(z, y);
            }
            out[i * H + h] = y;
        }
        for (long i = s; i < e; i++)
            if (mp_valid(__ldg(tgt + i), N)) out[i * H + h] = __fdiv_rn(out[i * H + h], z);
    }
}

// The softmax backward, the same threads: dot = sum over the valid entries of out_e * g_e from +0.0, then
// grad_e = out_e * (g_e - dot); +0.0 for an entry that is no edge.
__global__ void __launch_bounds__(256) k_mp_softmax_bwd(const long long* __restrict__ indptr,
                                                        const long long* __restrict__ tgt, const float* __restrict__ o,
                                                        const float* __restrict__ g, long N, long E, int H,
                                                        float* __restrict__ gs) {
    MP_FOR(N * H) {
        const long n = t / H;
        const int h = (int)(t - n * H);
        long s, e;
        mp_row(indptr, n, E, &s, &e);
        float dot = 0.f;
        for (long i = s; i < e; i++)
            if (mp_valid(__ldg(tgt + i), N)) dot = __fadd_rn(dot, __fmul_rn(__ldg(o + i * H + h), __ldg(g + i * H + h)));
        for (long i = s; i < e; i++) {
            const long k = i * H + h;
            gs[k] = mp_valid(__ldg(tgt + i), N) ? __fmul_rn(__ldg(o + k), __fsub_rn(__ldg(g + k), dot)) : 0.f;
        }
    }
}

// ---- the transposed order

// key[e] = t_e (N for an invalid target), val[e] = e; rowof[e] = the row of e (the last n < N with indptr[n] <= e, 0
// if there is none), by binary search over indptr
__global__ void __launch_bounds__(256) k_mp_keys(const long long* __restrict__ indptr, const long long* __restrict__ tgt,
                                                 long N, long E, uint32_t* __restrict__ key, uint32_t* __restrict__ val,
                                                 uint32_t* __restrict__ rowof) {
    MP_FOR(E) {
        const long long tt = __ldg(tgt + t);
        key[t] = mp_valid(tt, N) ? (uint32_t)tt : (uint32_t)N;
        val[t] = (uint32_t)t;
        long lo = 0, hi = N - 1;  // the answer is in [lo, hi]
        while (lo < hi) {
            const long mid = (lo + hi + 1) >> 1;
            if (__ldg(indptr + mid) <= t)
                lo = mid;
            else
                hi = mid - 1;
        }
        rowof[t] = (uint32_t)lo;
    }
}

// tptr[n] = the first sorted position whose key is >= n, for n in [0, N]: node n's in-entries are [tptr[n], tptr[n+1])
__global__ void __launch_bounds__(256) k_mp_bounds(const uint32_t* __restrict__ skey, long N, long E,
                                                   uint32_t* __restrict__ tptr) {
    MP_FOR(N + 1) {
        long lo = 0, hi = E;
        while (lo < hi) {
            const long mid = (lo + hi) >> 1;
            if (__ldg(skey + mid) < (uint32_t)t)
                lo = mid + 1;
            else
                hi = mid;
        }
        tptr[t] = (uint32_t)lo;
    }
}
