// fast_slic_b200/csrc/prepare.cuh -- the per-image bookkeeping between two assign passes.
//
//   1. finalise the previous update: integer round-divide of the accumulated sums (context.cpp:356-374, round_int
//      fast-slic-common.h:63-65), or the float quotients of ContextRealDistNoQ (context.cpp:375-381);
//   2. first pass only: re-seed the cluster colour from the quad image (context.cpp:128-135);
//   3. clamp centres into the image (context.cpp:209-212), truncate to int16 (context.cpp:266-267), derive the
//      visiting-order key, make the 16-byte CInfo record;
//   4. counting-sort the CInfo records into a uniform cell grid of pitch G >= S, so a tile can collect the clusters whose
//      window may touch it from a few contiguous ranges of the sorted array.
//
// Each step is written once, as a device function; the kernels differ in how they spread the clusters over threads and
// where the records wait for the sort:
//   k_prepare3       K <= 4096, one CTA per image, records in registers;
//   prepare_in_tail  k_prepare3's work in the tail of the fused k_assign5 update (1-2 images), records in shared memory;
//   k_prepare        one CTA per image, records through a global scratch; the only one with the `preemptive` rules;
//   k_prepare2       one thread per cluster over several CTAs per image, the last CTA of an image sorts.
// Loading and zeroing the accumulated sums stay with each kernel: they use different loads.
#pragma once
#include "cellgrid.cuh"
#include "common.cuh"

struct PrepParams {
    int H, W, K, S, T;
    int G, cellW, cellH, ncell;
    int first;     // 1: re-seed colours, no update to finalise
    int finalize;  // 1: fold `acc` into the clusters
    int last;      // 1: after the final update: set is_active / is_updatable like the reference leaves them
    int noq;       // 1: ContextRealDistNoQ -- centroids are float quotients, not rounded integers (context.cpp:375-381)
    // k_prepare only: the `preemptive` option (preempt.cuh; preemptive.h:113-141, context.cpp:360)
    int preempt;       // 1: only updatable clusters take their new centre; the movement test counts is_updatable down
    float l1_thres;    // max(roundf(2 S thres), 1)
    int* nactive;      // [B] number of active clusters (first pass: K = everything active)
};

// The geometry of a context with every pass flag off; the caller sets the flags of its pass.  T = 2S + 32 is the
// period of the visiting order (context.cpp:214-242).
__host__ __device__ __forceinline__ PrepParams prep_params(int H, int W, int K, int S, int G, int cellW, int cellH,
                                                           int ncell) {
    PrepParams pp = {H, W, K, S, 2 * S + 32, G, cellW, cellH, ncell};
    return pp;
}

// Step 1 for one cluster, from its packed sums: w0 = n | sum_y << 32, w1 = sum_x | sum_L << 32, w2 = sum_a | sum_b << 32.
// PREEMPT compiles the rules of the `preemptive` option (for k_prepare), which apply when `preempt` is set: a cluster
// that is not updatable keeps its centre and its member count (context.cpp:360); an updatable one counts is_updatable
// down when it moved less than l1_thres (L1) from the centre the assign used (PreemptiveGrid::set_new_clusters, first
// loop, preemptive.h:132-141).
template <bool PREEMPT = false>
__device__ __forceinline__ void finalize_cluster(fslic_cluster& c, unsigned long long w0, unsigned long long w1,
                                                 unsigned long long w2, bool noq, bool preempt = false,
                                                 float l1_thres = 0.f) {
    const float old_y = c.y, old_x = c.x;  // set_old_clusters (context.cpp:303): the centres the assign used
    const bool frozen = PREEMPT && preempt && !c.is_updatable;
    const uint32_t n = frozen ? 0u : (uint32_t)w0;
    if (!frozen) c.num_members = n;  // written even when n == 0 (context.cpp:360-362)
    if (n > 0 && noq) {  // (float)sum / n: int -> float conversion, IEEE division
        const float fn = __int2float_rn((int32_t)n);
        c.y = __fdiv_rn(__int2float_rn((int32_t)(w0 >> 32)), fn);
        c.x = __fdiv_rn(__int2float_rn((int32_t)(uint32_t)w1), fn);
        c.r = __fdiv_rn(__int2float_rn((int32_t)(w1 >> 32)), fn);
        c.g = __fdiv_rn(__int2float_rn((int32_t)(uint32_t)w2), fn);
        c.b = __fdiv_rn(__int2float_rn((int32_t)(w2 >> 32)), fn);
    } else if (n > 0) {
        const int32_t in = (int32_t)n, half = in / 2;
        c.y = (float)(((int32_t)(w0 >> 32) + half) / in);
        c.x = (float)(((int32_t)(uint32_t)w1 + half) / in);
        c.r = (float)(((int32_t)(w1 >> 32) + half) / in);
        c.g = (float)(((int32_t)(uint32_t)w2 + half) / in);
        c.b = (float)(((int32_t)(w2 >> 32) + half) / in);
    }
    if (PREEMPT && preempt && c.is_updatable) {
        const float l1 = __fadd_rn(fabsf(__fsub_rn(old_x, c.x)), fabsf(__fsub_rn(old_y, c.y)));
        c.is_updatable = l1 < l1_thres ? (uint8_t)(c.is_updatable - 1) : (uint8_t)2;
    }
}

// Step 2: the colour of the quad pixel under the centre, clamped into the image and truncated.  qd: the image's pixels.
__device__ __forceinline__ void reseed_colour(fslic_cluster& c, const uint32_t* __restrict__ qd, int H, int W) {
    const int y = min(max((int)c.y, 0), H - 1), x = min(max((int)c.x, 0), W - 1);
    const uint32_t q = qd[(size_t)y * W + x];
    c.r = (float)(q & 0xff);
    c.g = (float)((q >> 8) & 0xff);
    c.b = (float)((q >> 16) & 0xff);
}

// Step 3 on cluster k: the safeguard clamp, stored back like the reference does, its number and its flags.  Every
// cluster is active and updatable (PreemptiveGrid::initialize, preemptive.h:59-67) unless PREEMPT (k_prepare) and the
// pass has `preempt` set: then only the first pass resets both, the pass after the final update sets is_active
// (PreemptiveGrid::finalize, preemptive.h:69-74) and leaves is_updatable where it got to, and in between k_preempt_mark
// decides is_active from the new centres.
template <bool PREEMPT = false>
__device__ __forceinline__ void clamp_cluster(fslic_cluster& c, int k, const PrepParams& pp) {
    c.x = fminf(fmaxf(c.x, 0.f), (float)(pp.W - 1));
    c.y = fminf(fmaxf(c.y, 0.f), (float)(pp.H - 1));
    c.number = (uint16_t)k;
    if (!PREEMPT || !pp.preempt || pp.first) {
        c.is_active = 1;
        c.is_updatable = 2;
    } else if (pp.last) {
        c.is_active = 1;
    }
}

// Step 3: the record of cluster k (common.cuh) with its visiting-order key, phase = 2 ((cy/T) & 1) + ((cx/T) & 1).
__device__ __forceinline__ CInfo make_record(const fslic_cluster& c, int k, int T) {
    const int cy = (int16_t)c.y, cx = (int16_t)c.x;
    const int cr = (int16_t)c.r, cg = (int16_t)c.g, cb = (int16_t)c.b;
    const int phase = 2 * ((cy / T) & 1) + ((cx / T) & 1);
    CInfo r;
    r.cyx = (cy & 0xffff) | (cx << 16);
    r.color = (uint32_t)(cr & 0xff) | ((uint32_t)(cg & 0xff) << 8) | ((uint32_t)(cb & 0xff) << 16);
    r.sortkey = ((uint32_t)phase << 16) | (uint32_t)k;
    r.pad = 0;
    return r;
}

// Step 4: the cell of the grid that holds the centre of a record (its cyx word).
__device__ __forceinline__ int record_cell(int32_t cyx, const PrepParams& pp) {
    const int cy = (int16_t)(cyx & 0xffff), cx = cyx >> 16;
    return (cy / pp.G) * pp.cellW + (cx / pp.G);
}

// For a grid whose last CTA to arrive finishes the work of all of them: true in every thread of the CTA that takes the
// last of `count` tickets.  The fence before the ticket makes this thread's global writes visible before its CTA's
// ticket is taken; the one after it orders the last CTA's reads after them.  The counter is left at zero for the next
// launch.
__device__ __forceinline__ bool last_block_to_arrive(unsigned int* ticket, unsigned int count) {
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == count - 1u ? 1 : 0;
    __syncthreads();
    if (!s_last) return false;
    if (threadIdx.x == 0) *ticket = 0u;
    __threadfence();
    return true;
}

// ---------------------------------------------------------------------------------------------
// k_prepare: one CTA per image, two phases through global memory: the records by cluster index into `cinfo_tmp` and
// the cell histogram, then, after the scan, the records into their cells.  It handles any K, and it alone carries the
// `preemptive` bookkeeping (PrepParams.preempt).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_prepare(PrepParams pp, fslic_cluster* __restrict__ clusters,
                                                   unsigned long long* __restrict__ acc,
                                                   const uint32_t* __restrict__ quad, CInfo* __restrict__ cinfo,
                                                   int* __restrict__ cell_start,
                                                   CInfo* __restrict__ cinfo_tmp) {
    extern __shared__ int s_cnt[];  // ncell + 1 counters
    __shared__ int s_warp[32];
    const int b = blockIdx.x;
    const int tid = threadIdx.x, nt = blockDim.x;
    fslic_cluster* cl = clusters + (size_t)b * pp.K;
    unsigned long long* ac = acc + (size_t)b * pp.K * 4;
    const uint32_t* qd = quad + (size_t)b * pp.H * pp.W;
    CInfo* ci = cinfo_tmp + (size_t)b * pp.K;          // by cluster index (scratch)
    CInfo* ci_sorted = cinfo + (size_t)b * pp.K;       // by cell, what the assign kernels read
    int* cs = cell_start + (size_t)b * (pp.ncell + 1);

    for (int c = tid; c <= pp.ncell; c += nt) s_cnt[c] = 0;
    if (pp.preempt && pp.first && tid == 0) pp.nactive[b] = pp.K;  // b_all_active = true (preemptive.h:63)
    __syncthreads();

    for (int k = tid; k < pp.K; k += nt) {
        fslic_cluster c = cl[k];
        if (pp.finalize) {
            const unsigned long long w0 = ac[k * 4 + 0], w1 = ac[k * 4 + 1], w2 = ac[k * 4 + 2];
            ac[k * 4 + 0] = 0; ac[k * 4 + 1] = 0; ac[k * 4 + 2] = 0;
            finalize_cluster<true>(c, w0, w1, w2, pp.noq, pp.preempt, pp.l1_thres);
        }
        if (pp.first) reseed_colour(c, qd, pp.H, pp.W);
        clamp_cluster<true>(c, k, pp);
        cl[k] = c;
        const CInfo r = make_record(c, k, pp.T);
        ci[k] = r;
        atomicAdd(&s_cnt[record_cell(r.cyx, pp)], 1);
    }
    scan_cells(s_cnt, s_warp, cs, pp.ncell + 1, tid, nt);
    for (int k = tid; k < pp.K; k += nt) {
        const CInfo r = ci[k];
        const int slot = atomicAdd(&s_cnt[record_cell(r.cyx, pp)], 1);
        ci_sorted[slot] = r;  // order inside a cell is arbitrary: consumers rank by sortkey
    }
}

// ---------------------------------------------------------------------------------------------
// k_prepare3: k_prepare for K <= 4096 with the latency taken out.  k_prepare goes to global memory four times in a row
// per cluster (load record, store the unsorted CInfo, load it back after the scan, store it sorted) and handles its
// clusters one after the other.  Here every thread loads all its clusters up front, keeps the CInfo records in
// registers, and the shared-memory atomicAdd that counts a cell also hands out the record's rank inside the cell -- so
// after ONE scan the records go straight to their sorted slots: one global load round trip, one store, four barriers.
// Same results (order inside a cell is arbitrary for both; consumers rank by sort key).
// ---------------------------------------------------------------------------------------------
#define PREP3_PER 4  // clusters per thread at most (K <= 4096 with 1024 threads)
__global__ void __launch_bounds__(1024) k_prepare3(PrepParams pp, fslic_cluster* __restrict__ clusters,
                                                   unsigned long long* __restrict__ acc, const uint32_t* __restrict__ quad,
                                                   CInfo* __restrict__ cinfo, int* __restrict__ cell_start) {
    extern __shared__ int s_cnt[];  // ncell + 1 counters
    __shared__ int s_warp[32];
    const int b = blockIdx.x;
    const int tid = threadIdx.x, nt = blockDim.x;
    fslic_cluster* cl = clusters + (size_t)b * pp.K;
    unsigned long long* ac = acc + (size_t)b * pp.K * 4;
    const uint32_t* qd = quad + (size_t)b * pp.H * pp.W;
    CInfo* ci_sorted = cinfo + (size_t)b * pp.K;
    int* cs = cell_start + (size_t)b * (pp.ncell + 1);
    const int ncnt = pp.ncell + 1;
    for (int c = tid; c < ncnt; c += nt) s_cnt[c] = 0;

    // all global loads of this thread's clusters in flight together
    uint4 ca[PREP3_PER], cb[PREP3_PER];
    ulonglong2 a01[PREP3_PER];
    unsigned long long a2[PREP3_PER];
#pragma unroll
    for (int u = 0; u < PREP3_PER; u++) {
        const int k = tid + u * nt;
        if (k < pp.K) {
            const uint4* p = reinterpret_cast<const uint4*>(cl + k);
            ca[u] = p[0];
            cb[u] = p[1];
            if (pp.finalize) {
                a01[u] = *reinterpret_cast<const ulonglong2*>(ac + (size_t)k * 4);
                a2[u] = ac[(size_t)k * 4 + 2];
            }
        }
    }
    __syncthreads();  // histogram zeroed
    CInfo rec[PREP3_PER];
    int cell[PREP3_PER], rank[PREP3_PER];
#pragma unroll
    for (int u = 0; u < PREP3_PER; u++) {
        const int k = tid + u * nt;
        cell[u] = -1;
        if (k < pp.K) {
            fslic_cluster c;
            memcpy(&c, &ca[u], 16);
            memcpy(reinterpret_cast<char*>(&c) + 16, &cb[u], 16);
            if (pp.finalize) {
                finalize_cluster(c, a01[u].x, a01[u].y, a2[u], pp.noq);
                *reinterpret_cast<ulonglong2*>(ac + (size_t)k * 4) = make_ulonglong2(0ull, 0ull);
                ac[(size_t)k * 4 + 2] = 0ull;
            }
            if (pp.first) reseed_colour(c, qd, pp.H, pp.W);
            clamp_cluster(c, k, pp);
            uint4 o0, o1;
            memcpy(&o0, &c, 16);
            memcpy(&o1, reinterpret_cast<char*>(&c) + 16, 16);
            uint4* p = reinterpret_cast<uint4*>(cl + k);
            p[0] = o0;
            p[1] = o1;
            rec[u] = make_record(c, k, pp.T);
            cell[u] = record_cell(rec[u].cyx, pp);
            rank[u] = atomicAdd(&s_cnt[cell[u]], 1);  // count the cell and take a slot inside it
        }
    }
    scan_cells(s_cnt, s_warp, cs, ncnt, tid, nt);
#pragma unroll
    for (int u = 0; u < PREP3_PER; u++)
        if (cell[u] >= 0) ci_sorted[s_cnt[cell[u]] + rank[u]] = rec[u];
}

// ---------------------------------------------------------------------------------------------
// prepare_in_tail: the finalize / record / counting-sort work of k_prepare3 (no colour re-seed) as a device function
// for the TAIL of an assign+update launch: the last CTA of k_assign5 to finish (ticket counter) calls it, so that a
// single image's ten passes do not pay a kernel boundary between "update" and "next assign" (the eleven k_prepare
// launches were a third of a single image's device time).  The caller's registers are capped at 64 per thread, so the
// records wait in shared memory instead of registers: `smem` needs prepare_tail_smem_bytes(K, ncell) bytes.  K <= 4096.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ size_t prepare_tail_smem_bytes(int K, int ncell) {
    return (size_t)((ncell + 1 + 3) & ~3) * 4 + 32 * 4 + (size_t)K * 16 + (size_t)K * 4;
}

__device__ __forceinline__ void prepare_in_tail(const PrepParams& pp, fslic_cluster* __restrict__ cl,
                                                unsigned long long* __restrict__ ac, CInfo* __restrict__ ci_sorted,
                                                int* __restrict__ cs, unsigned char* smem, int tid, int nt) {
    const int ncnt = pp.ncell + 1;
    int* s_cnt = reinterpret_cast<int*>(smem);
    int* s_warp = s_cnt + ((ncnt + 3) & ~3);
    CInfo* s_rec = reinterpret_cast<CInfo*>(s_warp + 32);
    int* s_slot = reinterpret_cast<int*>(s_rec + pp.K);  // cell << 12 | rank inside the cell
    for (int c = tid; c < ncnt; c += nt) s_cnt[c] = 0;
    __syncthreads();
    for (int k = tid; k < pp.K; k += nt) {
        uint4* gp = reinterpret_cast<uint4*>(cl + k);
        const uint4 g0 = gp[0], g1 = gp[1];
        fslic_cluster c;
        memcpy(&c, &g0, 16);
        memcpy(reinterpret_cast<char*>(&c) + 16, &g1, 16);
        // the sums were written by RED.64 from other SMs: read them through L2 (ld.global.cg)
        const uint4 a01 = __ldcg(reinterpret_cast<const uint4*>(ac + (size_t)k * 4));
        const uint2 a2 = __ldcg(reinterpret_cast<const uint2*>(ac + (size_t)k * 4 + 2));
        finalize_cluster(c, a01.x | (unsigned long long)a01.y << 32, a01.z | (unsigned long long)a01.w << 32,
                         a2.x | (unsigned long long)a2.y << 32, false);
        *reinterpret_cast<ulonglong2*>(ac + (size_t)k * 4) = make_ulonglong2(0ull, 0ull);
        ac[(size_t)k * 4 + 2] = 0ull;
        clamp_cluster(c, k, pp);
        uint4 o0, o1;
        memcpy(&o0, &c, 16);
        memcpy(&o1, reinterpret_cast<char*>(&c) + 16, 16);
        gp[0] = o0;
        gp[1] = o1;
        const CInfo r = make_record(c, k, pp.T);
        s_rec[k] = r;
        const int cell = record_cell(r.cyx, pp);
        s_slot[k] = (cell << 12) | atomicAdd(&s_cnt[cell], 1);
    }
    scan_cells(s_cnt, s_warp, cs, ncnt, tid, nt);
    for (int k = tid; k < pp.K; k += nt) {
        const int sl = s_slot[k];
        ci_sorted[s_cnt[sl >> 12] + (sl & 4095)] = s_rec[k];
    }
    __syncthreads();  // the shared buffers are reused by the next image
}

// ---------------------------------------------------------------------------------------------
// k_prepare2: the same bookkeeping spread over ceil(K / 256) CTAs per image.  k_prepare is one CTA per image and
// latency bound; here every cluster has its own thread (steps 1-3, the cell histogram through global atomics), and the
// LAST CTA of an image to finish (ticket counter) runs step 4 for the whole image: cell histogram -> shared memory,
// exclusive scan, scatter of the records.  The histogram and the ticket are left zeroed for the next launch.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_prepare2(PrepParams pp, fslic_cluster* __restrict__ clusters,
                                                  unsigned long long* __restrict__ acc, const uint32_t* __restrict__ quad,
                                                  CInfo* __restrict__ cinfo, int* __restrict__ cell_start,
                                                  CInfo* __restrict__ cinfo_tmp, int* __restrict__ cell_cnt,
                                                  unsigned int* __restrict__ tickets) {
    extern __shared__ int s_cnt[];  // last CTA only: ncell + 1 counters
    __shared__ int s_warp[8];
    const int b = blockIdx.y;
    const int tid = threadIdx.x, nt = blockDim.x;
    fslic_cluster* cl = clusters + (size_t)b * pp.K;
    unsigned long long* ac = acc + (size_t)b * pp.K * 4;
    const uint32_t* qd = quad + (size_t)b * pp.H * pp.W;
    CInfo* ci = cinfo_tmp + (size_t)b * pp.K;          // by cluster index (scratch)
    CInfo* ci_sorted = cinfo + (size_t)b * pp.K;       // by cell, what the assign kernels read
    int* cs = cell_start + (size_t)b * (pp.ncell + 1);
    int* gcnt = cell_cnt + (size_t)b * (pp.ncell + 1);

    const int k = blockIdx.x * nt + tid;
    if (k < pp.K) {
        fslic_cluster c = cl[k];
        if (pp.finalize) {
            const unsigned long long w0 = ac[k * 4 + 0], w1 = ac[k * 4 + 1], w2 = ac[k * 4 + 2];
            ac[k * 4 + 0] = 0; ac[k * 4 + 1] = 0; ac[k * 4 + 2] = 0;
            finalize_cluster(c, w0, w1, w2, pp.noq);
        }
        if (pp.first) reseed_colour(c, qd, pp.H, pp.W);
        clamp_cluster(c, k, pp);
        cl[k] = c;
        const CInfo r = make_record(c, k, pp.T);
        ci[k] = r;
        atomicAdd(&gcnt[record_cell(r.cyx, pp)], 1);
    }
    // the last CTA of this image to get here sorts the records into the cell grid
    if (!last_block_to_arrive(&tickets[b], gridDim.x)) return;
    const int ncnt = pp.ncell + 1;
    for (int c = tid; c < ncnt; c += nt) {
        s_cnt[c] = __ldcg(&gcnt[c]);
        gcnt[c] = 0;  // ready for the next launch
    }
    scan_cells(s_cnt, s_warp, cs, ncnt, tid, nt);
    for (int kk = tid; kk < pp.K; kk += nt) {
        const uint4 r = __ldcg(reinterpret_cast<const uint4*>(&ci[kk]));  // written by other CTAs: read through L2
        const int slot = atomicAdd(&s_cnt[record_cell((int32_t)r.x, pp)], 1);
        *reinterpret_cast<uint4*>(&ci_sorted[slot]) = r;  // order inside a cell is arbitrary: consumers rank by sortkey
    }
}
