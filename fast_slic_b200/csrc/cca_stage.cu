// fast_slic_b200/csrc/cca_stage.cu -- the host side of connectivity enforcement: sizes and lays out the scratch,
// owns the side streams and timing events, and enqueues the kernels of cca.cuh over a batch in sub-batches.
#include <stdlib.h>
#include <algorithm>
#include <type_traits>

#include "capi_common.h"
#include "cca.cuh"
#include "cca_stage.h"

// Pointers into the scratch, every array [images][per image]
struct CcaScratch {
    int* par;                       // parent
    uint32_t* aux;                  // area at root pixel
    uint32_t* carea;                // area by component number
    uint16_t* cnew;                 // new label by component number
    uint16_t* fin;                  // final label at root pixel (second half of the cnew piece)
    int* rootbuf;                   // ordered root lists of k_ccl_flatten (its own array: two halves of a batch may be
                                    // in different phases at the same time)
    int* predbuf;                   // predecessor root of every rootbuf entry
    unsigned long long* chunkinfo;  // [nblk * 32] root mask and root-list offset of every 32-pixel chunk
    int* blkcnt;                    // [nblk] roots per block, then kept components per 1024-component chunk
    int* blkoff;                    // [nblk] component number of the first root of a block
    int* kblkoff;                   // [nblk] kept components in front of a 1024-component chunk
    CcaCounters* counters;          // [1]
    unsigned int* ahist;            // [CCA_HIST] histogram of candidate areas
    unsigned long long* heap;       // [CCA_HEAP_K]
    size_t total;                   // bytes of the whole scratch
};

// The scratch of `images` images at `base`, seen from image `slot` on (every pointer advanced by `slot` images).  With a
// null base it only counts: the allocation and every window come from this one function.
static CcaScratch cca_layout(void* base, int N, int images, int slot) {
    CcaScratch x;
    Carve c(base);
    auto take = [&](auto*& p, size_t per_image) {
        using T = std::remove_reference_t<decltype(*p)>;
        p = c.take<T>((size_t)images * per_image * sizeof(T));
        if (p) p += (size_t)slot * per_image;
    };
    const size_t n = (size_t)N, nblk = (size_t)ceil_div(N, CCA_BLOCK);
    take(x.par, n);
    take(x.aux, n);
    take(x.carea, n);
    x.cnew = c.take<uint16_t>((size_t)images * n * 2 * sizeof(uint16_t));  // cnew, then fin
    x.fin = x.cnew ? x.cnew + ((size_t)images + slot) * n : nullptr;
    if (x.cnew) x.cnew += (size_t)slot * n;
    take(x.rootbuf, n);
    take(x.predbuf, n);
    take(x.chunkinfo, nblk * (CCA_BLOCK / 32));
    take(x.blkcnt, nblk);
    take(x.blkoff, nblk);
    take(x.kblkoff, nblk);
    take(x.counters, 1);
    take(x.ahist, CCA_HIST);
    take(x.heap, CCA_HEAP_K);
    x.total = c.total;
    return x;
}

static CcaScratch cca_window(const CcaStage& s, int slot) { return cca_layout(s.scratch, s.N, s.batch, slot); }

cudaError_t cca_stage_create(CcaStage& s, int H, int W, int max_batch, size_t device_bytes, int num_sms, int max_smem_optin) {
    s.H = H; s.W = W; s.N = H * W; s.num_sms = num_sms; s.max_smem_optin = max_smem_optin;
    // 26 B/pixel/image (24.25 used); cap the resident set at an eighth of the device's memory (10 GB on an 80 GB H100,
    // so that several contexts per GPU fit beside their assign state) and at most 12 GB; larger batches run the
    // connectivity stage in sub-batches.  (The rule leaves out the selection heap, 512 KiB per image, and the area
    // histogram, 8 KiB per image: the allocation is cca_layout's total, which counts them.)
    const size_t per_img = (size_t)s.N * 26 + 4096;
    size_t cap = 12ull << 30;
    if (device_bytes && device_bytes / 8 < cap) cap = device_bytes / 8;
    size_t bc = cap / per_img;
    if (bc < 1) bc = 1;
    if (bc > (size_t)max_batch) bc = max_batch;
    if (const char* e = getenv("FSLIC_CCA_BATCH")) {  // test hook: force the sub-batched CCA path
        const long v = atol(e);
        if (v >= 1 && (size_t)v < bc) bc = (size_t)v;
    }
    s.batch = (int)bc;
    cudaError_t e = cudaMalloc(&s.scratch, cca_layout(nullptr, s.N, s.batch, 0).total);
    // the diagnostics entry may read the counters before the first run
    if (e == cudaSuccess) e = cudaMemset(cca_window(s, 0).counters, 0, bc * sizeof(CcaCounters));
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&s.h_counters), 64 * sizeof(CcaCounters));
    for (auto& ev : s.ev)
        if (e == cudaSuccess) e = cudaEventCreate(&ev);
    for (CcaLane& l : s.lanes) {
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&l.side, cudaStreamNonBlocking);
        for (cudaEvent_t* ev : {&l.fork, &l.join, &l.tail})
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
    }
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(k_cca_select, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin - 4 * 1024);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(k_debug_heap_select, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin - 4 * 1024);
    return e;
}

void cca_stage_destroy(CcaStage& s) {
    if (s.scratch) cudaFree(s.scratch);
    if (s.h_counters) cudaFreeHost(s.h_counters);
    for (cudaEvent_t e : s.ev)
        if (e) cudaEventDestroy(e);
    for (const CcaLane& l : s.lanes) {
        if (l.side) cudaStreamDestroy(l.side);
        for (cudaEvent_t e : {l.fork, l.join, l.tail})
            if (e) cudaEventDestroy(e);
    }
}

// CTAs per image of k_ccl_number: sized for full batches (a few CTAs per image); a small batch gets more CTAs per image
// instead, it is all dependent-load latency there
static int number_grid(int nblk, int nb) {
    return nb >= 8 ? CCA_NUMBER_GRID : std::min(std::max(ceil_div(nblk, 32), CCA_NUMBER_GRID), 64);
}

// Labelling of one sub-batch of nb images, up to the threshold decision: union-find, flatten, component numbers and
// areas, k_cca_threshold
static int cca_label(const CcaStage& s, const CcaScratch& x, const CcaParams& cp, const uint16_t* in, int nb, bool timed,
                     cudaStream_t st) {
    if (timed) CK(cudaEventRecord(s.ev[0], st));
    CK(cudaMemsetAsync(x.counters, 0, sizeof(CcaCounters) * nb, st));
    CK(cudaMemsetAsync(x.ahist, 0, sizeof(unsigned int) * CCA_HIST * nb, st));
    dim3 g(cp.nblk, nb);
    {
        const int ttx = ceil_div(s.W, CCL_T), tty = ceil_div(s.H, CCL_T);
        const long ntt = (long)ttx * tty * nb;
        k_ccl_tile<<<(int)((ntt + CCL_TW - 1) / CCL_TW), 32 * CCL_TW, 0, st>>>(cp, in, x.par, x.aux, ttx, tty, ntt);
    }
    {
        const int seam_px = ((s.W - 1) / CCL_T) * s.H + ((s.H - 1) / CCL_T) * s.W;
        if (seam_px > 0) {
            dim3 gs(ceil_div(seam_px, 256), nb);
            k_ccl_seams<<<gs, 256, 0, st>>>(cp, in, x.par);
        }
    }
    if (timed) CK(cudaEventRecord(s.ev[1], st));
    k_ccl_flatten<<<g, 256, 0, st>>>(cp, in, x.par, x.aux, x.blkcnt, x.rootbuf, x.predbuf, x.chunkinfo);
    k_scan_blocks<<<nb, 1024, 0, st>>>(x.blkcnt, x.blkoff, cp.nblk, cp.nblk, nullptr, 0, 1,
                                       &x.counters[0].ncomp, (int)(sizeof(CcaCounters) / sizeof(int)), nullptr, -1);
    k_ccl_number<<<dim3(number_grid(cp.nblk, nb), nb), CCA_BLOCK, 0, st>>>(cp, x.rootbuf, x.aux, x.blkcnt, x.blkoff,
                                                                            x.carea, x.counters, x.ahist);
    if (timed) CK(cudaEventRecord(s.ev[2], st));
    k_cca_threshold<<<nb, 1024, 0, st>>>(cp, x.carea, x.counters, x.ahist);
    if (timed) CK(cudaEventRecord(s.ev[3], st));
    return FSLIC_OK;
}

// The kernels after the threshold decision (kept labels, absorption, output) for the images `which` selects (-1 all,
// 0 the settled ones, 1 the replayed ones), on ts
static void cca_finish(const CcaStage& s, const CcaScratch& x, const CcaParams& cp, int which, uint16_t* out, int nb,
                       bool timed, cudaStream_t ts) {
    CcaParams cq = cp;
    cq.which = which;
    // (blkoff keeps the component number of each block's first root for k_cca_absorb: the kept offsets of the
    // 1024-component chunks go to kblkoff)
    const dim3 gk(std::min(cp.nblk, std::max(CCA_KEPT_GRID, 256 / nb)), nb);
    k_kept_count<<<gk, CCA_BLOCK, 0, ts>>>(cq, x.carea, x.counters, x.blkcnt);
    k_scan_blocks<<<nb, 1024, 0, ts>>>(x.blkcnt, x.kblkoff, cp.nblk, 0, &x.counters[0].ncomp,
                                       (int)(sizeof(CcaCounters) / sizeof(int)), CCA_BLOCK,
                                       &x.counters[0].nkept, (int)(sizeof(CcaCounters) / sizeof(int)),
                                       x.counters, which);
    k_kept_label<<<gk, CCA_BLOCK, 0, ts>>>(cq, x.carea, x.counters, x.kblkoff, x.cnew);
    if (timed) cudaEventRecord(s.ev[4], ts);
    // one warp per 1024-pixel block and its root list; below 4 images, 8 warps per block (all latency there)
    const int nsplit = nb < 4 ? 8 : 1;
    const dim3 ga(ceil_div(cp.nblk * nsplit, CCA_TAIL_WARPS), nb);
    k_cca_absorb<<<ga, 32 * CCA_TAIL_WARPS, 0, ts>>>(cq, x.rootbuf, x.predbuf, x.chunkinfo, x.blkoff, x.counters,
                                                      x.cnew, x.fin, nsplit);
    if (timed) cudaEventRecord(s.ev[5], ts);
    int ob = ceil_div(ceil_div(s.N, 8), 256);  // 8 pixels per thread on the vector path (any N works: grid-stride)
    if (ob > s.num_sms * 32) ob = s.num_sms * 32;
    dim3 go(ob, nb);
    k_cca_output<<<go, 256, 0, ts>>>(cq, x.par, x.fin, out, x.counters);
    if (timed) cudaEventRecord(s.ev[6], ts);
}

// D2H on ho's stream of the maximal runs of images whose need_sim flag (read back into hcnt) is `replayed`
static int cca_copy_runs(const CcaCounters* hcnt, int nb, bool replayed, const uint16_t* out, size_t N, const HostOut& ho) {
    int b = 0;
    while (b < nb) {
        if ((hcnt[b].need_sim != 0) != replayed) { b++; continue; }
        int e = b;
        while (e < nb && (hcnt[e].need_sim != 0) == replayed) e++;
        CK(cudaMemcpyAsync(ho.h_labels + (size_t)b * N, out + (size_t)b * N, (size_t)(e - b) * N * 2,
                           cudaMemcpyDeviceToHost, ho.out_stream));
        b = e;
    }
    return FSLIC_OK;
}

int cca_run(CcaStage& s, CcaDispatch& d, const uint16_t* d_in, uint16_t* d_out, int batch, int K, int thres,
            cudaStream_t st, int* launches, HostOut* ho, int slot, int lane) {
    const int N = s.N;
    if (slot != 0 && slot + batch > s.batch) return set_err(FSLIC_EINVAL, "scratch window out of range");
    const CcaScratch x = cca_window(s, slot);
    CcaCounters* const hcnt = s.h_counters + slot;
    const CcaLane& ln = s.lanes[lane];
    CcaParams cp;
    cp.H = s.H; cp.W = s.W; cp.N = N; cp.K = K; cp.thres = thres; cp.which = -1;
    cp.nblk = ceil_div(N, CCA_BLOCK);
    const size_t heap_bytes = (size_t)(2 * K + 4) * 8;  // live slots + the +infinity padding of the replay loop
    cp.heap_in_smem = heap_bytes + SEL_CHUNK * 8 <= (size_t)(s.max_smem_optin - 8 * 1024);
    if (K + 2 > CCA_HEAP_K) return set_err(FSLIC_EINVAL, "K too large for the selection heap");
    d.heap_smem = cp.heap_in_smem ? 1 : 0;
    d.heap_smem_max_k =
        (int)std::max<long>(0, ((long)s.max_smem_optin - 8 * 1024 - SEL_CHUNK * 8) / 8 / 2 - 2);  // (2K+4)*8 fits
    d.sub_batches = ceil_div(batch, s.batch);
    for (int b0 = 0; b0 < batch; b0 += s.batch) {
        const int nb = (batch - b0 < s.batch) ? (batch - b0) : s.batch;
        const uint16_t* in = d_in + (size_t)b0 * N;
        uint16_t* out = d_out + (size_t)b0 * N;
        const bool timed = s.timing && nb < 4 && batch <= s.batch;  // one stream, one sub-batch
        s.timed = timed;
        int rc = cca_label(s, x, cp, in, nb, timed, st);
        if (rc) return rc;
        if (b0 == 0) {
            d.split = nb >= 4;
            d.number_nb = ceil_div(cp.nblk, number_grid(cp.nblk, nb) * (CCA_BLOCK / 32));  // NB of k_ccl_number
        }
        // Everything after the threshold decision depends on the kept set.  For images k_cca_threshold settled
        // that is known now; for the (few) images whose ties need the sequential std::partial_sort replay it
        // is known only after k_cca_select, which keeps a handful of SMs busy for ~1 ms.  So for batches the
        // finishing kernels run twice: for the settled images on a side stream concurrently with the replay, and
        // for the replayed images afterwards.
        const bool split = nb >= 4;
        const bool early = split && ho && batch <= s.batch && nb <= 64;
        if (early) {
            // the host path is synchronous anyway: wait for the threshold decision and read the per-image flags
            CK(cudaMemcpyAsync(hcnt, x.counters, sizeof(CcaCounters) * nb, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        if (split) {
            CK(cudaEventRecord(ln.fork, st));
            CK(cudaStreamWaitEvent(ln.side, ln.fork, 0));
            cca_finish(s, x, cp, 0, out, nb, timed, ln.side);
            CK(cudaEventRecord(ln.join, ln.side));
        }
        if (early) {
            CK(cudaStreamWaitEvent(ho->out_stream, ln.join, 0));
            rc = cca_copy_runs(hcnt, nb, false, out, N, *ho);
            if (rc) return rc;
        }
        k_cca_select<<<nb, 1024, SEL_CHUNK * 8 + (cp.heap_in_smem ? heap_bytes : 0), st>>>(cp, x.carea, x.counters, x.heap);
        cca_finish(s, x, cp, split ? 1 : -1, out, nb, timed, st);
        if (early) {
            CK(cudaEventRecord(ln.tail, st));
            CK(cudaStreamWaitEvent(ho->out_stream, ln.tail, 0));
            rc = cca_copy_runs(hcnt, nb, true, out, N, *ho);
            if (rc) return rc;
            ho->done = true;
        }
        if (split) {
            CK(cudaStreamWaitEvent(st, ln.join, 0));
            if (launches) *launches += 5;
        }
        CK(cudaGetLastError());
        if (launches) *launches += 12;
    }
    return FSLIC_OK;
}

void cca_set_timing(CcaStage& s, bool on) {
    s.timing = on;
    s.timed = false;
}

void cca_read_timing(CcaStage& s) {
    for (int i = 0; i < 6; i++) {
        float ms;
        s.ms[i] = 0.f;
        if (s.timed && cudaEventElapsedTime(&ms, s.ev[i], s.ev[i + 1]) == cudaSuccess) s.ms[i] = ms;
    }
    cudaGetLastError();
}

void cca_sync_lanes(const CcaStage& s) {
    for (const CcaLane& l : s.lanes)
        if (l.side) cudaStreamSynchronize(l.side);
}

int cca_heap_select(const CcaStage& s, const int32_t* d_area, int n, int middle, uint8_t* d_kept, cudaStream_t st) {
    CK(cudaMemsetAsync(d_kept, 0, n, st));
    const size_t hb = (size_t)(2 * middle + 4) * 8;
    const int use_smem = hb + SEL_CHUNK * 8 <= (size_t)(s.max_smem_optin - 8 * 1024);
    k_debug_heap_select<<<1, 1024, SEL_CHUNK * 8 + (use_smem ? hb : 0), st>>>(reinterpret_cast<const uint32_t*>(d_area), n,
                                                                              middle, d_kept, cca_window(s, 0).heap, use_smem);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

int cca_read_counters(const CcaStage& s, int32_t* out8, int image) {
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out8, cca_window(s, image).counters, sizeof(CcaCounters), cudaMemcpyDeviceToHost));
    return FSLIC_OK;
}

void cca_read_dispatch(const CcaDispatch& d, int32_t* out, int count) {
    const int32_t v[FSLIC_CCA_DISPATCH_COUNT] = {d.heap_smem, d.heap_smem_max_k, d.sub_batches, d.split, d.number_nb};
    for (int i = 0; i < count && i < FSLIC_CCA_DISPATCH_COUNT; i++) out[i] = v[i];
}

void cca_read_ms(const CcaStage& s, float* out_ms, int count) {
    for (int i = 0; i < count && i < 6; i++) out_ms[i] = s.ms[i];
}
