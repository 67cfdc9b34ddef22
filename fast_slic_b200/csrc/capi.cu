// fast_slic_b200/csrc/capi.cu -- host orchestration + the extern "C" boundary (include/fslic_b200.h).
//
// Plays the role of BaseContext<uint16_t>::iterate (fast-slic/src/context.cpp:109-197) and of
// the Cython glue that drives it (cfast_slic.pyx:124-197): owns the scratch buffers, sequences the
// kernels on one stream, never touches the CPU for the data path.
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <algorithm>
#include <new>
#include <cstring>
#include <deque>
#include <string>
#include <unordered_set>
#include <vector>

#include "assign.cuh"
#include "assign5.cuh"
#include "capi_common.h"
#include "realdist.cuh"
#include "lsc.cuh"
#include "crf.cuh"
#include "crf_feed.cuh"
#include "preempt.cuh"
#include "cca.cuh"
#include "common.cuh"
#include "lab.cuh"
#include "trace.cuh"
#include "recorder_format.h"

#define SPT_MAX_ELEMS (128 * 1024)  // u16 elements per spatial patch buffer

typedef void (*assign_fn)(AssignParams, const uint32_t*, uint16_t*, const CInfo*, const int*, unsigned long long*,
                          const uint16_t*);
static assign_fn pick_assign(int TS, int stride, bool update);

typedef void (*assign5_fn)(const AssignParams, const CUtensorMap, const CUtensorMap, const uint32_t*, uint16_t*, const CInfo*,
                           const int*, unsigned long long*, const uint16_t*, fslic_cluster*, CInfo*, int*, unsigned int*);
static assign5_fn pick_assign5(int TS, bool update, int tps, bool fuse = false);

// The one message fslic_b200_last_error() returns, for the entry points of every translation unit
static thread_local std::string g_err;
int set_err(int code, const std::string& msg) {
    g_err = msg;
    return code;
}

// What the host enqueued for one assign pass (fslic_b200_debug_dispatch): kernel 5 = TMA-staged, 4 = LDG warp tiles,
// 0 = generic, 10 / 11 / 12 = float-distance variant 0 / 1 / 2, 13 = preemptive, 14 = LSC, -1 = none yet.  Workers
// are warps per CTA for the tile kernels and threads per CTA for the per-pixel ones; items are super tiles or pixels.
struct PassDispatch {
    int kernel = -1, tps = 0, grid = 0, workers = 0;
    long long items = 0;
    int trips = 0;  // ceil(items / (grid * workers)): rounds of the kernel's grid-stride walk
};
struct DispatchRecord {
    PassDispatch upd, full;  // the last update pass launched, the full-assign pass
    int prepare = 0;         // kernel of the last run_prepare: 3 = k_prepare3, 2 = k_prepare2, 1 = k_prepare
    int fused = 0;           // update passes whose TMA tail ran the next pass's prepare
    int lsc_trips = 0;       // rounds of k_lsc_features
    // connectivity stage (run_cca), recorded when enqueued
    int cca_heap_smem = -1;       // k_cca_select's heap: 1 = shared memory, 0 = global memory, -1 = no connectivity stage ran
    int cca_heap_smem_max_k = 0;  // largest K whose heap fits shared memory on this device
    int cca_sub_batches = 0;      // sub-batches of at most cca_batch images
    int cca_split = 0;            // first sub-batch: settled images' tail on the side stream (nb >= 4)
    int cca_number_nb = 0;        // first sub-batch: 1024-pixel blocks per k_ccl_number warp
};

struct fslic_ctx {
    int device = 0, H = 0, W = 0, K = 0, maxB = 0, S = 0, N = 0;
    bool cca_only = false;  // fslic_b200_create_cca: connectivity scratch only
    int num_sms = 132;
    // tables
    uint16_t *d_gamma = nullptr, *d_labtbl = nullptr;
    LabConsts lc;
    // assign state
    uint32_t* quad = nullptr;      // [B][N]   Lab quad image
    uint16_t* labels = nullptr;    // [B][N]   pre-CCA labels
    CInfo* cinfo = nullptr;        // [B][K]
    unsigned long long* acc = nullptr;  // [B][K][4] packed sums (assign.cuh)
    int* cell_start = nullptr;     // [B][ncell+1]
    CInfo* cinfo_tmp = nullptr;    // [B][K] scratch of k_prepare (records by cluster index)
    int* cell_cnt = nullptr;       // [B][ncell+1] cell histogram of k_prepare2 (zero between launches)
    unsigned int* prep_tickets = nullptr;  // [B] arrival counters of k_prepare2 (zero between launches)
    uint16_t* sptable = nullptr;   // two linear spatial patches: [0] subsampled passes, [1] full pass
    int G = 1, cellW = 1, cellH = 1, ncell = 1;
    // cca state (sized for cca_batch images at a time)
    int cca_batch = 1;
    int* par = nullptr;            // [Bc][N]
    uint32_t* aux = nullptr;       // [Bc][N]  area at root pixel
    uint32_t* carea = nullptr;     // [Bc][N]  area by component number
    uint16_t* cnew = nullptr;      // [Bc][N]  new label by component number
    uint16_t* fin = nullptr;       // [Bc][N]  final label at root pixel (second half of the cnew allocation)
    int* rootbuf = nullptr;        // [Bc][N] ordered root lists of k_ccl_flatten
    int* predbuf = nullptr;        // [Bc][N] predecessor root of every rootbuf entry
    unsigned long long* chunkinfo = nullptr;  // [Bc][nblk * 32] root mask and root-list offset of every 32-pixel chunk
    int* blkcnt = nullptr;         // [Bc][nblk] roots per block, then kept components per 1024-component chunk
    int* blkoff = nullptr;         // [Bc][nblk] component number of the first root of a block
    int* kblkoff = nullptr;        // [Bc][nblk] kept components in front of a 1024-component chunk
    CcaCounters* counters = nullptr;  // [Bc]
    unsigned int* ahist = nullptr;    // [Bc][CCA_HIST] histogram of candidate areas
    unsigned long long* heap = nullptr;  // [Bc][Kheap]
    int heap_K = 0;
    // staging for the host entry points
    uint8_t* d_img = nullptr;
    fslic_cluster* d_cl = nullptr;
    uint16_t* d_lab = nullptr;
    cudaStream_t own_stream = nullptr, in_stream = nullptr, out_stream = nullptr, side_stream = nullptr;
    cudaEvent_t side_fork = nullptr, side_join = nullptr, tail_done = nullptr;
    // second lane of the blocking host path (the two halves of a batch overlap on the device)
    cudaStream_t own_stream2 = nullptr, side_stream2 = nullptr;
    cudaEvent_t side_fork2 = nullptr, side_join2 = nullptr, tail_done2 = nullptr, front_done = nullptr;
    // the `preemptive` option (preempt.cuh), allocated at the first such call
    uint8_t* pre_cellmap = nullptr;     // [B][ceil(H/2S) * ceil(W/2S)] active 2S x 2S cells
    int* pre_nactive = nullptr;         // [B] active clusters
    float preempt_l1 = 0.f;             // max(roundf(2 S thres), 1) of the call in progress
    long long* selprof = nullptr;       // FSLIC_SELPROF=1: 8 words per image written by k_cca_select (diagnostics)
    CcaCounters* h_counters = nullptr;  // pinned, 64 entries: lets the host path learn which images need the replay
    std::vector<cudaEvent_t> pipe_ev;  // [2 * chunks]: input-ready / compute-done events of iterate_host
    // timing
    cudaEvent_t ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    // the reference's sub-sections of "cca" (cca.cpp:194-263): build_disjoint_set, flatten, threshold_by_area, sort,
    // substitute, output -- event-timed when collect_timing is on and the batch is not split across streams
    cudaEvent_t cev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    float cca_ms[6] = {0, 0, 0, 0, 0, 0};
    bool cca_timing = false, cca_timed = false;
    float stage_ms[FSLIC_T_COUNT] = {0, 0, 0, 0, 0, 0, 0, 0};
    int last_launches = 0;
    int slice = 0;  // first image of the batch slice the front half (Lab + passes) currently works on
    int max_smem_optin = 0;
    // per-launch timing of the dominant kernel (k_assign_tiles on the subsampled passes)
    std::vector<cudaEvent_t> kev;
    int kev_used = 0;
    bool kev_on = false;
    bool pending = false;  // an iterate_host_async batch is in flight on this context's streams
    // small host batches replay one captured CUDA graph per call instead of ~45 launches (FSLIC_GRAPH=0 turns it off)
    bool graphs_enabled = true;
    cudaGraphExec_t gexec = nullptr;
    struct GraphKey {
        const void *img, *cl, *lab;
        int batch;
        fslic_params p;
        int manhattan;
    } gkey = {nullptr, nullptr, nullptr, 0, {0.f, 0.f, 0, 0, 0, 0}, 0}, gkey_seen = {nullptr, nullptr, nullptr, 0, {0.f, 0.f, 0, 0, 0, 0}, 0};
    int glaunches = 0;
    int graph_captures = 0, graph_replays = 0;  // fslic_b200_debug_graph_counts
    float assign_kernel_ms = 0.f;
    int assign_kernel_launches = 0;
    bool spt_valid = false, spt_has_sub = false;  // what c->sptable currently holds (build_patches)
    int spt_stride = 0;
    cudaStream_t spt_stream = nullptr;
    uint32_t spt_coef_bits = 0;
    int spt_manhattan = 1;
    int manhattan = 1;         // manhattan_spatial_dist (fslic_b200_set_manhattan_spatial_dist): read by every iterate
    // LSC (lsc.cuh), allocated at the first fslic_b200_iterate_lsc call
    float* lsc_feat = nullptr;      // [B][10][N] normalised features
    float* lsc_w = nullptr;         // [B][N]     pixel weights
    float* lsc_tab = nullptr;       // [1024 + 2W + 2H] feature tables (lsc.cuh)
    float* lsc_means = nullptr;     // [B][10]    feature means
    float* lsc_cf = nullptr;        // [B][K][LSC_CF] centroid features
    float* lsc_cf_init = nullptr;   // [B][K][10] centroid features after before_iteration (debug read-out)
    LscBox* lsc_box = nullptr;      // [B][K]     label bounding boxes of the current pass
    std::vector<float> lsc_htab;    // host copy of lsc_tab and the compactness it was built for
    uint32_t lsc_tab_key = 0;
    bool lsc_tab_valid = false;
    std::vector<cudaEvent_t> lev;   // start / end events of each after_update launch (collect_timing)
    int lev_used = 0;
    int assign_impl = 5;       // 5: TMA-staged kernel where it applies (default), 4: always the LDG kernel (FSLIC_ASSIGN=4)
    DispatchRecord disp;       // launch decisions of the last iterate (tests, bench)
    DispatchRecord gdisp;      // ... of the call captured into gexec: a replay makes the same ones
    // debug_mode (fslic_b200_set_trace, trace.cuh): snapshots of the last traced iterate, [B][T] slots, allocated on demand
    bool trace_on = false;
    int tr_T = 0, tr_B = 0, tr_dist_bytes = 0;  // what the buffers hold (tr_T == 0: nothing recorded)
    size_t tr_cap = 0;                          // bytes allocated at tr_buf
    void* tr_buf = nullptr;                     // clusters [B][T][K], then assignment [B][T][N], then min_dists [B][T][N]
    unsigned int* tr_bad = nullptr;             // pixels whose label disagreed with the trace kernel's argmin
};

extern "C" const char* fslic_b200_last_error(void) { return g_err.c_str(); }
extern "C" const char* fslic_b200_version(void) { return "fast_slic_b200 0.1 (sm_90a)"; }
extern "C" int fslic_b200_sizeof_cluster(void) { return (int)sizeof(fslic_cluster); }
extern "C" int fslic_b200_get_S(const fslic_ctx* ctx) { return ctx ? ctx->S : -1; }
extern "C" int fslic_b200_launches_last_iterate(const fslic_ctx* ctx) { return ctx ? ctx->last_launches : -1; }
extern "C" int fslic_b200_debug_assign_impl(const fslic_ctx* ctx) {
    if (!ctx) return -1;
    const int k = ctx->disp.full.kernel;
    return k == 5 || k == 4 ? k : 0;
}
extern "C" int fslic_b200_debug_dispatch(const fslic_ctx* ctx, int32_t* out, int count) {
    if (!ctx || !out) return set_err(FSLIC_EINVAL, "NULL argument");
    const DispatchRecord& d = ctx->disp;
    int32_t v[FSLIC_DISPATCH_COUNT];
    int n = 0;
    for (const PassDispatch* p : {&d.upd, &d.full}) {
        v[n++] = p->kernel; v[n++] = p->tps; v[n++] = p->grid; v[n++] = p->workers;
        v[n++] = (int32_t)std::min<long long>(p->items, INT32_MAX);
        v[n++] = p->trips;
    }
    v[n++] = d.prepare; v[n++] = d.fused; v[n++] = d.lsc_trips;
    for (int i = 0; i < count && i < FSLIC_DISPATCH_COUNT; i++) out[i] = v[i];
    return FSLIC_OK;
}
extern "C" int fslic_b200_debug_cca_dispatch(const fslic_ctx* ctx, int32_t* out, int count) {
    if (!ctx || !out) return set_err(FSLIC_EINVAL, "NULL argument");
    const DispatchRecord& d = ctx->disp;
    const int32_t v[FSLIC_CCA_DISPATCH_COUNT] = {d.cca_heap_smem, d.cca_heap_smem_max_k, d.cca_sub_batches, d.cca_split,
                                                 d.cca_number_nb};
    for (int i = 0; i < count && i < FSLIC_CCA_DISPATCH_COUNT; i++) out[i] = v[i];
    return FSLIC_OK;
}
static void record_pass(fslic_ctx* c, bool update, int kernel, int tps, long grid, int workers, long items) {
    PassDispatch& d = update ? c->disp.upd : c->disp.full;
    const long per_round = grid * workers;
    d.kernel = kernel; d.tps = tps; d.grid = (int)grid; d.workers = workers; d.items = items;
    d.trips = (int)((items + per_round - 1) / per_round);
}
extern "C" int fslic_b200_set_manhattan_spatial_dist(fslic_ctx* ctx, int on) {
    if (!ctx) return set_err(FSLIC_EINVAL, "NULL context");
    ctx->manhattan = on ? 1 : 0;
    return FSLIC_OK;
}

// ---- Lab tables: FastCIELabCvt ctor, fast-slic/src/cielab.h:297-305 ----------------------
// _srgb_gamma_tbl (cielab.h:22-279) is the sRGB inverse companding curve documented at
// cielab.h:12-20; it is regenerated here from that formula (bit-identical, checked in tests over the
// whole 2^24 colour cube against the compiled reference).
static void build_lab_tables(std::vector<uint16_t>& gamma, std::vector<uint16_t>& labtbl, LabConsts& lc) {
    static const float C[9] = {0.43395633f, 0.37621531f, 0.18984309f, 0.2126729f, 0.7151522f,
                               0.072175f,   0.01775782f, 0.1094756f,  0.87283638f};
    gamma.resize(256);
    labtbl.resize(8193);
    for (int i = 0; i < 256; i++) {
        const double v = i / 255.0;
        const double X = (v <= 0.04045) ? v / 12.92 : pow((v + 0.055) / 1.055, 2.4);
        gamma[i] = (uint16_t)(int)((float)X * 8192);
    }
    for (int i = 0; i < 9; i++) lc.Cb[i] = (int)roundf(C[i] * 65536);
    for (int i = 0; i <= 8192; i++) {
        const float v = (float)i / 8192;
        const float lo = 7.787f * v + 0.137931f;
        const float hi = powf(v, 0.333333f);
        labtbl[i] = (uint16_t)(int)roundf(((v > 0.008856f) ? hi : lo) * 8192);
    }
}

template <typename T>
static cudaError_t dalloc(T** p, size_t count) {
    return cudaMalloc(reinterpret_cast<void**>(p), count * sizeof(T) + 256);
}

extern "C" int fslic_b200_destroy(fslic_ctx* c) {
    if (!c) return FSLIC_OK;
    DeviceGuard dev_guard__(c->device);
    void* ptrs[] = {c->d_gamma, c->d_labtbl, c->quad,   c->labels,  c->cinfo,  c->acc,    c->cell_start,
                    c->cinfo_tmp, c->cell_cnt, c->prep_tickets, c->sptable, c->par,  c->aux,    c->predbuf, c->carea,
                    c->cnew,    c->chunkinfo, c->rootbuf, c->blkcnt, c->blkoff,  c->kblkoff, c->counters, c->ahist, c->heap, c->d_img,
                    c->d_cl,    c->d_lab};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    for (auto& e : c->ev)
        if (e) cudaEventDestroy(e);
    for (auto& e : c->cev)
        if (e) cudaEventDestroy(e);
    for (auto& e : c->kev) cudaEventDestroy(e);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    if (c->in_stream) cudaStreamDestroy(c->in_stream);
    if (c->out_stream) cudaStreamDestroy(c->out_stream);
    if (c->side_stream) cudaStreamDestroy(c->side_stream);
    if (c->side_fork) cudaEventDestroy(c->side_fork);
    if (c->side_join) cudaEventDestroy(c->side_join);
    if (c->tail_done) cudaEventDestroy(c->tail_done);
    if (c->own_stream2) cudaStreamDestroy(c->own_stream2);
    if (c->side_stream2) cudaStreamDestroy(c->side_stream2);
    for (cudaEvent_t e : {c->side_fork2, c->side_join2, c->tail_done2, c->front_done})
        if (e) cudaEventDestroy(e);
    if (c->gexec) cudaGraphExecDestroy(c->gexec);
    if (c->h_counters) cudaFreeHost(c->h_counters);
    if (c->selprof) cudaFree(c->selprof);
    if (c->pre_cellmap) cudaFree(c->pre_cellmap);
    if (c->pre_nactive) cudaFree(c->pre_nactive);
    for (auto& e : c->pipe_ev) cudaEventDestroy(e);
    for (void* p : {(void*)c->lsc_feat, (void*)c->lsc_w, (void*)c->lsc_tab, (void*)c->lsc_means, (void*)c->lsc_cf,
                    (void*)c->lsc_cf_init, (void*)c->lsc_box, c->tr_buf, (void*)c->tr_bad})
        if (p) cudaFree(p);
    for (auto& e : c->lev) cudaEventDestroy(e);
    delete c;
    return FSLIC_OK;
}

static int create_impl(int device, int H, int W, int K, int max_batch, bool cca_only, fslic_ctx** out) {
    if (!out) return set_err(FSLIC_EINVAL, "out is NULL");
    *out = nullptr;
    if (H <= 0 || W <= 0) return set_err(FSLIC_EINVAL, "H and W must be positive");
    if (K <= 0) return set_err(FSLIC_EINVAL, "num_components should be a non-negative integer");  // cfast_slic.pyx:26-27
    if (K >= 65534) return set_err(FSLIC_EINVAL, "num_components cannot exceed 65534");              // cfast_slic.pyx:24-25
    if (max_batch <= 0) return set_err(FSLIC_EINVAL, "max_batch must be positive");
    if ((long)H * W >= (1L << 30)) return set_err(FSLIC_EINVAL, "image too large (H*W must be < 2^30)");
    if (H > 32767 || W > 32767) return set_err(FSLIC_EINVAL, "H and W must fit int16 (the reference truncates centres to int16)");
    USE_DEVICE(device);
    fslic_ctx* c = new (std::nothrow) fslic_ctx();
    if (!c) return set_err(FSLIC_ENOMEM, "out of host memory");
    c->device = device;
    c->cca_only = cca_only;
    c->H = H; c->W = W; c->K = K; c->maxB = max_batch; c->N = H * W;
    c->S = (int)(int16_t)sqrt((double)(H * W / K));  // context.h:60 (integer division first)
    if (c->S < 1 && !cca_only) {  // the reference divides by zero here (PreemptiveGrid: ceil_int(W, 2*S), preemptive.h:37-38)
        delete c;
        return set_err(FSLIC_EINVAL, "num_components exceeds the number of pixels (S = 0): the reference crashes on this input");
    }
    cudaDeviceProp prop;
    size_t device_bytes = 0;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
        c->num_sms = prop.multiProcessorCount;
        c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
        device_bytes = prop.totalGlobalMem;
    }
    const size_t B = (size_t)max_batch, N = (size_t)c->N;
#define CKC(call)                                                                                  \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess) {                                                                  \
            std::string m = std::string(#call) + ": " + cudaGetErrorString(e__);                   \
            fslic_b200_destroy(c);                                                                 \
            return set_err(e__ == cudaErrorMemoryAllocation ? FSLIC_ENOMEM : FSLIC_ECUDA, m);      \
        }                                                                                          \
    } while (0)
    std::vector<uint16_t> gamma, labtbl;
    build_lab_tables(gamma, labtbl, c->lc);
    CKC(dalloc(&c->d_gamma, 256));
    CKC(dalloc(&c->d_labtbl, 8200));
    CKC(cudaMemcpy(c->d_gamma, gamma.data(), 256 * 2, cudaMemcpyHostToDevice));
    CKC(cudaMemcpy(c->d_labtbl, labtbl.data(), 8193 * 2, cudaMemcpyHostToDevice));

    // candidate cell grid: pitch G >= max(S,1), at most ~16K cells so the histogram fits in smem
    int G = c->S > 2 ? c->S : 2;  // >= 2 so that ceil(2^32/G) fits 32 bits (div_g)
    while ((long)ceil_div(H, G) * ceil_div(W, G) > 16000) G++;
    c->G = G; c->cellW = ceil_div(W, G); c->cellH = ceil_div(H, G); c->ncell = c->cellW * c->cellH;

    if (!cca_only) {  // assign state (a connectivity-only context needs none of it)
        CKC(dalloc(&c->quad, B * N));
        CKC(dalloc(&c->labels, B * N));
        CKC(dalloc(&c->cinfo, B * K));
        CKC(dalloc(&c->acc, B * K * 4));
        CKC(cudaMemset(c->acc, 0, B * K * 4 * sizeof(unsigned long long)));
        CKC(dalloc(&c->cell_start, B * (c->ncell + 1)));
        CKC(dalloc(&c->cinfo_tmp, B * K));
        CKC(dalloc(&c->cell_cnt, B * (c->ncell + 1)));
        CKC(cudaMemset(c->cell_cnt, 0, B * (c->ncell + 1) * sizeof(int)));
        CKC(dalloc(&c->prep_tickets, B));
        CKC(cudaMemset(c->prep_tickets, 0, B * sizeof(unsigned int)));
        CKC(dalloc(&c->sptable, (size_t)2 * SPT_MAX_ELEMS));
    }

    // CCA scratch: 26 B/pixel/image (24.25 used); cap the resident set at an eighth of the device's memory (10 GB on an 80 GB H100,
    // so that several contexts per GPU fit beside their assign state) and at most 12 GB; larger batches run the
    // connectivity stage in sub-batches
    const size_t per_img = N * 26 + 4096;
    size_t cca_cap = 12ull << 30;
    if (device_bytes && device_bytes / 8 < cca_cap) cca_cap = device_bytes / 8;
    size_t bc = cca_cap / per_img;
    if (bc < 1) bc = 1;
    if (bc > B) bc = B;
    if (const char* e = getenv("FSLIC_CCA_BATCH")) {  // test hook: force the sub-batched CCA path
        const long v = atol(e);
        if (v >= 1 && (size_t)v < bc) bc = (size_t)v;
    }
    c->cca_batch = (int)bc;
    if (const char* e = getenv("FSLIC_GRAPH")) c->graphs_enabled = atoi(e) != 0;
    const int nblk = ceil_div(c->N, CCA_BLOCK);
    CKC(dalloc(&c->par, bc * N));
    CKC(dalloc(&c->aux, bc * N));
    CKC(dalloc(&c->carea, bc * N));
    CKC(dalloc(&c->cnew, 2 * bc * N));
    c->fin = c->cnew + bc * N;
    CKC(dalloc(&c->rootbuf, bc * N));  // (its own array: two halves of a batch may be in different phases at the same time)
    CKC(dalloc(&c->predbuf, bc * N));
    CKC(dalloc(&c->chunkinfo, bc * nblk * (CCA_BLOCK / 32)));
    CKC(dalloc(&c->blkcnt, bc * nblk));
    CKC(dalloc(&c->blkoff, bc * nblk));
    CKC(dalloc(&c->kblkoff, bc * nblk));
    CKC(dalloc(&c->counters, bc));
    CKC(cudaMemset(c->counters, 0, bc * sizeof(CcaCounters)));  // the diagnostics entry may read them before the first run
    CKC(dalloc(&c->ahist, bc * CCA_HIST));
    c->heap_K = 65536 + 8;
    CKC(dalloc(&c->heap, bc * (size_t)c->heap_K));
    for (auto& e : c->ev) CKC(cudaEventCreate(&e));
    for (auto& e : c->cev) CKC(cudaEventCreate(&e));
    CKC(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->in_stream, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->out_stream, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking));
    CKC(cudaEventCreateWithFlags(&c->side_fork, cudaEventDisableTiming));
    CKC(cudaEventCreateWithFlags(&c->side_join, cudaEventDisableTiming));
    CKC(cudaEventCreateWithFlags(&c->tail_done, cudaEventDisableTiming));
    CKC(cudaStreamCreateWithFlags(&c->own_stream2, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->side_stream2, cudaStreamNonBlocking));
    CKC(cudaEventCreateWithFlags(&c->side_fork2, cudaEventDisableTiming));
    CKC(cudaEventCreateWithFlags(&c->side_join2, cudaEventDisableTiming));
    CKC(cudaEventCreateWithFlags(&c->tail_done2, cudaEventDisableTiming));
    CKC(cudaEventCreateWithFlags(&c->front_done, cudaEventDisableTiming));
    CKC(cudaMallocHost(reinterpret_cast<void**>(&c->h_counters), 64 * sizeof(CcaCounters)));
    if (const char* e = getenv("FSLIC_SELPROF")) {
        if (atoi(e) != 0) {
            CKC(cudaMalloc(reinterpret_cast<void**>(&c->selprof), (size_t)c->cca_batch * 8 * sizeof(long long)));
            CKC(cudaMemset(c->selprof, 0, (size_t)c->cca_batch * 8 * sizeof(long long)));
        }
    }

    // opt in to large dynamic shared memory once
    for (int ts : {128, 192, 256, 384})
        for (int stride : {0, 1, 3})
            for (int upd = 0; upd < 2; upd++)
                CKC(cudaFuncSetAttribute(pick_assign(ts, stride, upd != 0), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         c->max_smem_optin - 1024));
    for (int ts : {128, 192, 256})
        for (int upd = 0; upd < 2; upd++)
            for (int tps : {1, 4})
                for (int fuse = 0; fuse <= upd; fuse++)
                    CKC(cudaFuncSetAttribute(pick_assign5(ts, upd != 0, tps, fuse != 0), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             c->max_smem_optin - 1024));
    if (const char* e = getenv("FSLIC_ASSIGN")) c->assign_impl = atoi(e) == 4 ? 4 : 5;
    CKC(cudaFuncSetAttribute(k_cca_select, cudaFuncAttributeMaxDynamicSharedMemorySize, c->max_smem_optin - 4 * 1024));
    CKC(cudaFuncSetAttribute(k_debug_heap_select, cudaFuncAttributeMaxDynamicSharedMemorySize, c->max_smem_optin - 4 * 1024));
    CKC(cudaFuncSetAttribute(k_prepare, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
    CKC(cudaFuncSetAttribute(k_prepare2, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
    CKC(cudaFuncSetAttribute(k_prepare3, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
    CKC(cudaFuncSetAttribute(k_rgb_to_lab16, cudaFuncAttributeMaxDynamicSharedMemorySize, LAB16_SMEM));
    *out = c;
    return FSLIC_OK;
}

extern "C" int fslic_b200_create(int device, int H, int W, int K, int max_batch, fslic_ctx** out) {
    return create_impl(device, H, W, K, max_batch, false, out);
}

extern "C" int fslic_b200_create_cca(int device, int H, int W, int max_batch, fslic_ctx** out) {
    return create_impl(device, H, W, 1, max_batch, true, out);
}

static int check_batch(fslic_ctx* c, int batch, bool needs_assign_state = true) {
    if (!c) return set_err(FSLIC_EINVAL, "ctx is NULL");
    if (batch <= 0 || batch > c->maxB) return set_err(FSLIC_EINVAL, "batch out of range for this context");
    if (needs_assign_state && c->cca_only)
        return set_err(FSLIC_EINVAL, "this context was created by fslic_b200_create_cca: only enforce_connectivity is available");
    return FSLIC_OK;
}

extern "C" int fslic_b200_initialize_clusters(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters,
                                              int batch, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    dim3 grid(ceil_div(c->K, 128), batch);
    k_init_clusters<<<grid, 128, 0, (cudaStream_t)stream>>>(d_images, d_clusters, c->H, c->W, c->K, batch);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

static int launch_lab(fslic_ctx* c, const uint8_t* d_images, uint32_t* quad, int batch, int convert_to_lab,
                      cudaStream_t st) {
    const long npix = (long)batch * c->N;
    long blocks = (npix / 4 + 255) / 256;
    const long cap = (long)c->num_sms * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    if (convert_to_lab && ((reinterpret_cast<uintptr_t>(d_images) | reinterpret_cast<uintptr_t>(quad)) & 15) == 0 && npix >= 4096) {
        // persistent CTAs: the 48 KB of tables are filled once per CTA
        long nb = (npix / 16 + 255) / 256;
        if (nb > (long)c->num_sms * 4) nb = (long)c->num_sms * 4;
        if (nb < 1) nb = 1;
        k_rgb_to_lab16<<<(int)nb, 256, LAB16_SMEM, st>>>(d_images, quad, npix, c->d_gamma, c->d_labtbl, c->lc);
    } else {
        k_rgb_to_quad<<<(int)blocks, 256, 0, st>>>(d_images, quad, npix, c->d_gamma, c->d_labtbl, c->lc, convert_to_lab);
    }
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_rgb_to_quad(fslic_ctx* c, const uint8_t* d_images, uint8_t* d_quad_out, int batch,
                                      int convert_to_lab, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    return launch_lab(c, d_images, reinterpret_cast<uint32_t*>(d_quad_out), batch, convert_to_lab, (cudaStream_t)stream);
}

// ---- connectivity enforcement over `batch` images, chunked by cca_batch -------------------------
// Host-output hook of run_cca (iterate_host only): label maps are copied to the host as soon as they are final --
// for the images k_cca_threshold settled that is while the std::partial_sort replay of the others still runs.
struct HostOut {
    uint16_t* h_labels;      // destination of image 0 of this call
    cudaStream_t out_stream;
    bool done;               // set when run_cca issued the label copies itself
};

// `slot` / `lane`: the blocking host path runs the two halves of a batch as two independent calls that overlap on the
// device; each gets its own window of the scratch arrays (images slot .. slot + batch) and its own side stream / events.
static int run_cca(fslic_ctx* c, const uint16_t* d_in, uint16_t* d_out, int batch, int K, int thres, cudaStream_t st,
                   int* launches, HostOut* ho = nullptr, int slot = 0, int lane = 0) {
    const int N = c->N;
    if (slot != 0 && slot + batch > c->cca_batch) return set_err(FSLIC_EINVAL, "scratch window out of range");
    const size_t so = (size_t)slot;
    const int nblk_all = ceil_div(N, CCA_BLOCK);
    int* const x_par = c->par + so * N;
    uint32_t* const x_aux = c->aux + so * N;
    uint32_t* const x_carea = c->carea + so * N;
    uint16_t* const x_cnew = c->cnew + so * N;
    uint16_t* const x_fin = c->fin + so * N;
    int* const x_rootbuf = c->rootbuf + so * N;
    int* const x_predbuf = c->predbuf + so * N;
    unsigned long long* const x_chunkinfo = c->chunkinfo + so * nblk_all * (CCA_BLOCK / 32);
    int* const x_blkcnt = c->blkcnt + so * nblk_all;
    int* const x_blkoff = c->blkoff + so * nblk_all;
    int* const x_kblkoff = c->kblkoff + so * nblk_all;
    CcaCounters* const x_counters = c->counters + so;
    unsigned int* const x_ahist = c->ahist + so * CCA_HIST;
    unsigned long long* const x_heap = c->heap + so * (size_t)c->heap_K;
    long long* const x_selprof = c->selprof ? c->selprof + 8 * so : nullptr;
    CcaCounters* const x_hcnt = c->h_counters + so;
    cudaStream_t const x_side = lane ? c->side_stream2 : c->side_stream;
    cudaEvent_t const x_fork = lane ? c->side_fork2 : c->side_fork, x_join = lane ? c->side_join2 : c->side_join,
                      x_tail = lane ? c->tail_done2 : c->tail_done;
    CcaParams cp;
    cp.H = c->H; cp.W = c->W; cp.N = N; cp.K = K; cp.thres = thres; cp.which = -1;
    cp.nblk = ceil_div(N, CCA_BLOCK);
    const size_t heap_bytes = (size_t)(2 * K + 4) * 8;  // live slots + the +infinity padding of the replay loop
    cp.heap_in_smem = heap_bytes + SEL_CHUNK * 8 <= (size_t)(c->max_smem_optin - 8 * 1024);
    static const int sel_sync = (getenv("FSLIC_SELSYNC") && atoi(getenv("FSLIC_SELSYNC")) == 0) ? 0 : 1;
    cp.sel_sync = sel_sync;
    if (K + 2 > c->heap_K) return set_err(FSLIC_EINVAL, "K too large for the selection heap");
    c->disp.cca_heap_smem = cp.heap_in_smem ? 1 : 0;
    c->disp.cca_heap_smem_max_k =
        (int)std::max<long>(0, ((long)c->max_smem_optin - 8 * 1024 - SEL_CHUNK * 8) / 8 / 2 - 2);  // (2K+4)*8 fits
    c->disp.cca_sub_batches = ceil_div(batch, c->cca_batch);
    for (int b0 = 0; b0 < batch; b0 += c->cca_batch) {
        const int nb = (batch - b0 < c->cca_batch) ? (batch - b0) : c->cca_batch;
        const uint16_t* in = d_in + (size_t)b0 * N;
        uint16_t* out = d_out + (size_t)b0 * N;
        const bool timed = c->cca_timing && nb < 4 && batch <= c->cca_batch;  // one stream, one sub-batch
        c->cca_timed = timed;
        if (timed) CK(cudaEventRecord(c->cev[0], st));
        CK(cudaMemsetAsync(x_counters, 0, sizeof(CcaCounters) * nb, st));
        CK(cudaMemsetAsync(x_ahist, 0, sizeof(unsigned int) * CCA_HIST * nb, st));
        dim3 g(cp.nblk, nb);
        {
            const int ttx = ceil_div(c->W, CCL_T), tty = ceil_div(c->H, CCL_T);
            const long ntt = (long)ttx * tty * nb;
            k_ccl_tile<<<(int)((ntt + CCL_TW - 1) / CCL_TW), 32 * CCL_TW, 0, st>>>(cp, in, x_par, x_aux, ttx, tty, ntt);
        }
        {
            const int seam_px = ((c->W - 1) / CCL_T) * c->H + ((c->H - 1) / CCL_T) * c->W;
            if (seam_px > 0) {
                dim3 gs(ceil_div(seam_px, 256), nb);
                k_ccl_seams<<<gs, 256, 0, st>>>(cp, in, x_par);
            }
        }
        if (timed) CK(cudaEventRecord(c->cev[1], st));
        k_ccl_flatten<<<g, 256, 0, st>>>(cp, in, x_par, x_aux, x_blkcnt, x_rootbuf, x_predbuf, x_chunkinfo);
        k_scan_blocks<<<nb, 1024, 0, st>>>(x_blkcnt, x_blkoff, cp.nblk, cp.nblk, nullptr, 0, 1,
                                           &x_counters[0].ncomp, (int)(sizeof(CcaCounters) / sizeof(int)), nullptr, -1);
        // grids of the per-component walks: sized for full batches (a few CTAs per image); a small batch gets more
        // CTAs per image instead, it is all dependent-load latency there
        const int number_grid = nb >= 8 ? CCA_NUMBER_GRID : std::min(std::max(ceil_div(cp.nblk, 32), CCA_NUMBER_GRID), 64);
        if (b0 == 0) {
            c->disp.cca_split = nb >= 4;
            c->disp.cca_number_nb = ceil_div(cp.nblk, number_grid * (CCA_BLOCK / 32));  // NB of k_ccl_number
        }
        k_ccl_number<<<dim3(number_grid, nb), CCA_BLOCK, 0, st>>>(cp, x_rootbuf, x_aux, x_blkcnt, x_blkoff, x_carea, x_counters,
                                                                      x_ahist);
        if (timed) CK(cudaEventRecord(c->cev[2], st));
        k_cca_threshold<<<nb, 1024, 0, st>>>(cp, x_carea, x_counters, x_ahist);
        if (timed) CK(cudaEventRecord(c->cev[3], st));
        // Everything after the threshold decision depends on the kept set.  For images k_cca_threshold settled
        // that is known now; for the (few) images whose ties need the sequential std::partial_sort replay it
        // is known only after k_cca_select, which keeps a handful of SMs busy for ~1 ms.  So for batches the
        // tail runs twice: for the settled images on a side stream concurrently with the replay, and for the
        // replayed images afterwards.
        auto tail = [&](int which, cudaStream_t ts) {
            CcaParams cq = cp;
            cq.which = which;
            // (blkoff keeps the component number of each block's first root for k_cca_absorb: the kept offsets of the
            // 1024-component chunks go to kblkoff)
            const dim3 gk(std::min(cp.nblk, std::max(CCA_KEPT_GRID, 256 / nb)), nb);
            k_kept_count<<<gk, CCA_BLOCK, 0, ts>>>(cq, x_carea, x_counters, x_blkcnt);
            k_scan_blocks<<<nb, 1024, 0, ts>>>(x_blkcnt, x_kblkoff, cp.nblk, 0, &x_counters[0].ncomp,
                                               (int)(sizeof(CcaCounters) / sizeof(int)), CCA_BLOCK,
                                               &x_counters[0].nkept, (int)(sizeof(CcaCounters) / sizeof(int)),
                                               x_counters, which);
            k_kept_label<<<gk, CCA_BLOCK, 0, ts>>>(cq, x_carea, x_counters, x_kblkoff, x_cnew);
            if (timed) cudaEventRecord(c->cev[4], ts);
            // one warp per 1024-pixel block and its root list; below 4 images, 8 warps per block (all latency there)
            const int nsplit = nb < 4 ? 8 : 1;
            const dim3 ga(ceil_div(cp.nblk * nsplit, CCA_TAIL_WARPS), nb);
            k_cca_absorb<<<ga, 32 * CCA_TAIL_WARPS, 0, ts>>>(cq, x_rootbuf, x_predbuf, x_chunkinfo, x_blkoff, x_counters,
                                                              x_cnew, x_fin, nsplit);
            if (timed) cudaEventRecord(c->cev[5], ts);
            int ob = ceil_div(ceil_div(N, 8), 256);  // 8 pixels per thread on the vector path (any N works: grid-stride)
            if (ob > c->num_sms * 32) ob = c->num_sms * 32;
            dim3 go(ob, nb);
            k_cca_output<<<go, 256, 0, ts>>>(cq, x_par, x_fin, out, x_counters);
            if (timed) cudaEventRecord(c->cev[6], ts);
        };
        const bool split = nb >= 4;
        const bool early = split && ho && batch <= c->cca_batch && nb <= 64;
        if (early) {
            // the host path is synchronous anyway: wait for the threshold decision and read the per-image flags
            CK(cudaMemcpyAsync(x_hcnt, x_counters, sizeof(CcaCounters) * nb, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
        }
        if (split) {
            CK(cudaEventRecord(x_fork, st));
            CK(cudaStreamWaitEvent(x_side, x_fork, 0));
            tail(0, x_side);
            CK(cudaEventRecord(x_join, x_side));
        }
        auto copy_runs = [&](int want) -> int {  // D2H of maximal runs of images whose need_sim flag == want
            int b = 0;
            while (b < nb) {
                if ((x_hcnt[b].need_sim != 0) != (want != 0)) { b++; continue; }
                int e = b;
                while (e < nb && (x_hcnt[e].need_sim != 0) == (want != 0)) e++;
                CK(cudaMemcpyAsync(ho->h_labels + (size_t)b * N, out + (size_t)b * N, (size_t)(e - b) * N * 2,
                                   cudaMemcpyDeviceToHost, ho->out_stream));
                b = e;
            }
            return FSLIC_OK;
        };
        if (early) {
            CK(cudaStreamWaitEvent(ho->out_stream, x_join, 0));
            int rc2 = copy_runs(0);
            if (rc2) return rc2;
        }
        k_cca_select<<<nb, 1024, SEL_CHUNK * 8 + (cp.heap_in_smem ? heap_bytes : 0), st>>>(cp, x_carea, x_counters, x_heap, x_selprof);
        tail(split ? 1 : -1, st);
        if (early) {
            CK(cudaEventRecord(x_tail, st));
            CK(cudaStreamWaitEvent(ho->out_stream, x_tail, 0));
            int rc2 = copy_runs(1);
            if (rc2) return rc2;
            ho->done = true;
        }
        if (split) {
            CK(cudaStreamWaitEvent(st, x_join, 0));
            if (launches) *launches += 5;
        }
        CK(cudaGetLastError());
        if (launches) *launches += 12;
    }
    return FSLIC_OK;
}

extern "C" int fslic_b200_enforce_connectivity(fslic_ctx* c, uint16_t* d_labels, int batch, int K, int min_threshold,
                                               void* stream) {
    int rc = check_batch(c, batch, false);
    if (rc) return rc;
    if (K <= 0) return FSLIC_OK;  // context.cpp:17
    if (K > 65535) return set_err(FSLIC_EINVAL, "K must fit the u16 label type");
    USE_DEVICE(c->device);
    c->disp = DispatchRecord();
    return run_cca(c, d_labels, d_labels, batch, K, min_threshold, (cudaStream_t)stream, nullptr);
}

extern "C" int fslic_b200_debug_heap_select(fslic_ctx* c, const int32_t* d_area, int n, int middle, uint8_t* d_kept,
                                            void* stream) {
    if (!c) return set_err(FSLIC_EINVAL, "ctx is NULL");
    if (middle + 2 > c->heap_K || middle < 1 || n < 1) return set_err(FSLIC_EINVAL, "bad n/middle");
    USE_DEVICE(c->device);
    CK(cudaMemsetAsync(d_kept, 0, n, (cudaStream_t)stream));
    const size_t hb = (size_t)(2 * middle + 4) * 8;
    const int use_smem = hb + SEL_CHUNK * 8 <= (size_t)(c->max_smem_optin - 8 * 1024);
    k_debug_heap_select<<<1, 1024, SEL_CHUNK * 8 + (use_smem ? hb : 0), (cudaStream_t)stream>>>(reinterpret_cast<const uint32_t*>(d_area), n,
                                                                              middle, d_kept, c->heap, use_smem);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// per-slice views of the batched buffers (c->slice = first image of the slice)
#define SL_QUAD(c) ((c)->quad + (size_t)(c)->slice * (c)->N)
#define SL_LABELS(c) ((c)->labels + (size_t)(c)->slice * (c)->N)
#define SL_CINFO(c) ((c)->cinfo + (size_t)(c)->slice * (c)->K)
#define SL_CELLS(c) ((c)->cell_start + (size_t)(c)->slice * ((c)->ncell + 1))
#define SL_ACC(c) ((c)->acc + (size_t)(c)->slice * (c)->K * 4)

// ---- one assign pass (warp kernel, or the generic kernel when the patch cannot live in shared memory) ----
struct PassGeom {
    int R;
    bool fast;
    int OY, OX, TS, tbl_elems;
    size_t smem;
};

static PassGeom pass_geometry(const fslic_ctx* c, int stride) {
    PassGeom g;
    const int S = c->S;
    g.R = AS_R;
    g.OX = S + 31;
    g.OY = S + stride * (g.R - 1);
    // row pitch from a fixed menu so it is a compile-time constant of the kernel (immediate LDS offsets)
    const int need = 2 * g.OX + 1;
    g.TS = need <= 128 ? 128 : need <= 192 ? 192 : need <= 256 ? 256 : need <= 384 ? 384 : 0;
    const long elems = (long)(2 * g.OY + 1) * (g.TS ? g.TS : need);
    g.tbl_elems = (int)(elems < (1L << 30) ? elems : (1L << 30));
    g.smem = align_up((size_t)g.tbl_elems * 2, 16) + AS_STAGE_BYTES;
    g.fast = g.TS != 0 && elems <= SPT_MAX_ELEMS && g.smem <= (size_t)(c->max_smem_optin - 2 * 1024);
    return g;
}

// kernel menu: TS in {128,192,256,384} x (STRIDE 3 + update | STRIDE 1 no update | runtime stride)
template <int TS>
static assign_fn pick_assign_ts(int stride, bool update) {
    if (update) return stride == 3 ? k_assign_warp<TS, 3, true> : k_assign_warp<TS, 0, true>;
    return stride == 1 ? k_assign_warp<TS, 1, false> : k_assign_warp<TS, 0, false>;
}
static assign_fn pick_assign(int TS, int stride, bool update) {
    switch (TS) {
        case 128: return pick_assign_ts<128>(stride, update);
        case 192: return pick_assign_ts<192>(stride, update);
        case 256: return pick_assign_ts<256>(stride, update);
        default: return pick_assign_ts<384>(stride, update);
    }
}

// kernel menu of the TMA-staged kernel: TS in {128,192,256} x (stride 3 + update | stride 1, no update) x TPS in {1,4}
template <int TS>
static assign5_fn pick_assign5_ts(bool update, int tps, bool fuse) {
    if (update && fuse) return tps == 4 ? k_assign5<TS, 3, true, 4, true> : k_assign5<TS, 3, true, 1, true>;
    if (update) return tps == 4 ? k_assign5<TS, 3, true, 4> : k_assign5<TS, 3, true, 1>;
    return tps == 4 ? k_assign5<TS, 1, false, 4> : k_assign5<TS, 1, false, 1>;
}
static assign5_fn pick_assign5(int TS, bool update, int tps, bool fuse) {
    switch (TS) {
        case 128: return pick_assign5_ts<128>(update, tps, fuse);
        case 192: return pick_assign5_ts<192>(update, tps, fuse);
        default: return pick_assign5_ts<256>(update, tps, fuse);
    }
}

// cuTensorMapEncodeTiled through the runtime's driver entry point table (no link against libcuda)
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static encode_tiled_fn tensor_map_encoder() {
    static encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<encode_tiled_fn>(p);
        cudaGetLastError();
    }
    return fn;
}

// 3-D view (x, sub-row, image) of the rows i = rem + sr * stride of a [B][H][W] array of `esize`-byte pixels;
// box = box_w columns x 4 sub-rows x 1 image.  Out-of-range parts of a box read as zero and are not written.
static bool make_subrow_map(CUtensorMap* m, CUtensorMapDataType dt, int esize, void* base, int H, int W, int B, int stride,
                            int rem, int nsub, int box_w) {
    encode_tiled_fn enc = tensor_map_encoder();
    if (!enc) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)nsub, (cuuint64_t)B};
    const cuuint64_t strides[2] = {(cuuint64_t)stride * W * esize, (cuuint64_t)H * W * esize};
    const cuuint32_t box[3] = {(cuuint32_t)box_w, 4u, 1u};
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    unsigned char* p = static_cast<unsigned char*>(base) + (size_t)rem * W * esize;
    return enc(m, dt, 3, p, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int build_patches(fslic_ctx* c, int stride, bool need_sub, float coef, cudaStream_t st, int* launches) {
    // The two patches depend on (S, stride, coef, manhattan) only: consecutive calls with the same parameters reuse them (two
    // launches less per call, four on the sliced host path).  Inside a stream capture they are always rebuilt, so a
    // replayed graph never depends on what an unrelated call left in the buffers.
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    uint32_t coef_bits;
    memcpy(&coef_bits, &coef, 4);
    const bool warm = cap == cudaStreamCaptureStatusNone && c->spt_valid && c->spt_stream == st && c->spt_stride == stride &&
                      c->spt_coef_bits == coef_bits && c->spt_manhattan == c->manhattan && (c->spt_has_sub || !need_sub);
    if (warm) return FSLIC_OK;
    c->spt_valid = true;
    c->spt_stream = st;  // a call on another stream is not ordered after this build: it rebuilds
    c->spt_stride = stride;
    c->spt_coef_bits = coef_bits;
    c->spt_manhattan = c->manhattan;
    c->spt_has_sub = need_sub;
    if (need_sub) {
        const PassGeom g = pass_geometry(c, stride);
        if (g.fast) {
            k_build_sptable<<<64, 256, 0, st>>>(c->sptable, c->S, g.OY, g.OX, g.TS, coef, c->manhattan);
            if (launches) *launches += 1;
        }
    }
    const PassGeom gf = pass_geometry(c, 1);
    if (gf.fast) {
        k_build_sptable<<<64, 256, 0, st>>>(c->sptable + SPT_MAX_ELEMS, c->S, gf.OY, gf.OX, gf.TS, coef, c->manhattan);
        if (launches) *launches += 1;
    }
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// fuse_clusters / fused_out: when the TMA kernel takes an update pass of a small batch, its last CTA also does the
// bookkeeping for the NEXT pass (prepare_in_tail) on these cluster records; *fused_out tells the caller to skip k_prepare.
static int run_assign_pass(fslic_ctx* c, int batch, int stride, int rem, int cfg_stride, int fresh_from, bool update,
                           float coef, cudaStream_t st, int* launches, int variant = -1,
                           const fslic_cluster* d_clusters = nullptr, fslic_cluster* fuse_clusters = nullptr,
                           bool* fused_out = nullptr) {
    if (fused_out) *fused_out = false;
    if (variant == 3 && update) {  // the `preemptive` option (preempt.cuh); its full assign is the ordinary one
        AssignParams ap;
        memset(&ap, 0, sizeof(ap));
        ap.H = c->H; ap.W = c->W; ap.K = c->K; ap.S = c->S; ap.B = batch;
        ap.stride = stride; ap.rem = rem;
        ap.nsub = (c->H - rem + stride - 1) / stride;
        if (ap.nsub <= 0) return FSLIC_OK;
        ap.cfg_stride = cfg_stride; ap.fresh_from = fresh_from;
        ap.G = c->G; ap.cellW = c->cellW; ap.cellH = c->cellH; ap.ncell = c->ncell;
        ap.coef = coef;
        ap.manhattan = c->manhattan;
        const long px = (long)ap.nsub * c->W * batch;
        long grid = (px + 255) / 256;
        if (grid > (long)c->num_sms * 32) grid = (long)c->num_sms * 32;
        const int CW2 = ceil_div(c->W, 2 * c->S), ncell2 = CW2 * ceil_div(c->H, 2 * c->S);
        k_assign_preempt<true><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), d_clusters,
                                                          SL_ACC(c), c->pre_cellmap + (size_t)c->slice * ncell2, CW2, ncell2,
                                                          c->pre_nactive + c->slice);
        record_pass(c, true, 13, 1, grid, 256, px);
        if (launches) *launches += 1;
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    if (variant == 3) variant = -1;
    if (variant == 4) {  // LSC (lsc.cuh): one thread per pixel over the cell grid
        AssignParams ap;
        memset(&ap, 0, sizeof(ap));
        ap.H = c->H; ap.W = c->W; ap.K = c->K; ap.S = c->S; ap.B = batch;
        ap.stride = stride; ap.rem = rem;
        ap.nsub = (c->H - rem + stride - 1) / stride;
        if (ap.nsub <= 0) return FSLIC_OK;
        ap.cfg_stride = cfg_stride; ap.fresh_from = fresh_from;
        ap.G = c->G; ap.cellW = c->cellW; ap.cellH = c->cellH; ap.ncell = c->ncell;
        const long px = (long)ap.nsub * c->W * batch;
        long grid = (px + 255) / 256;
        if (grid > (long)c->num_sms * 32) grid = (long)c->num_sms * 32;
        if (update)
            k_assign_lsc<true><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), c->lsc_feat,
                                                          c->lsc_cf, SL_ACC(c), c->lsc_box);
        else
            k_assign_lsc<false><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), c->lsc_feat,
                                                           c->lsc_cf, SL_ACC(c), c->lsc_box);
        record_pass(c, update, 14, 1, grid, 256, px);
        if (launches) *launches += 1;
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    if (variant >= 0) {  // float-distance variants (realdist.cuh): one thread per pixel over the cell grid
        AssignParams ap;
        memset(&ap, 0, sizeof(ap));
        ap.H = c->H; ap.W = c->W; ap.K = c->K; ap.S = c->S; ap.B = batch;
        ap.stride = stride; ap.rem = rem;
        ap.nsub = (c->H - rem + stride - 1) / stride;
        if (ap.nsub <= 0) return FSLIC_OK;
        ap.cfg_stride = cfg_stride; ap.fresh_from = fresh_from;
        ap.G = c->G; ap.cellW = c->cellW; ap.cellH = c->cellH; ap.ncell = c->ncell;
        ap.coef = coef;
        ap.manhattan = c->manhattan;
        const long px = (long)ap.nsub * c->W * batch;
        long grid = (px + 255) / 256;
        if (grid > (long)c->num_sms * 32) grid = (long)c->num_sms * 32;
        const fslic_cluster* cl = d_clusters;
#define REAL_LAUNCH(V)                                                                                             \
    if (update)                                                                                                    \
        k_assign_real<V, true><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), cl, SL_ACC(c)); \
    else                                                                                                           \
        k_assign_real<V, false><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), cl, SL_ACC(c));
        if (variant == 0) { REAL_LAUNCH(0) } else if (variant == 1) { REAL_LAUNCH(1) } else { REAL_LAUNCH(2) }
#undef REAL_LAUNCH
        record_pass(c, update, 10 + variant, 1, grid, 256, px);
        if (launches) *launches += 1;
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    const PassGeom g = pass_geometry(c, stride);
    AssignParams ap;
    ap.H = c->H; ap.W = c->W; ap.K = c->K; ap.S = c->S; ap.B = batch;
    ap.stride = stride; ap.rem = rem;
    ap.nsub = (c->H - rem + stride - 1) / stride;
    if (ap.nsub <= 0) return FSLIC_OK;
    ap.cfg_stride = cfg_stride; ap.fresh_from = fresh_from;
    ap.G = c->G; ap.cellW = c->cellW; ap.cellH = c->cellH; ap.ncell = c->ncell;
    ap.Ginv = (uint32_t)(((1ull << 32) + (unsigned)c->G - 1) / (unsigned)c->G);
    ap.OY = g.OY; ap.OX = g.OX; ap.TS = g.TS; ap.tbl_elems = g.tbl_elems;
    ap.tiles_x = ceil_div(c->W, 32);
    ap.tiles_y = ceil_div(ap.nsub, g.R);
    ap.ntiles = ap.tiles_x * ap.tiles_y;
    ap.coef = coef;
    ap.manhattan = c->manhattan;  // the warp-tile kernels read the patch built with it; k_assign_generic reads it
    ap.tps = AS_T;
    ap.fuse_prepare = 0;
    // The TMA-staged kernel: row strides of the tensor maps must be multiples of 16 bytes (W % 8 == 0 for the u16
    // labels), the sub-row pitch is an immediate of its patch loads (stride 3 with the update, 1 without), and its
    // per-warp shared blocks must fit beside the patch.  Everything else takes the LDG kernel below.
    bool use5 = g.fast && c->assign_impl == 5 && (c->W % 8) == 0 && g.TS <= 256 && (update ? stride == 3 : stride == 1) &&
                (long)ceil_div(c->W, 32) * ap.tiles_y * batch < (1L << 30) && tensor_map_encoder() != nullptr;
    int warps5 = 0;
    size_t smem5 = 0;
    if (use5) {
        const size_t tblb = align_up((size_t)g.tbl_elems * 2, 128);
        for (int w : {32, 16, 8}) {
            smem5 = tblb + (size_t)w * A5_WBLK;
            if (smem5 <= (size_t)(c->max_smem_optin - 1024)) {
                warps5 = w;
                break;
            }
        }
        if (!warps5) use5 = false;
    }
    if (use5) {
        // super tiles of 4 tiles when that still gives every warp of the grid work and the union list stays well below
        // its 32 slots; single tiles otherwise (single images, small S)
        const double est4 = (double)(2 * c->S + stride * 3 + 1) * (2 * c->S + 128) / ((double)c->S * c->S);
        const long supers4 = (long)ceil_div(ap.tiles_x, 4) * ap.tiles_y * batch;
        const int tps = (est4 <= 24.0 && supers4 >= (long)c->num_sms * warps5) ? 4 : 1;
        ap.tps = tps;
        CUtensorMap tmq, tml;
        uint32_t* qbase = SL_QUAD(c);
        uint16_t* lbase = SL_LABELS(c);
        if (!make_subrow_map(&tmq, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, qbase, c->H, c->W, batch, stride, rem, ap.nsub, 32 * tps) ||
            !make_subrow_map(&tml, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, lbase, c->H, c->W, batch, stride, rem, ap.nsub, 32 * tps)) {
            use5 = false;
        } else {
            const uint16_t* tbl = c->sptable + (update ? 0 : SPT_MAX_ELEMS);
            const long supers = (long)ceil_div(ap.tiles_x, tps) * ap.tiles_y * batch;
            // Super tiles are handed out statically, so a launch lasts ceil(supers / warps) rounds: with ~4 rounds (720p x 32)
            // a full grid of 32-warp CTAs idles a fifth of the time in the last round.  The kernel is issue bound and
            // saturates an SM with fewer warps, so take the warp count (>= 3/4 of the maximum) that wastes the least.
            if (supers > (long)c->num_sms * warps5) {
                int best_w = warps5;
                double best_cost = 1e30;
                for (int w = warps5; w >= (warps5 * 3) / 4; w--) {
                    const long workers = (long)c->num_sms * w;
                    const double cost = (double)((supers + workers - 1) / workers) * w;  // rounds x warps sharing an SM
                    if (cost < best_cost * 0.995) {
                        best_cost = cost;
                        best_w = w;
                    }
                }
                warps5 = best_w;
                smem5 = align_up((size_t)g.tbl_elems * 2, 128) + (size_t)warps5 * A5_WBLK;
            }
            else if (supers < (long)c->num_sms * warps5) {
                // not even one super tile per warp (single images): spread them over all SMs instead of filling a few
                const int w = std::max(4, (int)ceil_div((int)supers, c->num_sms));
                if (w < warps5) {
                    warps5 = w;
                    smem5 = align_up((size_t)g.tbl_elems * 2, 128) + (size_t)warps5 * A5_WBLK;
                }
            }
            static const bool fuse_allowed = !(getenv("FSLIC_FUSE") && atoi(getenv("FSLIC_FUSE")) == 0);
            const size_t tail_smem = prepare_tail_smem_bytes(c->K, c->ncell);
            if (update && fuse_clusters && fused_out && fuse_allowed && batch <= 2 && c->K <= 4096 &&
                tail_smem <= (size_t)(c->max_smem_optin - 1024)) {
                ap.fuse_prepare = 1;
                if (smem5 < tail_smem) smem5 = tail_smem;
                *fused_out = true;
                c->disp.fused++;
            }
            const assign5_fn fn = pick_assign5(g.TS, update, tps, ap.fuse_prepare != 0);
            long grid = (supers + warps5 - 1) / warps5;
            if (grid > c->num_sms) grid = c->num_sms;
            // the warp-uniform walk constants (constant bank; see the note on code generation in assign5.cuh)
            ap.stx = ceil_div(ap.tiles_x, tps);
            ap.per_img = ap.stx * ap.tiles_y;
            ap.total = (int)supers;
            ap.wstride = (int)grid * warps5;
            ap.db = ap.wstride / ap.per_img;
            ap.dty = (ap.wstride % ap.per_img) / ap.stx;
            ap.dsx = (ap.wstride % ap.per_img) % ap.stx;
            ap.tbl_bytes = (uint32_t)align_up((size_t)g.tbl_elems * 2, 128);
            ap.cinfo_img_bytes = (uint32_t)c->K * (uint32_t)sizeof(CInfo);
            ap.cells_img_bytes = (uint32_t)(c->ncell + 1) * 4u;
            ap.acc_img_bytes = (uint32_t)c->K * 32u;
            cudaEvent_t e0 = nullptr, e1 = nullptr;
            if (c->kev_on && update) {
                while ((int)c->kev.size() < c->kev_used + 2) {
                    cudaEvent_t e;
                    CK(cudaEventCreate(&e));
                    c->kev.push_back(e);
                }
                e0 = c->kev[c->kev_used++];
                e1 = c->kev[c->kev_used++];
                CK(cudaEventRecord(e0, st));
            }
            fn<<<(int)grid, 32 * warps5, smem5, st>>>(ap, tmq, tml, qbase, lbase, SL_CINFO(c), SL_CELLS(c), SL_ACC(c), tbl,
                                                      fuse_clusters, SL_CINFO(c), SL_CELLS(c), c->prep_tickets + c->slice);
            if (e1) CK(cudaEventRecord(e1, st));
            record_pass(c, update, 5, tps, grid, warps5, supers);
        }
    }
    if (use5) {
        // launched above
    } else if (g.fast) {
        const uint16_t* tbl = c->sptable + (update ? 0 : SPT_MAX_ELEMS);
        const assign_fn fn = pick_assign(g.TS, stride, update);
        int occ = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, AS_THREADS, g.smem);
        if (occ < 1) occ = 1;
        long grid = (long)c->num_sms * occ;
        // small launches (single images): one tile per warp step so that every SM gets work
        ap.tps = ((long)ap.ntiles * batch < (long)c->num_sms * occ * AS_WARPS * AS_T) ? 1 : AS_T;
        const long supers = (long)ceil_div(ap.tiles_x, ap.tps) * ap.tiles_y * batch;
        const long need = (supers + AS_WARPS - 1) / AS_WARPS;
        if (grid > need) grid = need;
        cudaEvent_t e0 = nullptr, e1 = nullptr;
        if (c->kev_on && update) {
            while ((int)c->kev.size() < c->kev_used + 2) {
                cudaEvent_t e;
                CK(cudaEventCreate(&e));
                c->kev.push_back(e);
            }
            e0 = c->kev[c->kev_used++];
            e1 = c->kev[c->kev_used++];
            CK(cudaEventRecord(e0, st));
        }
        fn<<<(int)grid, AS_THREADS, g.smem, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), SL_ACC(c), tbl);
        if (e1) CK(cudaEventRecord(e1, st));
        record_pass(c, update, 4, ap.tps, grid, AS_WARPS, supers);
    } else {
        const long px = (long)ap.nsub * c->W * batch;
        long grid = (px + 255) / 256;
        if (grid > (long)c->num_sms * 64) grid = (long)c->num_sms * 64;
        record_pass(c, update, 0, 1, grid, 256, px);
        if (update)
            k_assign_generic<true><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c),
                                                              SL_ACC(c));
        else
            k_assign_generic<false><<<(int)grid, 256, 0, st>>>(ap, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c),
                                                               SL_ACC(c));
    }
    if (launches) *launches += 1;
    CK(cudaGetLastError());
    return FSLIC_OK;
}

static int run_prepare(fslic_ctx* c, fslic_cluster* d_clusters, int batch, int first, int finalize, cudaStream_t st,
                       int* launches, int noq = 0, int preempt = 0, int last = 0) {
    PrepParams pp;
    pp.H = c->H; pp.W = c->W; pp.K = c->K; pp.S = c->S; pp.T = 2 * c->S + 32;
    pp.G = c->G; pp.cellW = c->cellW; pp.cellH = c->cellH; pp.ncell = c->ncell;
    pp.first = first; pp.finalize = finalize; pp.last = last; pp.noq = noq;
    pp.preempt = preempt; pp.l1_thres = c->preempt_l1; pp.nactive = preempt ? c->pre_nactive + c->slice : nullptr;
    const size_t smem = (size_t)(c->ncell + 2) * sizeof(int);
    if (preempt) {  // k_prepare carries the option's bookkeeping; after an update k_preempt_mark derives the active set
        k_prepare<<<batch, 1024, smem, st>>>(pp, d_clusters, SL_ACC(c), SL_QUAD(c), SL_CINFO(c), SL_CELLS(c),
                                             c->cinfo_tmp + (size_t)c->slice * c->K);
        c->disp.prepare = 1;
        if (launches) *launches += 1;
        if (finalize && !last) {
            const int CW2 = ceil_div(c->W, 2 * c->S), ncell2 = CW2 * ceil_div(c->H, 2 * c->S);
            k_preempt_mark<<<batch, 1024, 0, st>>>(c->K, c->S, c->H, c->W, c->G, c->cellW, c->cellH, c->ncell, d_clusters, SL_CINFO(c),
                                                   SL_CELLS(c), c->pre_cellmap + (size_t)c->slice * ncell2, CW2, ncell2,
                                                   c->pre_nactive + c->slice);
            if (launches) *launches += 1;
        }
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    // k_prepare2 (one thread per cluster, several CTAs per image) is quicker for a handful of images (single image:
    // 0.412 vs 0.431 ms per blocking call); with a full batch its extra CTAs only contend (18 vs 13 us at 32 images)
    static const int forced = getenv("FSLIC_PREPARE") ? atoi(getenv("FSLIC_PREPARE")) : 0;
    const bool old_prepare = forced == 1 || (forced != 2 && batch >= 8);
    if (forced != 1 && forced != 2 && c->K <= 1024 * PREP3_PER) {
        k_prepare3<<<batch, 1024, smem, st>>>(pp, d_clusters, SL_ACC(c), SL_QUAD(c), SL_CINFO(c), SL_CELLS(c));
        c->disp.prepare = 3;
    } else if (old_prepare) {
        k_prepare<<<batch, 1024, smem, st>>>(pp, d_clusters, SL_ACC(c), SL_QUAD(c), SL_CINFO(c), SL_CELLS(c),
                                             c->cinfo_tmp + (size_t)c->slice * c->K);
        c->disp.prepare = 1;
    } else {
        k_prepare2<<<dim3(ceil_div(c->K, 256), batch), 256, smem, st>>>(
            pp, d_clusters, SL_ACC(c), SL_QUAD(c), SL_CINFO(c), SL_CELLS(c), c->cinfo_tmp + (size_t)c->slice * c->K,
            c->cell_cnt + (size_t)c->slice * (c->ncell + 1), c->prep_tickets + c->slice);
        c->disp.prepare = 2;
    }
    CK(cudaGetLastError());
    if (launches) *launches += 1;
    return FSLIC_OK;
}

static int check_params(const fslic_ctx* c, const fslic_params* p, float* coef_out) {
    if (!p) return set_err(FSLIC_EINVAL, "params is NULL");
    if (p->subsample_stride <= 0 || p->subsample_stride > 255) return set_err(FSLIC_EINVAL, "subsample_stride must be in 1..255");
    if (p->max_iter < 0) return set_err(FSLIC_EINVAL, "max_iter must be >= 0");
    if (!(p->compactness >= 0.f)) return set_err(FSLIC_EINVAL, "compactness must be >= 0");
    const int S = c->S;
    const int color_shift = p->convert_to_lab ? 1 : 0;  // cielab.h:25,352 / context.cpp:127
    // BaseContext::set_spatial_patch, context.cpp:25-26 (same float operations, same order)
    float coef = 1.0f / ((float)S / p->compactness);
    coef *= (float)(1 << color_shift);
    if (S > 0 && !(coef * (float)(2 * S) < (float)(FSLIC_BIGSP - 766)))
        return set_err(FSLIC_ERANGE, "compactness too large: the u16 distance of the reference would overflow");
    if (S == 0) coef = 0.f;  // 1/(0/compactness) = inf in the reference; with S == 0 only m = 0 is ever used -> inf*0 = NaN -> (u16) UB; use 0
    *coef_out = coef;
    return FSLIC_OK;
}

// ---- LSC (lsc.cuh) -----------------------------------------------------------------------------------------------
// The feature tables of ContextLSC::map_image_into_feature_space (lsc.cpp:25-28, 69-101), computed with the libm calls
// of the reference's object code: glibc's double sincos of a float angle (GCC merges each sin / cos pair into one call);
// the colour tables round the cosine / sine to float and multiply in float, the others multiply in double.  Bit-identical
// to the reference's as long as this machine's glibc computes the same double sin / cos (DESIGN.md section 4.9).
static void build_lsc_tables(int H, int W, int S, float compactness, std::vector<float>& tab) {
    tab.assign(LSC_TAB_FIXED + 2 * (size_t)W + 2 * (size_t)H, 0.f);
    const float PI = (float)3.1415926;
    const float halfPI = PI / 2;
    const float ratio = compactness / 100.0f;
    const float C_color = 20.0f;  // lsc.h:8
    const float C_spatial = C_color * ratio;
    double s, co;
    for (int X = 0; X < 256; X++) {
        const float theta = halfPI * ((float)X / 255.0f);
        sincos((double)theta, &s, &co);
        const float cosine = (float)co, sine = (float)s;
        tab[512 + X] = C_color * cosine * 2.55f;
        tab[768 + X] = C_color * sine * 2.55f;
        tab[X] = (float)((double)C_color * co);
        tab[256 + X] = (float)((double)C_color * s);
    }
    const float step = halfPI / (float)S;
    for (int j = 0; j < W; j++) {
        sincos((double)((float)j * step), &s, &co);
        tab[LSC_TAB_FIXED + j] = (float)((double)C_spatial * co);
        tab[LSC_TAB_FIXED + W + j] = (float)((double)C_spatial * s);
    }
    for (int i = 0; i < H; i++) {
        sincos((double)((float)i * step), &s, &co);
        tab[LSC_TAB_FIXED + 2 * W + i] = (float)((double)C_spatial * co);
        tab[LSC_TAB_FIXED + 2 * W + H + i] = (float)((double)C_spatial * s);
    }
}

static int ensure_lsc(fslic_ctx* c) {
    if (c->lsc_feat) return FSLIC_OK;
    const size_t B = (size_t)c->maxB, N = (size_t)c->N, K = (size_t)c->K;
    float *feat = nullptr, *w = nullptr, *tab = nullptr, *means = nullptr, *cf = nullptr, *cfi = nullptr;
    LscBox* box = nullptr;
    if (dalloc(&feat, B * LSC_NF * N) != cudaSuccess || dalloc(&w, B * N) != cudaSuccess ||
        dalloc(&tab, LSC_TAB_FIXED + 2 * (size_t)c->W + 2 * (size_t)c->H) != cudaSuccess ||
        dalloc(&means, B * LSC_NF) != cudaSuccess || dalloc(&cf, B * K * LSC_CF) != cudaSuccess ||
        dalloc(&cfi, B * K * LSC_NF) != cudaSuccess || dalloc(&box, B * K) != cudaSuccess) {
        for (void* p : {(void*)feat, (void*)w, (void*)tab, (void*)means, (void*)cf, (void*)cfi, (void*)box})
            if (p) cudaFree(p);
        cudaGetLastError();
        return set_err(FSLIC_ENOMEM, "out of device memory (LSC scratch)");
    }
    c->lsc_feat = feat; c->lsc_w = w; c->lsc_tab = tab; c->lsc_means = means; c->lsc_cf = cf; c->lsc_cf_init = cfi;
    c->lsc_box = box;
    c->lsc_tab_valid = false;
    return FSLIC_OK;
}

// before_iteration (lsc.cpp:12-15): tables, feature means, weights and normalised features, initial centroid features.
// Runs after the Lab kernel and before the first prepare, which clamps the centres (context.cpp:209-212) that
// map_centroids_into_feature_space reads unclamped.
static int lsc_before_iteration(fslic_ctx* c, const fslic_cluster* d_clusters, int batch, const fslic_params* p,
                                cudaStream_t st, int* launches) {
    uint32_t key;
    memcpy(&key, &p->compactness, 4);
    if (!c->lsc_tab_valid || key != c->lsc_tab_key) {
        build_lsc_tables(c->H, c->W, c->S, p->compactness, c->lsc_htab);
        // pageable source: the copy is staged before cudaMemcpyAsync returns, so the vector may change afterwards
        CK(cudaMemcpyAsync(c->lsc_tab, c->lsc_htab.data(), c->lsc_htab.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        c->lsc_tab_key = key;
        c->lsc_tab_valid = true;
    }
    k_lsc_means<<<batch * LSC_NF, 32, 0, st>>>(SL_QUAD(c), c->lsc_tab, c->H, c->W, c->lsc_means);
    const long px = (long)c->N * batch;
    long grid = (px + 255) / 256;
    if (grid > (long)c->num_sms * 32) grid = (long)c->num_sms * 32;
    k_lsc_features<<<(int)grid, 256, 0, st>>>(SL_QUAD(c), c->lsc_tab, c->H, c->W, batch, c->lsc_means, c->lsc_feat, c->lsc_w);
    c->disp.lsc_trips = (int)((px + grid * 256 - 1) / (grid * 256));
    k_lsc_centroids<<<ceil_div(batch * c->K, 256), 256, 0, st>>>(c->lsc_feat, c->H, c->W, c->K, c->S, batch, d_clusters,
                                                                 c->lsc_cf, c->lsc_cf_init, c->lsc_box);
    if (launches) *launches += 3;
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// after_update (lsc.cpp:226-307) of the pass just assigned; timed launch by launch when collect_timing is on.
static int lsc_after_update(fslic_ctx* c, int batch, int stride, cudaStream_t st, int* launches, bool timing) {
    cudaEvent_t e1 = nullptr;
    if (timing) {
        while ((int)c->lev.size() < c->lev_used + 2) {
            cudaEvent_t e;
            CK(cudaEventCreate(&e));
            c->lev.push_back(e);
        }
        CK(cudaEventRecord(c->lev[c->lev_used++], st));
        e1 = c->lev[c->lev_used++];
    }
    k_lsc_after_update<<<ceil_div(batch * c->K, LSC_AU_WARPS), LSC_AU_WARPS * 32, 0, st>>>(
        c->H, c->W, c->K, batch, stride, SL_LABELS(c), c->lsc_feat, c->lsc_w, c->lsc_cf, c->lsc_box);
    if (e1) CK(cudaEventRecord(e1, st));
    if (launches) *launches += 1;
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// ---- debug_mode tracing (trace.cuh) -------------------------------------------------------------------------------
// Snapshot s of image b (s = 0 is the reference's iteration -1, s = i + 1 its iteration i) lives in slot b * T + s of
// three regions of one allocation: clusters [B][T][K], min_dists [B][T][N] (u16 or float), assignment [B][T][N].
static fslic_cluster* tr_clusters(const fslic_ctx* c) { return static_cast<fslic_cluster*>(c->tr_buf); }
static char* tr_dist(const fslic_ctx* c) {
    return static_cast<char*>(c->tr_buf) + (size_t)c->tr_B * c->tr_T * c->K * sizeof(fslic_cluster);
}
static uint16_t* tr_assign(const fslic_ctx* c) {
    return reinterpret_cast<uint16_t*>(tr_dist(c) + (size_t)c->tr_B * c->tr_T * c->N * c->tr_dist_bytes);
}

// Sizes the snapshot buffers for this call (they grow, never shrink) and clears the self-check counter.
static int trace_begin(fslic_ctx* c, int batch, int max_iter, int variant, cudaStream_t st) {
    c->tr_T = 0;
    const int T = max_iter + 1, db = (variant >= 0 && variant <= 2) || variant == 4 ? 4 : 2;  // float contexts: float distances
    const size_t need = (size_t)T * batch * ((size_t)c->K * sizeof(fslic_cluster) + (size_t)c->N * (2 + db));
    if (!c->tr_bad && cudaMalloc(reinterpret_cast<void**>(&c->tr_bad), sizeof(unsigned int)) != cudaSuccess) {
        c->tr_bad = nullptr;
        cudaGetLastError();
        return set_err(FSLIC_ENOMEM, "out of device memory (trace counter)");
    }
    if (need > c->tr_cap) {
        if (c->tr_buf) cudaFree(c->tr_buf);
        c->tr_buf = nullptr;
        c->tr_cap = 0;
        if (cudaMalloc(&c->tr_buf, need) != cudaSuccess) {
            c->tr_buf = nullptr;
            cudaGetLastError();
            return set_err(FSLIC_ENOMEM, "out of device memory (" + std::to_string(need >> 20) + " MiB of debug_mode snapshots)");
        }
        c->tr_cap = need;
    }
    c->tr_T = T;
    c->tr_B = batch;
    c->tr_dist_bytes = db;
    CK(cudaMemsetAsync(c->tr_bad, 0, sizeof(unsigned int), st));
    return FSLIC_OK;
}

// Snapshot -1: assignment all 0xFFFF (context.cpp:140-145), min_dists all 0 (a fresh context's calloc'd array,
// simd-helper.hpp:65), the cluster records of k_trace_seed.
static int trace_seed(fslic_ctx* c, const fslic_cluster* d_clusters, int batch, cudaStream_t st, int* launches) {
    const size_t N = c->N, T = c->tr_T;
    k_trace_seed<<<ceil_div(batch * c->K, 256), 256, 0, st>>>(c->H, c->W, c->K, batch, SL_QUAD(c), d_clusters, tr_clusters(c),
                                                             (long long)T * c->K);
    CK(cudaGetLastError());
    CK(cudaMemset2DAsync(tr_assign(c), T * N * 2, 0xFF, N * 2, batch, st));
    CK(cudaMemset2DAsync(tr_dist(c), T * N * c->tr_dist_bytes, 0, N * c->tr_dist_bytes, batch, st));
    (*launches)++;
    return FSLIC_OK;
}

// Assignment and minimum distances after update pass `it` (slot it + 1), from the records that pass read.  Runs before
// the next prepare rewrites them and, for LSC, before after_update.
static int trace_pass(fslic_ctx* c, int batch, int it, int stride, int rem, float coef, int variant,
                      const fslic_cluster* d_clusters, cudaStream_t st, int* launches) {
    TraceParams tp;
    memset(&tp, 0, sizeof(tp));
    AssignParams& ap = tp.ap;
    ap.H = c->H; ap.W = c->W; ap.K = c->K; ap.S = c->S; ap.B = batch;
    ap.stride = stride; ap.rem = rem; ap.cfg_stride = stride;
    ap.G = c->G; ap.cellW = c->cellW; ap.cellH = c->cellH; ap.ncell = c->ncell;
    ap.coef = coef;
    ap.manhattan = c->manhattan;
    tp.fresh_after = it + 1;
    tp.preempt = variant == 3;
    tp.img_pitch = (long long)c->tr_T * c->N;
    tp.feat = c->lsc_feat;
    tp.cf = c->lsc_cf;
    const size_t slot = (size_t)(it + 1) * c->N;
    uint16_t* oa = tr_assign(c) + slot;
    void* od = tr_dist(c) + slot * c->tr_dist_bytes;
    const long px = (long)c->N * batch;
    long grid = (px + 255) / 256;
    if (grid > (long)c->num_sms * 32) grid = (long)c->num_sms * 32;
#define TRACE_LAUNCH(KIND) \
    k_trace_pass<KIND><<<(int)grid, 256, 0, st>>>(tp, SL_QUAD(c), SL_LABELS(c), SL_CINFO(c), SL_CELLS(c), d_clusters, oa, od, c->tr_bad)
    if (variant == 0) TRACE_LAUNCH(0);
    else if (variant == 1) TRACE_LAUNCH(1);
    else if (variant == 2) TRACE_LAUNCH(2);
    else if (variant == 4) TRACE_LAUNCH(4);
    else TRACE_LAUNCH(-1);
#undef TRACE_LAUNCH
    CK(cudaGetLastError());
    (*launches)++;
    return FSLIC_OK;
}

// The cluster records after update `slot - 1`, i.e. after the prepare that finalised it (division, clamp, preemptive
// bookkeeping; capi.cu splits the reference's update() across the assign kernel and that prepare).
static int trace_clusters(fslic_ctx* c, const fslic_cluster* d_clusters, int batch, int slot, cudaStream_t st) {
    const size_t rec = (size_t)c->K * sizeof(fslic_cluster);
    CK(cudaMemcpy2DAsync(tr_clusters(c) + (size_t)slot * c->K, rec * c->tr_T, d_clusters, rec, rec, batch,
                         cudaMemcpyDeviceToDevice, st));
    return FSLIC_OK;
}

// Front half of iterate (context.cpp:114-181): Lab LUT, max_iter x (assign + update), full assign, for the
// `batch` images starting at image `b0` of the context's buffers.  Leaves the pre-CCA labels in c->labels.
static int iterate_front(fslic_ctx* c, int b0, const uint8_t* d_images, fslic_cluster* d_clusters, int batch,
                         const fslic_params* p, float coef, cudaStream_t st, int* launches, bool timing,
                         bool lab_done = false, int variant = -1) {
    c->slice = b0;
    int rc = FSLIC_OK;
    if (!lab_done) rc = launch_lab(c, d_images, SL_QUAD(c), batch, p->convert_to_lab, st);  // else: the caller ran it
    if (rc) return rc;
    (*launches)++;
    if (timing) CK(cudaEventRecord(c->ev[1], st));
    if (variant == 4) {  // LSC: before_iteration (context.cpp:151-154)
        rc = lsc_before_iteration(c, d_clusters, batch, p, st, launches);
        if (rc) return rc;
        if (timing) CK(cudaEventRecord(c->ev[5], st));
    }
    const int stride = p->subsample_stride;
    const int noq = variant == 2 ? 1 : 0;
    const int preempt = variant == 3 ? 1 : 0;
    if (variant < 0 || preempt) {
        rc = build_patches(c, stride, p->max_iter > 0, coef, st, launches);
        if (rc) return rc;
    }
    const fslic_cluster* cl = d_clusters;  // the NoQ variant reads its float centroids from the cluster records themselves
    // debug_mode: snapshots between the stages below; a traced call never fuses the next prepare into an assign tail
    const bool trace = c->trace_on;
    if (trace) {
        rc = trace_seed(c, d_clusters, batch, st, launches);
        if (rc) return rc;
    }
    int rem = 0;
    bool prepared = false;  // the previous assign+update launch already did the bookkeeping in its tail
    for (int it = 0; it < p->max_iter; it++) {
        if (!prepared) {
            rc = run_prepare(c, d_clusters, batch, it == 0, it > 0, st, launches, noq, preempt, 0);
            if (rc) return rc;
            if (trace && it > 0) rc = trace_clusters(c, d_clusters, batch, it, st);
            if (rc) return rc;
        }
        rc = run_assign_pass(c, batch, stride, rem, stride, it, true, coef, st, launches, variant, cl,
                             variant < 0 && !trace ? d_clusters : nullptr, &prepared);
        if (rc) return rc;
        if (trace) {
            rc = trace_pass(c, batch, it, stride, rem, coef, variant, d_clusters, st, launches);
            if (rc) return rc;
        }
        if (variant == 4) {  // LSC: after_update (context.cpp:169-172); its Cluster update is the next prepare's
            rc = lsc_after_update(c, batch, stride, st, launches, timing);
            if (rc) return rc;
        }
        rem = (rem + 1) % stride;
    }
    if (timing) CK(cudaEventRecord(c->ev[2], st));
    if (!prepared) {
        // The last snapshot precedes PreemptiveGrid::finalize (context.cpp:173-176): a traced `preemptive` call lets this
        // prepare derive the final update's active set like the earlier ones, records it, then sets every is_active.
        const bool hold = trace && preempt && p->max_iter > 0;
        rc = run_prepare(c, d_clusters, batch, p->max_iter == 0, p->max_iter > 0, st, launches, noq, preempt, hold ? 0 : 1);
        if (rc) return rc;
        if (trace && p->max_iter > 0) rc = trace_clusters(c, d_clusters, batch, p->max_iter, st);
        if (rc) return rc;
        if (hold) {
            k_trace_activate<<<ceil_div(batch * c->K, 256), 256, 0, st>>>(d_clusters, batch * c->K);
            CK(cudaGetLastError());
            (*launches)++;
        }
    }
    rc = run_assign_pass(c, batch, 1, 0, stride, p->max_iter < stride ? p->max_iter : stride, false, coef, st, launches,
                         variant, cl);
    c->slice = 0;
    return rc;
}

// Back half (context.cpp:191-194): connectivity enforcement of images [0, batch) of c->labels into d_labels.
static int iterate_back(fslic_ctx* c, uint16_t* d_labels, int batch, const fslic_params* p, cudaStream_t st, int* launches,
                        HostOut* ho = nullptr, int slot = 0, int lane = 0) {
    const int thres = (int)round((double)(c->S * c->S) * (double)p->min_size_factor);  // context.cpp:16
    return run_cca(c, c->labels + (size_t)slot * c->N, d_labels, batch, c->K, thres, st, launches, ho, slot, lane);
}

static int iterate_graphed(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels, int batch,
                           const fslic_params* p, cudaStream_t st);

static int iterate_plain(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                         int batch, const fslic_params* p, void* stream, bool lab_done = false, int variant = -1) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    float coef;
    rc = check_params(c, p, &coef);
    if (rc) return rc;
    USE_DEVICE(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    int launches = 0;
    c->disp = DispatchRecord();
    const bool timing = p->collect_timing != 0;
    c->kev_on = p->collect_timing >= 2;
    c->kev_used = 0;
    c->lev_used = 0;
    c->cca_timing = timing;
    c->cca_timed = false;
    if (c->trace_on) {
        rc = trace_begin(c, batch, p->max_iter, variant, st);
        if (rc) return rc;
    }
    if (timing) CK(cudaEventRecord(c->ev[0], st));
    rc = iterate_front(c, 0, d_images, d_clusters, batch, p, coef, st, &launches, timing, lab_done, variant);
    if (rc) return rc;
    if (timing) CK(cudaEventRecord(c->ev[3], st));
    rc = iterate_back(c, d_labels, batch, p, st, &launches);
    if (rc) return rc;
    if (timing) {
        CK(cudaEventRecord(c->ev[4], st));
        CK(cudaEventSynchronize(c->ev[4]));
        float ms;
        CK(cudaEventElapsedTime(&ms, c->ev[0], c->ev[1])); c->stage_ms[FSLIC_T_CIELAB] = ms;
        CK(cudaEventElapsedTime(&ms, c->ev[1], c->ev[2])); c->stage_ms[FSLIC_T_ASSIGN] = ms;
        c->stage_ms[FSLIC_T_UPDATE] = 0.f;  // fused into assign
        c->stage_ms[FSLIC_T_BEFORE_ITERATION] = 0.f;
        c->stage_ms[FSLIC_T_AFTER_UPDATE] = 0.f;
        if (variant == 4) {  // LSC: before_iteration and the after_update launches are their own stages
            CK(cudaEventElapsedTime(&ms, c->ev[1], c->ev[5])); c->stage_ms[FSLIC_T_BEFORE_ITERATION] = ms;
            CK(cudaEventElapsedTime(&ms, c->ev[5], c->ev[2])); c->stage_ms[FSLIC_T_ASSIGN] = ms;
            for (int i = 0; i + 1 < c->lev_used; i += 2) {
                CK(cudaEventElapsedTime(&ms, c->lev[i], c->lev[i + 1]));
                c->stage_ms[FSLIC_T_AFTER_UPDATE] += ms;
            }
            c->stage_ms[FSLIC_T_ASSIGN] -= c->stage_ms[FSLIC_T_AFTER_UPDATE];
        }
        CK(cudaEventElapsedTime(&ms, c->ev[2], c->ev[3])); c->stage_ms[FSLIC_T_FULL_ASSIGN] = ms;
        CK(cudaEventElapsedTime(&ms, c->ev[3], c->ev[4])); c->stage_ms[FSLIC_T_CCA] = ms;
        CK(cudaEventElapsedTime(&ms, c->ev[0], c->ev[4])); c->stage_ms[FSLIC_T_TOTAL] = ms;
        for (int i = 0; i < 6; i++) {
            c->cca_ms[i] = 0.f;
            if (c->cca_timed && cudaEventElapsedTime(&ms, c->cev[i], c->cev[i + 1]) == cudaSuccess) c->cca_ms[i] = ms;
        }
        cudaGetLastError();
        c->assign_kernel_ms = 0.f;
        c->assign_kernel_launches = 0;
        for (int i = 0; i + 1 < c->kev_used; i += 2) {
            CK(cudaEventElapsedTime(&ms, c->kev[i], c->kev[i + 1]));
            c->assign_kernel_ms += ms;
            c->assign_kernel_launches++;
        }
    }
    c->last_launches = launches;
    c->cca_timing = false;
    return FSLIC_OK;
}

extern "C" int fslic_b200_cca_stage_ms(fslic_ctx* c, float* out_ms, int count) {
    if (!c || !out_ms) return set_err(FSLIC_EINVAL, "NULL argument");
    for (int i = 0; i < count && i < 6; i++) out_ms[i] = c->cca_ms[i];
    return FSLIC_OK;
}

// Public entry.  A small batch is ~45 launches of kernels that each run a few microseconds: when the same buffers,
// batch and parameters come back (second consecutive call) the call is captured into a CUDA graph once and replayed
// from then on.  Needs a capturable stream (not the legacy default stream) and no timing; anything else launches plainly.
extern "C" int fslic_b200_iterate(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                                  int batch, const fslic_params* p, void* stream) {
    // A traced call launches plainly and leaves the graph and its key alone: the next untraced call replays as before.
    if (c && p && c->graphs_enabled && !c->trace_on && batch > 0 && batch < 4 && p->collect_timing == 0 && stream != nullptr) {
        fslic_ctx::GraphKey k;
        memset(&k, 0, sizeof(k));
        k.img = nullptr; k.cl = d_clusters; k.lab = d_labels; k.batch = batch; k.p = *p; k.manhattan = c->manhattan;
        const bool have = c->gexec && memcmp(&k, &c->gkey, sizeof(k)) == 0;
        const bool again = memcmp(&k, &c->gkey_seen, sizeof(k)) == 0;
        memcpy(&c->gkey_seen, &k, sizeof(k));
        if (have || again) return iterate_graphed(c, d_images, d_clusters, d_labels, batch, p, (cudaStream_t)stream);
    }
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream);
}

// The float-distance contexts of the reference (context.h:100-125; cfast_slic.pyx:198-252): variant 0 = ContextRealDist
// ("standard"), 1 = ContextRealDistL2, 2 = ContextRealDistNoQ; c->manhattan selects the spatial term of variants 0 and 2.
extern "C" int fslic_b200_iterate_real(fslic_ctx* c, int variant, const uint8_t* d_images, fslic_cluster* d_clusters,
                                       uint16_t* d_labels, int batch, const fslic_params* p, void* stream) {
    if (variant < 0 || variant > 2) return set_err(FSLIC_EINVAL, "variant must be 0 (standard), 1 (l2) or 2 (noq)");
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream, false, variant);
}

// The reference's ContextLSC (src/lsc.cpp; cfast_slic.pyx:207-214) driven with num_threads = 1 (lsc.cuh).
extern "C" int fslic_b200_iterate_lsc(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                                      int batch, const fslic_params* p, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    rc = ensure_lsc(c);
    if (rc) return rc;
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream, false, 4);
}

extern "C" int fslic_b200_debug_lsc_stages(fslic_ctx* c, float* d_means_out, float* d_weights_out, float* d_cinit_out,
                                           int batch, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    if (!c->lsc_feat) return set_err(FSLIC_EINVAL, "no LSC iterate has run on this context");
    USE_DEVICE(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (d_means_out)
        CK(cudaMemcpyAsync(d_means_out, c->lsc_means, sizeof(float) * LSC_NF * batch, cudaMemcpyDeviceToDevice, st));
    if (d_weights_out)
        CK(cudaMemcpyAsync(d_weights_out, c->lsc_w, sizeof(float) * (size_t)c->N * batch, cudaMemcpyDeviceToDevice, st));
    if (d_cinit_out)
        CK(cudaMemcpyAsync(d_cinit_out, c->lsc_cf_init, sizeof(float) * LSC_NF * (size_t)c->K * batch,
                           cudaMemcpyDeviceToDevice, st));
    return FSLIC_OK;
}

extern "C" int fslic_b200_iterate_preemptive(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                                             int batch, const fslic_params* p, float preemptive_thres, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    if (c->S <= 0) return set_err(FSLIC_EINVAL, "preemptive needs S >= 1 (the reference divides by 2 S, preemptive.h:37-38)");
    if (!(preemptive_thres >= 0.f)) return set_err(FSLIC_EINVAL, "preemptive_thres must be >= 0");
    USE_DEVICE(c->device);
    if (!c->pre_cellmap) {
        const size_t ncell2 = (size_t)ceil_div(c->W, 2 * c->S) * ceil_div(c->H, 2 * c->S);
        uint8_t* cm = nullptr;
        int* na = nullptr;
        if (cudaMalloc(reinterpret_cast<void**>(&cm), ncell2 * c->maxB) != cudaSuccess ||
            cudaMalloc(reinterpret_cast<void**>(&na), sizeof(int) * c->maxB) != cudaSuccess) {
            if (cm) cudaFree(cm);
            cudaGetLastError();
            return set_err(FSLIC_ENOMEM, "out of device memory (preemptive scratch)");
        }
        c->pre_cellmap = cm;
        c->pre_nactive = na;
    }
    c->preempt_l1 = fmaxf(roundf((float)(2 * c->S) * preemptive_thres), 1.0f);  // preemptive.h:126
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream, false, 3);
}

extern "C" int fslic_b200_assign_kernel_time(fslic_ctx* c, float* total_ms, int* launches) {
    if (!c || !total_ms || !launches) return set_err(FSLIC_EINVAL, "NULL argument");
    *total_ms = c->assign_kernel_ms;
    *launches = c->assign_kernel_launches;
    return FSLIC_OK;
}

extern "C" int fslic_b200_debug_cca_counters(fslic_ctx* c, int32_t* out8, int image) {
    if (!c || !out8 || image < 0 || image >= c->cca_batch) return set_err(FSLIC_EINVAL, "bad argument");
    USE_DEVICE(c->device);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out8, c->counters + image, sizeof(CcaCounters), cudaMemcpyDeviceToHost));
    return FSLIC_OK;
}

extern "C" int fslic_b200_debug_select_profile(fslic_ctx* c, long long* out8, int image) {
    if (!c || !out8 || image < 0 || image >= c->cca_batch) return set_err(FSLIC_EINVAL, "bad argument");
    if (!c->selprof) return set_err(FSLIC_EINVAL, "the context was created without FSLIC_SELPROF=1");
    USE_DEVICE(c->device);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out8, c->selprof + 8 * image, 8 * sizeof(long long), cudaMemcpyDeviceToHost));
    return FSLIC_OK;
}

extern "C" int fslic_b200_stage_ms(fslic_ctx* c, float* out_ms, int count) {
    if (!c || !out_ms) return set_err(FSLIC_EINVAL, "NULL argument");
    for (int i = 0; i < count && i < FSLIC_T_COUNT; i++) out_ms[i] = c->stage_ms[i];
    return FSLIC_OK;
}

extern "C" int fslic_b200_debug_stages(fslic_ctx* c, uint8_t* d_quad_out, uint16_t* d_precca_out, int batch,
                                       void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (d_quad_out) CK(cudaMemcpyAsync(d_quad_out, c->quad, (size_t)batch * c->N * 4, cudaMemcpyDeviceToDevice, st));
    if (d_precca_out) CK(cudaMemcpyAsync(d_precca_out, c->labels, (size_t)batch * c->N * 2, cudaMemcpyDeviceToDevice, st));
    return FSLIC_OK;
}

// ---- host-buffer entry points (what the reference-facing plugin calls) --------------------------
static int ensure_staging(fslic_ctx* c) {
    if (c->d_img && c->d_cl && c->d_lab) return FSLIC_OK;
    const size_t B = (size_t)c->maxB, N = (size_t)c->N;
    // allocate into temporaries and commit all three together: a failed second or third allocation must not
    // leave a half-initialised staging set behind for the next call to trip over
    uint8_t* img = nullptr;
    fslic_cluster* cl = nullptr;
    uint16_t* lab = nullptr;
    cudaError_t e = dalloc(&img, B * N * 3);
    if (e == cudaSuccess) e = dalloc(&cl, B * c->K);
    if (e == cudaSuccess) e = dalloc(&lab, B * N);
    if (e != cudaSuccess) {
        if (img) cudaFree(img);
        if (cl) cudaFree(cl);
        if (lab) cudaFree(lab);
        cudaGetLastError();
        return set_err(e == cudaErrorMemoryAllocation ? FSLIC_ENOMEM : FSLIC_ECUDA,
                       std::string("staging buffers: ") + cudaGetErrorString(e));
    }
    c->d_img = img; c->d_cl = cl; c->d_lab = lab;
    return FSLIC_OK;
}

extern "C" int fslic_b200_initialize_clusters_host(fslic_ctx* c, const uint8_t* h_images, fslic_cluster* h_clusters,
                                                   int batch) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    rc = ensure_staging(c);
    if (rc) return rc;
    cudaStream_t st = c->own_stream;
    const size_t ib = (size_t)batch * c->N * 3, cb = (size_t)batch * c->K * sizeof(fslic_cluster);
    CK(cudaMemcpyAsync(c->d_img, h_images, ib, cudaMemcpyHostToDevice, st));
    rc = fslic_b200_initialize_clusters(c, c->d_img, c->d_cl, batch, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h_clusters, c->d_cl, cb, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return FSLIC_OK;
}

// One iterate() of a small batch on the context's own stream, replayed from a captured CUDA graph when the same
// buffers, batch and parameters come back (the host entry points always use the context's staging buffers, so
// that is every call after the first).  Falls back to plain launches if the capture fails.
static int iterate_graphed(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels, int batch,
                           const fslic_params* p, cudaStream_t st) {
    // Only the Lab kernel reads the images: it is launched plainly, everything after it is the graph, so a caller that
    // feeds a new image buffer every call (a video stream) with the same cluster / label buffers still replays.
    int rc = check_batch(c, batch);
    if (rc) return rc;
    float coef;
    rc = check_params(c, p, &coef);
    if (rc) return rc;
    fslic_ctx::GraphKey k;
    memset(&k, 0, sizeof(k));
    k.img = nullptr; k.cl = d_clusters; k.lab = d_labels; k.batch = batch; k.p = *p; k.manhattan = c->manhattan;
    {
        USE_DEVICE(c->device);
        c->slice = 0;
        rc = launch_lab(c, d_images, c->quad, batch, p->convert_to_lab, st);
        if (rc) return rc;
    }
    // A replay rebuilds the spatial patches for the graph's parameters behind the cache's back (build_patches keeps
    // what the last plain build left), so after any graph launch the next plain call must rebuild them.
    if (c->gexec && memcmp(&k, &c->gkey, sizeof(k)) == 0) {
        CK(cudaGraphLaunch(c->gexec, st));
        c->graph_replays++;
        c->spt_valid = false;
        c->last_launches = c->glaunches;
        c->disp = c->gdisp;
        return FSLIC_OK;
    }
    if (c->gexec) {
        cudaGraphExecDestroy(c->gexec);
        c->gexec = nullptr;
    }
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
        cudaGetLastError();
        return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, st, true);
    }
    rc = iterate_plain(c, d_images, d_clusters, d_labels, batch, p, st, true);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(st, &g);
    if (rc != FSLIC_OK || e != cudaSuccess || !g) {
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();
        if (rc != FSLIC_OK) return rc;  // a parameter error: nothing was launched
        return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, st, true);
    }
    const cudaError_t ei = cudaGraphInstantiate(&c->gexec, g, 0);
    cudaGraphDestroy(g);
    if (ei != cudaSuccess) {
        c->gexec = nullptr;
        cudaGetLastError();
        return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, st, true);
    }
    memcpy(&c->gkey, &k, sizeof(k));
    c->graph_captures++;
    c->glaunches = c->last_launches;
    c->gdisp = c->disp;
    CK(cudaGraphLaunch(c->gexec, st));
    c->spt_valid = false;
    return FSLIC_OK;
}

// Enqueues H2D -> kernels -> D2H for one host batch on the context's three streams.  With may_sync the caller is
// going to block anyway, so the connectivity stage may read its per-image decisions back mid-way and start the
// label download of settled images early; without it nothing here waits for the device.
static int iterate_host_enqueue_body(fslic_ctx* c, const uint8_t* h_images, fslic_cluster* h_clusters,
                                     uint16_t* h_labels, int batch, const fslic_params* p, bool may_sync) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    rc = ensure_staging(c);
    if (rc) return rc;
    if (c->pending) {  // one batch in flight per context: its staging buffers are about to be overwritten
        CK(cudaStreamSynchronize(c->out_stream));
        CK(cudaStreamSynchronize(c->own_stream));
        c->pending = false;
    }
    c->disp = DispatchRecord();
    // Software pipeline over chunks of the batch: H2D(chunk i+1) | compute(chunk i) | D2H(chunk i-1) on three
    // streams, so for batches the PCIe copies hide behind the kernels (and vice versa).  With pinned host
    // buffers the copies are truly asynchronous; pageable buffers still work, just without overlap.
    const size_t N = (size_t)c->N;
    // chunks of 32: smaller chunks would pay the fixed latencies of the pipeline (notably the sequential
    // std::partial_sort replay of ambiguous images) once per chunk, which costs more than the overlap wins
    int chunk = batch < 32 ? batch : 32;
    if (const char* e = getenv("FSLIC_HOST_CHUNK")) {  // test hook: force the multi-chunk pipeline
        const int v = atoi(e);
        if (v >= 1 && v < chunk) chunk = v;
    }
    const int nchunks = (batch + chunk - 1) / chunk;
    while ((int)c->pipe_ev.size() < 3 * nchunks) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        c->pipe_ev.push_back(e);
    }
    fslic_params pp = *p;
    if (nchunks > 1) pp.collect_timing = 0;  // per-stage timings are only meaningful for an unchunked run
    const bool trace = may_sync && getenv("FSLIC_TRACE") != nullptr;
    std::vector<cudaEvent_t> tev;
    if (trace) {
        tev.resize(1 + 4 * nchunks);
        for (auto& e : tev) cudaEventCreate(&e);
        cudaEventRecord(tev[0], c->in_stream);
    }
    for (int k = 0; k < nchunks; k++) {
        const int b0 = k * chunk, nb = (batch - b0 < chunk) ? (batch - b0) : chunk;
        // Upload in two halves: the front half of the pipeline (Lab + passes) of the first half runs while the
        // second half is still on the wire; the back half (connectivity enforcement, whose replay latency is per
        // launch, not per image) then runs once over the whole chunk.
        bool labels_copied = false;
        static const bool no_split = getenv("FSLIC_HOST_SPLIT") && atoi(getenv("FSLIC_HOST_SPLIT")) == 0;
        if (nb >= 8 && !no_split) {
            float coef;
            rc = check_params(c, &pp, &coef);
            if (rc) return rc;
            int launches = 0;
            c->kev_on = false;  // per-launch kernel timing belongs to fslic_b200_iterate(collect_timing >= 2) only
            c->kev_used = 0;
            const int h0 = nb / 2;
            static const bool no_lanes = getenv("FSLIC_HOST_LANES") && atoi(getenv("FSLIC_HOST_LANES")) == 0;
            if (may_sync && !no_lanes && nchunks == 1 && nb >= 16 && nb <= c->cca_batch && nb <= 64) {
                // Blocking call: the caller waits anyway, so the two halves run as two independent pipelines that overlap
                // on the device -- half A's connectivity stage (incl. the ~0.7 ms std::partial_sort replay of its ambiguous
                // images, a handful of SMs) and its label download run while half B is still on the wire / in its assign
                // passes.  Each half has its own compute + side stream and its own window of the scratch arrays.
                for (int hpart = 0; hpart < 2; hpart++) {
                    const int s0 = b0 + (hpart ? h0 : 0), sn = hpart ? nb - h0 : h0;
                    CK(cudaMemcpyAsync(c->d_img + (size_t)s0 * N * 3, h_images + (size_t)s0 * N * 3, (size_t)sn * N * 3,
                                       cudaMemcpyHostToDevice, c->in_stream));
                    CK(cudaMemcpyAsync(c->d_cl + (size_t)s0 * c->K, h_clusters + (size_t)s0 * c->K,
                                       (size_t)sn * c->K * sizeof(fslic_cluster), cudaMemcpyHostToDevice, c->in_stream));
                    CK(cudaEventRecord(hpart ? c->pipe_ev[3 * k] : c->pipe_ev[3 * k + 2], c->in_stream));
                }
                for (int hpart = 0; hpart < 2; hpart++) {  // both front halves first: nothing in them waits for the host
                    const int s0 = b0 + (hpart ? h0 : 0), sn = hpart ? nb - h0 : h0;
                    cudaStream_t cs = hpart ? c->own_stream2 : c->own_stream;
                    CK(cudaStreamWaitEvent(cs, hpart ? c->pipe_ev[3 * k] : c->pipe_ev[3 * k + 2], 0));
                    // (the second front half starts behind the first: they share the cached spatial patches, which the first
                    //  call may still be building, and the first half's data is there earlier anyway)
                    if (hpart) CK(cudaStreamWaitEvent(cs, c->front_done, 0));
                    rc = iterate_front(c, s0 - b0, c->d_img + (size_t)s0 * N * 3, c->d_cl + (size_t)s0 * c->K, sn, &pp, coef, cs,
                                       &launches, false);
                    if (rc) return rc;
                    if (!hpart) CK(cudaEventRecord(c->front_done, cs));
                }
                for (int hpart = 0; hpart < 2; hpart++) {  // back halves: each reads its per-image decisions back mid-way
                    const int s0 = b0 + (hpart ? h0 : 0), sn = hpart ? nb - h0 : h0;
                    cudaStream_t cs = hpart ? c->own_stream2 : c->own_stream;
                    HostOut ho;
                    ho.h_labels = h_labels + (size_t)s0 * N;
                    ho.out_stream = c->out_stream;
                    ho.done = false;
                    rc = iterate_back(c, c->d_lab + (size_t)s0 * N, sn, &pp, cs, &launches, &ho, s0 - b0, hpart);
                    if (rc) return rc;
                    // clusters of this half (and its labels if run_cca did not download them itself)
                    CK(cudaEventRecord(c->pipe_ev[3 * k + 1], cs));
                    CK(cudaStreamWaitEvent(c->out_stream, c->pipe_ev[3 * k + 1], 0));
                    if (!ho.done)
                        CK(cudaMemcpyAsync(h_labels + (size_t)s0 * N, c->d_lab + (size_t)s0 * N, (size_t)sn * N * 2,
                                           cudaMemcpyDeviceToHost, c->out_stream));
                    CK(cudaMemcpyAsync(h_clusters + (size_t)s0 * c->K, c->d_cl + (size_t)s0 * c->K,
                                       (size_t)sn * c->K * sizeof(fslic_cluster), cudaMemcpyDeviceToHost, c->out_stream));
                }
                c->last_launches = launches;
                c->pending = true;
                CK(cudaStreamSynchronize(c->out_stream));
                CK(cudaStreamSynchronize(c->own_stream));
                CK(cudaStreamSynchronize(c->own_stream2));
                c->pending = false;
                return FSLIC_OK;
            }
            for (int hpart = 0; hpart < 2; hpart++) {
                const int s0 = b0 + (hpart ? h0 : 0), sn = hpart ? nb - h0 : h0;
                CK(cudaMemcpyAsync(c->d_img + (size_t)s0 * N * 3, h_images + (size_t)s0 * N * 3, (size_t)sn * N * 3,
                                   cudaMemcpyHostToDevice, c->in_stream));
                CK(cudaMemcpyAsync(c->d_cl + (size_t)s0 * c->K, h_clusters + (size_t)s0 * c->K,
                                   (size_t)sn * c->K * sizeof(fslic_cluster), cudaMemcpyHostToDevice, c->in_stream));
                cudaEvent_t ev = hpart ? c->pipe_ev[3 * k] : c->pipe_ev[3 * k + 2];
                CK(cudaEventRecord(ev, c->in_stream));
                if (trace && hpart == 1) cudaEventRecord(tev[1 + 4 * k], c->in_stream);
                CK(cudaStreamWaitEvent(c->own_stream, ev, 0));
                if (trace && hpart == 0) cudaEventRecord(tev[2 + 4 * k], c->own_stream);
                // slice s0 - b0 of the context buffers <-> images s0 .. s0+sn of this chunk
                rc = iterate_front(c, s0 - b0, c->d_img + (size_t)s0 * N * 3, c->d_cl + (size_t)s0 * c->K, sn, &pp, coef,
                                   c->own_stream, &launches, false);
                if (rc) return rc;
            }
            HostOut ho;
            ho.h_labels = h_labels + (size_t)b0 * N;
            ho.out_stream = c->out_stream;
            ho.done = false;
            rc = iterate_back(c, c->d_lab + (size_t)b0 * N, nb, &pp, c->own_stream, &launches, may_sync ? &ho : nullptr);
            if (rc) return rc;
            labels_copied = ho.done;
            c->last_launches = launches;
        } else {
        CK(cudaMemcpyAsync(c->d_img + (size_t)b0 * N * 3, h_images + (size_t)b0 * N * 3, (size_t)nb * N * 3,
                           cudaMemcpyHostToDevice, c->in_stream));
        CK(cudaMemcpyAsync(c->d_cl + (size_t)b0 * c->K, h_clusters + (size_t)b0 * c->K,
                           (size_t)nb * c->K * sizeof(fslic_cluster), cudaMemcpyHostToDevice, c->in_stream));
        CK(cudaEventRecord(c->pipe_ev[3 * k], c->in_stream));
        if (trace) cudaEventRecord(tev[1 + 4 * k], c->in_stream);
        CK(cudaStreamWaitEvent(c->own_stream, c->pipe_ev[3 * k], 0));
        if (trace) cudaEventRecord(tev[2 + 4 * k], c->own_stream);
        if (c->graphs_enabled && nb < 4 && nchunks == 1 && pp.collect_timing == 0)  // nb < 4: one stream, no host sync inside
            rc = iterate_graphed(c, c->d_img, c->d_cl, c->d_lab, nb, &pp, c->own_stream);
        else
            rc = iterate_plain(c, c->d_img + (size_t)b0 * N * 3, c->d_cl + (size_t)b0 * c->K, c->d_lab + (size_t)b0 * N, nb,
                                    &pp, c->own_stream);
        if (rc) return rc;
        }
        CK(cudaEventRecord(c->pipe_ev[3 * k + 1], c->own_stream));
        if (trace) cudaEventRecord(tev[3 + 4 * k], c->own_stream);
        CK(cudaStreamWaitEvent(c->out_stream, c->pipe_ev[3 * k + 1], 0));
        if (!labels_copied)
            CK(cudaMemcpyAsync(h_labels + (size_t)b0 * N, c->d_lab + (size_t)b0 * N, (size_t)nb * N * 2, cudaMemcpyDeviceToHost,
                               c->out_stream));
        CK(cudaMemcpyAsync(h_clusters + (size_t)b0 * c->K, c->d_cl + (size_t)b0 * c->K,
                           (size_t)nb * c->K * sizeof(fslic_cluster), cudaMemcpyDeviceToHost, c->out_stream));
        if (trace) cudaEventRecord(tev[4 + 4 * k], c->out_stream);
    }
    c->pending = true;
    if (!may_sync) return FSLIC_OK;
    CK(cudaStreamSynchronize(c->out_stream));
    CK(cudaStreamSynchronize(c->own_stream));
    c->pending = false;
    if (trace) {
        float ms;
        for (int k = 0; k < nchunks; k++) {
            float a, b2, c2, d2;
            cudaEventElapsedTime(&a, tev[0], tev[1 + 4 * k]);
            cudaEventElapsedTime(&b2, tev[0], tev[2 + 4 * k]);
            cudaEventElapsedTime(&c2, tev[0], tev[3 + 4 * k]);
            cudaEventElapsedTime(&d2, tev[0], tev[4 + 4 * k]);
            fprintf(stderr, "[fslic trace] chunk %d: h2d done %.3f | compute %.3f..%.3f | d2h done %.3f ms\n", k, a, b2, c2, d2);
        }
        (void)ms;
        for (auto e : tev) cudaEventDestroy(e);
    }
    return FSLIC_OK;
}

static int iterate_host_enqueue(fslic_ctx* c, const uint8_t* h_images, fslic_cluster* h_clusters, uint16_t* h_labels,
                                int batch, const fslic_params* p, bool may_sync) {
    const int rc = iterate_host_enqueue_body(c, h_images, h_clusters, h_labels, batch, p, may_sync);
    if (rc != FSLIC_OK && c && c->in_stream) {
        // an error after copies / kernels were enqueued: nothing may stay in flight on the staging buffers or the
        // caller's host buffers once the error is reported
        const std::string keep = g_err;
        DeviceGuard g(c->device);
        cudaStreamSynchronize(c->in_stream);
        cudaStreamSynchronize(c->own_stream);
        cudaStreamSynchronize(c->side_stream);
        if (c->own_stream2) cudaStreamSynchronize(c->own_stream2);
        if (c->side_stream2) cudaStreamSynchronize(c->side_stream2);
        cudaStreamSynchronize(c->out_stream);
        cudaGetLastError();
        c->pending = false;
        g_err = keep;
    }
    return rc;
}

extern "C" int fslic_b200_iterate_host(fslic_ctx* c, const uint8_t* h_images, fslic_cluster* h_clusters,
                                       uint16_t* h_labels, int batch, const fslic_params* p) {
    if (c && c->trace_on) return set_err(FSLIC_EINVAL, "the host entry points are not traced: turn tracing off or use fslic_b200_iterate");
    return iterate_host_enqueue(c, h_images, h_clusters, h_labels, batch, p, true);
}

extern "C" int fslic_b200_iterate_host_async(fslic_ctx* c, const uint8_t* h_images, fslic_cluster* h_clusters,
                                             uint16_t* h_labels, int batch, const fslic_params* p) {
    if (c && c->trace_on) return set_err(FSLIC_EINVAL, "the host entry points are not traced: turn tracing off or use fslic_b200_iterate");
    return iterate_host_enqueue(c, h_images, h_clusters, h_labels, batch, p, false);
}

// ---- debug_mode (trace.cuh, recorder_format.h) ---------------------------------------------------------------------
extern "C" int fslic_b200_debug_graph_counts(const fslic_ctx* c, int* captures, int* replays) {
    if (!c || !captures || !replays) return set_err(FSLIC_EINVAL, "NULL argument");
    *captures = c->graph_captures;
    *replays = c->graph_replays;
    return FSLIC_OK;
}

extern "C" int fslic_b200_set_trace(fslic_ctx* c, int on) {
    if (!c || c->cca_only) return set_err(FSLIC_EINVAL, "NULL or connectivity-only context");
    c->trace_on = on != 0;
    return FSLIC_OK;
}

extern "C" int fslic_b200_trace_info(const fslic_ctx* c, int* snapshots, int* batch, int* dist_bytes) {
    if (!c || !snapshots || !batch || !dist_bytes) return set_err(FSLIC_EINVAL, "NULL argument");
    *snapshots = c->tr_T;
    *batch = c->tr_B;
    *dist_bytes = c->tr_dist_bytes;
    return FSLIC_OK;
}

extern "C" int fslic_b200_trace_snapshots(fslic_ctx* c, int image, uint16_t* h_assignment, void* h_min_dists,
                                          fslic_cluster* h_clusters, uint32_t* h_mismatches) {
    if (!c) return set_err(FSLIC_EINVAL, "NULL context");
    if (c->tr_T == 0) return set_err(FSLIC_EINVAL, "no traced iterate has been recorded on this context");
    if (image < 0 || image >= c->tr_B) return set_err(FSLIC_EINVAL, "image outside the traced batch");
    USE_DEVICE(c->device);
    CK(cudaDeviceSynchronize());
    const size_t T = c->tr_T, N = c->N, K = c->K, slot = (size_t)image * T;
    if (h_clusters) CK(cudaMemcpy(h_clusters, tr_clusters(c) + slot * K, T * K * sizeof(fslic_cluster), cudaMemcpyDeviceToHost));
    if (h_min_dists)
        CK(cudaMemcpy(h_min_dists, tr_dist(c) + slot * N * c->tr_dist_bytes, T * N * c->tr_dist_bytes, cudaMemcpyDeviceToHost));
    if (h_assignment) CK(cudaMemcpy(h_assignment, tr_assign(c) + slot * N, T * N * 2, cudaMemcpyDeviceToHost));
    uint32_t bad = 0;
    CK(cudaMemcpy(&bad, c->tr_bad, sizeof(bad), cudaMemcpyDeviceToHost));
    if (h_mismatches) *h_mismatches = bad;
    if (bad)
        return set_err(FSLIC_ECHECK, "debug_mode self-check: " + std::to_string(bad) +
                                         " pixels were labelled differently from the trace kernel's argmin");
    return FSLIC_OK;
}

extern "C" int fslic_b200_format_report(int H, int W, int K, int snapshots, int dist_is_float, const uint16_t* assignment,
                                        const void* min_dists, const fslic_cluster* clusters, char** out, size_t* len) {
    if (!out || !len || H < 0 || W < 0 || K < 0 || snapshots < 0) return set_err(FSLIC_EINVAL, "bad argument");
    if (snapshots > 0 && ((H * W > 0 && (!assignment || !min_dists)) || (K > 0 && !clusters)))
        return set_err(FSLIC_EINVAL, "NULL array");
    *out = recorder_fmt::format_report(H, W, K, snapshots, dist_is_float != 0, assignment, min_dists, clusters, len);
    if (!*out) return set_err(FSLIC_ENOMEM, "out of host memory (debug_mode report)");
    return FSLIC_OK;
}

extern "C" void fslic_b200_free_report(char* p) { free(p); }

extern "C" int fslic_b200_wait(fslic_ctx* c) {
    if (!c) return set_err(FSLIC_EINVAL, "ctx is NULL");
    if (!c->pending) return FSLIC_OK;
    USE_DEVICE(c->device);
    CK(cudaStreamSynchronize(c->out_stream));
    CK(cudaStreamSynchronize(c->own_stream));
    c->pending = false;
    return FSLIC_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// SimpleCRF (src/simple-crf.{h,hpp,cpp}; csimple_crf.pyx).  The frames live in a deque in time order, exactly like the
// reference's; each owns its device buffers (crf.cuh) plus host copies of its clusters and adjacency lists, which the
// getters and the pairwise-energy queries read.  Slots of popped frames are kept and reused by the next push.
// Every copy, memset and kernel of a CRF goes to the CRF's stream (the last one passed to inference, NULL at first), so
// they are ordered whatever kind of stream that is.  inference / initialize / reset_inferred return at once; every
// other entry point synchronises that stream before it returns.
struct CrfSlot {
    int time = 0;
    fslic_cluster* clusters = nullptr;
    int32_t* offsets = nullptr;
    int32_t* nbr = nullptr;
    float* e_sp = nullptr;
    float* r_sp = nullptr;
    size_t edge_cap = 0;
    float *unary = nullptr, *q0 = nullptr, *q1 = nullptr, *msg = nullptr, *tmp = nullptr;
    std::vector<fslic_cluster> h_clusters;
    std::vector<int32_t> h_off, h_nbr;
    bool h_stale = false;  // a device push (fslic_b200_crfdev_push_label_frames) wrote the frame: h_* are out of date
};

struct fslic_crf {
    int device = 0, C = 0, N = 0;
    CrfParams p{};
    int next_time = 0, cur = 0;
    std::deque<CrfSlot*> frames;
    std::vector<CrfSlot*> pool;
    CrfFrameDev* d_table = nullptr;
    size_t table_cap = 0;
    float* d_scalar = nullptr;
    cudaStream_t st = nullptr;
};

static void crf_free_slot(CrfSlot* s) {
    cudaFree(s->clusters); cudaFree(s->offsets); cudaFree(s->nbr); cudaFree(s->e_sp); cudaFree(s->r_sp);
    cudaFree(s->unary); cudaFree(s->q0); cudaFree(s->q1); cudaFree(s->msg); cudaFree(s->tmp);
    delete s;
}

// A slot from the pool, or a new one with its node buffers allocated; the edge buffers are left to the caller.
static int crf_take_slot(fslic_crf* c, CrfSlot** out) {
    if (!c->pool.empty()) {
        *out = c->pool.back();
        c->pool.pop_back();
        return FSLIC_OK;
    }
    const size_t N = (size_t)c->N, CN = (size_t)c->C * c->N;
    CrfSlot* s = new (std::nothrow) CrfSlot();
    if (!s) return set_err(FSLIC_ENOMEM, "out of host memory");
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess && N) e = cudaMalloc(&s->clusters, sizeof(fslic_cluster) * N);
    if (e == cudaSuccess) e = cudaMalloc(&s->offsets, sizeof(int32_t) * (N + 1));
    if (e == cudaSuccess && CN) e = cudaMalloc(&s->unary, sizeof(float) * CN);
    if (e == cudaSuccess && CN) e = cudaMalloc(&s->q0, sizeof(float) * CN);
    if (e == cudaSuccess && CN) e = cudaMalloc(&s->q1, sizeof(float) * CN);
    if (e == cudaSuccess && CN) e = cudaMalloc(&s->msg, sizeof(float) * CN);
    if (e == cudaSuccess && N) e = cudaMalloc(&s->tmp, sizeof(float) * 4 * N);
    if (e != cudaSuccess) {
        crf_free_slot(s);
        return set_err(e == cudaErrorMemoryAllocation ? FSLIC_ENOMEM : FSLIC_ECUDA,
                       std::string("cudaMalloc: ") + cudaGetErrorString(e));
    }
    *out = s;
    return FSLIC_OK;
}

#define CKA(call)                                                                                     \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess)                                                                       \
            return set_err(e__ == cudaErrorMemoryAllocation ? FSLIC_ENOMEM : FSLIC_ECUDA,              \
                           std::string(#call) + ": " + cudaGetErrorString(e__));                      \
    } while (0)

// Enqueues the upload of the frame table on the CRF's stream from `h`, which must live until that stream is
// synchronised.
static int crf_stage_table(fslic_crf* c, std::vector<CrfFrameDev>& h) {
    const size_t T = c->frames.size();
    if (T > c->table_cap) {
        cudaFree(c->d_table);
        c->d_table = nullptr;
        c->table_cap = 0;
        CKA(cudaMalloc(&c->d_table, sizeof(CrfFrameDev) * T * 2));
        c->table_cap = T * 2;
    }
    h.resize(T);
    for (size_t t = 0; t < T; t++) {
        const CrfSlot* s = c->frames[t];
        h[t] = CrfFrameDev{s->clusters, s->offsets, s->nbr, s->unary, {s->q0, s->q1}, s->msg, s->e_sp, s->r_sp, s->tmp};
    }
    if (T) CK(cudaMemcpyAsync(c->d_table, h.data(), sizeof(CrfFrameDev) * T, cudaMemcpyHostToDevice, c->st));
    return FSLIC_OK;
}

static int crf_upload_table(fslic_crf* c) {
    std::vector<CrfFrameDev> h;
    int rc = crf_stage_table(c, h);
    if (rc) return rc;
    CK(cudaStreamSynchronize(c->st));
    return FSLIC_OK;
}

static int crf_frame(fslic_crf* c, int time, CrfSlot** out) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    if (c->frames.empty() || time < c->frames.front()->time || time > c->frames.back()->time)
        return set_err(FSLIC_ENOFRAME, "Time out of range");  // SimpleCRF::get_frame (simple-crf.hpp:111-119)
    *out = c->frames[(size_t)(time - c->frames.front()->time)];
    return FSLIC_OK;
}

// Look up the frame `time`, switch to the CRF's device and wait for its stream.
#define CRF_FRAME(c, time, s)                                                                         \
    CrfSlot* s = nullptr;                                                                             \
    { int rc__ = crf_frame(c, time, &s); if (rc__) return rc__; }                                     \
    USE_DEVICE((c)->device);                                                                          \
    CK(cudaStreamSynchronize((c)->st))

extern "C" int fslic_b200_crf_create(int device, int num_classes, int num_nodes, fslic_crf** out) {
    if (!out) return set_err(FSLIC_EINVAL, "out is NULL");
    *out = nullptr;
    if (num_classes < 0 || num_nodes < 0) return set_err(FSLIC_EINVAL, "num_classes and num_nodes must be >= 0");
    if ((long long)num_classes * num_nodes > (1LL << 31) - 1)
        return set_err(FSLIC_EINVAL, "num_classes * num_nodes must be < 2^31");
    USE_DEVICE(device);
    fslic_crf* c = new (std::nothrow) fslic_crf();
    if (!c) return set_err(FSLIC_ENOMEM, "out of host memory");
    c->device = device;
    c->C = num_classes;
    c->N = num_nodes;
    c->p = CrfParams{10, 10, 13, 13, 80, 0, 3};  // SimpleCRF::SimpleCRF (simple-crf.hpp:80-89)
    cudaError_t e = cudaMalloc(&c->d_scalar, sizeof(float));
    if (e != cudaSuccess) {
        delete c;
        return set_err(e == cudaErrorMemoryAllocation ? FSLIC_ENOMEM : FSLIC_ECUDA,
                       std::string("cudaMalloc: ") + cudaGetErrorString(e));
    }
    *out = c;
    return FSLIC_OK;
}

extern "C" int fslic_b200_crf_destroy(fslic_crf* c) {
    if (!c) return FSLIC_OK;
    DeviceGuard dev_guard__(c->device);
    cudaStreamSynchronize(c->st);
    for (CrfSlot* s : c->frames) crf_free_slot(s);
    for (CrfSlot* s : c->pool) crf_free_slot(s);
    cudaFree(c->d_table);
    cudaFree(c->d_scalar);
    delete c;
    return FSLIC_OK;
}

extern "C" int fslic_b200_crf_get_params(const fslic_crf* c, fslic_crf_params* out) {
    if (!c || !out) return set_err(FSLIC_EINVAL, "NULL argument");
    static_assert(sizeof(CrfParams) == sizeof(fslic_crf_params), "params layout");
    memcpy(out, &c->p, sizeof(CrfParams));
    return FSLIC_OK;
}

extern "C" int fslic_b200_crf_set_params(fslic_crf* c, const fslic_crf_params* params) {
    if (!c || !params) return set_err(FSLIC_EINVAL, "NULL argument");
    memcpy(&c->p, params, sizeof(CrfParams));  // read by the next inference() when it enqueues
    return FSLIC_OK;
}

// first_time, last_time (-1 when there are no frames) and the number of frames
extern "C" int fslic_b200_crf_times(const fslic_crf* c, int* first, int* last, int* num_frames) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    if (first) *first = c->frames.empty() ? -1 : c->frames.front()->time;
    if (last) *last = c->frames.empty() ? -1 : c->frames.back()->time;
    if (num_frames) *num_frames = (int)c->frames.size();
    return FSLIC_OK;
}

extern "C" int fslic_b200_crf_push_frame(fslic_crf* c, int* time_out) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    USE_DEVICE(c->device);
    CK(cudaStreamSynchronize(c->st));
    const size_t N = (size_t)c->N, CN = (size_t)c->C * c->N;
    CrfSlot* s;
    { int rc = crf_take_slot(c, &s); if (rc) return rc; }
    // SimpleCRFFrame::SimpleCRFFrame (simple-crf.hpp:29-33): value-initialised clusters with num_members = 1, empty
    // adjacency lists, unaries and q zero
    fslic_cluster blank;
    memset(&blank, 0, sizeof(blank));
    blank.num_members = 1;
    s->h_clusters.assign(N, blank);
    s->h_off.assign(N + 1, 0);
    s->h_nbr.clear();
    s->h_stale = false;
    if (N) CK(cudaMemcpyAsync(s->clusters, s->h_clusters.data(), sizeof(fslic_cluster) * N, cudaMemcpyHostToDevice, c->st));
    CK(cudaMemsetAsync(s->offsets, 0, sizeof(int32_t) * (N + 1), c->st));
    if (CN) {
        CK(cudaMemsetAsync(s->unary, 0, sizeof(float) * CN, c->st));
        CK(cudaMemsetAsync(s->q0, 0, sizeof(float) * CN, c->st));
        CK(cudaMemsetAsync(s->q1, 0, sizeof(float) * CN, c->st));
    }
    s->time = c->next_time++;
    c->frames.push_back(s);
    int rc = crf_upload_table(c);
    if (rc) {
        c->frames.pop_back();
        c->pool.push_back(s);
        c->next_time--;
        return rc;
    }
    if (time_out) *time_out = s->time;
    return FSLIC_OK;
}

// SimpleCRF::pop_frame (simple-crf.hpp:103-109): drops the first frame; *time_out = its time, -1 when empty
extern "C" int fslic_b200_crf_pop_frame(fslic_crf* c, int* time_out) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    if (c->frames.empty()) {
        if (time_out) *time_out = -1;
        return FSLIC_OK;
    }
    USE_DEVICE(c->device);
    CK(cudaStreamSynchronize(c->st));
    CrfSlot* s = c->frames.front();
    c->frames.pop_front();
    c->pool.push_back(s);
    if (time_out) *time_out = s->time;
    return crf_upload_table(c);
}

// Brings the host copies of a device-pushed frame up to date: one wait for the CRF's stream and a download of its
// records and CSR.  Every reader of h_clusters / h_off / h_nbr calls it first; for a host-fed frame it does nothing.
static int crf_refresh_host(fslic_crf* c, CrfSlot* s) {
    if (!s->h_stale) return FSLIC_OK;
    USE_DEVICE(c->device);
    const int N = c->N;
    s->h_clusters.resize(N);
    s->h_off.resize(N + 1);
    CK(cudaStreamSynchronize(c->st));
    if (N) CK(cudaMemcpyAsync(s->h_clusters.data(), s->clusters, sizeof(fslic_cluster) * N, cudaMemcpyDeviceToHost, c->st));
    CK(cudaMemcpyAsync(s->h_off.data(), s->offsets, sizeof(int32_t) * (N + 1), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    s->h_nbr.resize(s->h_off[N]);
    if (s->h_off[N]) {
        CK(cudaMemcpyAsync(s->h_nbr.data(), s->nbr, sizeof(int32_t) * s->h_off[N], cudaMemcpyDeviceToHost, c->st));
        CK(cudaStreamSynchronize(c->st));
    }
    s->h_stale = false;
    return FSLIC_OK;
}

extern "C" int fslic_b200_crf_set_clusters(fslic_crf* c, int time, const fslic_cluster* h_clusters) {
    if (!h_clusters && c && c->N) return set_err(FSLIC_EINVAL, "NULL argument");
    CRF_FRAME(c, time, s);
    if (c->N) {
        memcpy(s->h_clusters.data(), h_clusters, sizeof(fslic_cluster) * c->N);
        CK(cudaMemcpyAsync(s->clusters, h_clusters, sizeof(fslic_cluster) * c->N, cudaMemcpyHostToDevice, c->st));
        CK(cudaStreamSynchronize(c->st));
    }
    return FSLIC_OK;
}

extern "C" int fslic_b200_crf_get_clusters(fslic_crf* c, int time, fslic_cluster* h_out) {
    CrfSlot* s = nullptr;
    int rc = crf_frame(c, time, &s);
    if (!rc) rc = crf_refresh_host(c, s);
    if (rc) return rc;
    if (c->N) memcpy(h_out, s->h_clusters.data(), sizeof(fslic_cluster) * c->N);
    return FSLIC_OK;
}

// SimpleCRFFrame::set_connectivity (simple-crf.cpp:11-19): rows 0..num_rows-1 get the lists of the CSR (h_offsets
// [num_rows + 1], h_neighbors [h_offsets[num_rows]]), the other rows keep theirs.  Every neighbour must be a node of
// the frame; otherwise nothing changes.
extern "C" int fslic_b200_crf_set_connectivity(fslic_crf* c, int time, int num_rows, const int32_t* h_offsets,
                                               const int32_t* h_neighbors) {
    CrfSlot* s = nullptr;
    int rc = crf_frame(c, time, &s);
    if (!rc) rc = crf_refresh_host(c, s);
    if (rc) return rc;
    const int N = c->N;
    if (num_rows < 0 || num_rows > N) return set_err(FSLIC_EINVAL, "more adjacency lists than nodes");
    if (!h_offsets) return set_err(FSLIC_EINVAL, "NULL argument");
    if (h_offsets[0] != 0) return set_err(FSLIC_EINVAL, "offsets must start at 0");
    for (int i = 0; i < num_rows; i++)
        if (h_offsets[i + 1] < h_offsets[i]) return set_err(FSLIC_EINVAL, "offsets must not decrease");
    const int32_t E_new = h_offsets[num_rows];
    if (E_new && !h_neighbors) return set_err(FSLIC_EINVAL, "NULL argument");
    for (int32_t k = 0; k < E_new; k++)
        if (h_neighbors[k] < 0 || h_neighbors[k] >= N)
            return set_err(FSLIC_EINVAL, "neighbour index out of range");
    std::vector<int32_t> off(N + 1), nb;
    const long long E = (long long)E_new + (s->h_off[N] - s->h_off[num_rows]);
    if (E > (1LL << 31) - 1) return set_err(FSLIC_EINVAL, "too many edges");
    nb.reserve((size_t)E);
    nb.insert(nb.end(), h_neighbors, h_neighbors + E_new);
    memcpy(off.data(), h_offsets, sizeof(int32_t) * (num_rows + 1));
    nb.insert(nb.end(), s->h_nbr.begin() + s->h_off[num_rows], s->h_nbr.end());
    for (int i = num_rows; i < N; i++) off[i + 1] = off[i] + (s->h_off[i + 1] - s->h_off[i]);
    USE_DEVICE(c->device);
    CK(cudaStreamSynchronize(c->st));
    if ((size_t)E > s->edge_cap) {
        cudaFree(s->nbr); cudaFree(s->e_sp); cudaFree(s->r_sp);
        s->nbr = nullptr; s->e_sp = s->r_sp = nullptr; s->edge_cap = 0;
        s->h_off.assign(N + 1, 0);  // until the new lists are in place the frame has none
        s->h_nbr.clear();
        CKA(cudaMemsetAsync(s->offsets, 0, sizeof(int32_t) * (N + 1), c->st));
        const size_t cap = (size_t)E + (size_t)E / 2;
        CKA(cudaMalloc(&s->nbr, sizeof(int32_t) * cap));
        CKA(cudaMalloc(&s->e_sp, sizeof(float) * cap));
        CKA(cudaMalloc(&s->r_sp, sizeof(float) * cap));
        s->edge_cap = cap;
        rc = crf_upload_table(c);
        if (rc) return rc;
    }
    if (E) CK(cudaMemcpyAsync(s->nbr, nb.data(), sizeof(int32_t) * E, cudaMemcpyHostToDevice, c->st));
    CK(cudaMemcpyAsync(s->offsets, off.data(), sizeof(int32_t) * (N + 1), cudaMemcpyHostToDevice, c->st));
    CK(cudaStreamSynchronize(c->st));
    s->h_off.swap(off);
    s->h_nbr.swap(nb);
    return FSLIC_OK;
}

// The adjacency lists as CSR: h_offsets [N + 1]; h_neighbors (may be NULL) receives the first `cap` neighbours.
extern "C" int fslic_b200_crf_get_connectivity(fslic_crf* c, int time, int32_t* h_offsets, int32_t* h_neighbors,
                                               long long cap) {
    CrfSlot* s = nullptr;
    int rc = crf_frame(c, time, &s);
    if (!rc) rc = crf_refresh_host(c, s);
    if (rc) return rc;
    if (h_offsets) memcpy(h_offsets, s->h_off.data(), sizeof(int32_t) * (c->N + 1));
    if (h_neighbors) {
        const size_t n = std::min((size_t)(cap < 0 ? 0 : cap), s->h_nbr.size());
        if (n) memcpy(h_neighbors, s->h_nbr.data(), sizeof(int32_t) * n);
    }
    return FSLIC_OK;
}

static int crf_put_unary(fslic_crf* c, CrfSlot* s, const float* h) {
    const size_t CN = (size_t)c->C * c->N;
    if (CN) CK(cudaMemcpyAsync(s->unary, h, sizeof(float) * CN, cudaMemcpyHostToDevice, c->st));
    CK(cudaStreamSynchronize(c->st));
    return FSLIC_OK;
}

// SimpleCRFFrame::set_unary / get_unary (simple-crf.hpp:53-61): float [C][N]
extern "C" int fslic_b200_crf_set_unary(fslic_crf* c, int time, const float* h_unary) {
    CRF_FRAME(c, time, s);
    return crf_put_unary(c, s, h_unary);
}

extern "C" int fslic_b200_crf_get_unary(fslic_crf* c, int time, float* h_out) {
    CRF_FRAME(c, time, s);
    const size_t CN = (size_t)c->C * c->N;
    if (CN) CK(cudaMemcpyAsync(h_out, s->unary, sizeof(float) * CN, cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    return FSLIC_OK;
}

// The unary setters run on the host with glibc's logf, as the reference's do.  Their float arithmetic is the object
// code's: set_mask's active probability is one fused multiply-add.
// SimpleCRFFrame::set_unbiased (simple-crf.cpp:34-37)
extern "C" int fslic_b200_crf_set_unbiased(fslic_crf* c, int time) {
    CRF_FRAME(c, time, s);
    std::vector<float> u((size_t)c->C * c->N, logf((float)c->C));
    return crf_put_unary(c, s, u.data());
}

// SimpleCRFFrame::set_mask (simple-crf.cpp:39-50).  Every class must be in [0, C); otherwise nothing changes.
extern "C" int fslic_b200_crf_set_mask(fslic_crf* c, int time, const int32_t* h_classes, float confidence) {
    CRF_FRAME(c, time, s);
    const int C = c->C, N = c->N;
    for (int i = 0; i < N; i++)
        if (h_classes[i] < 0 || h_classes[i] >= C) return set_err(FSLIC_EINVAL, "class index out of range");
    const float lowest = 1.0f / (float)C;
    const float active = fmaf(1.0f - lowest, confidence, lowest);
    const float inactive = (1.0f - active) / (float)(C - 1);
    const float active_unary = -logf(active), inactive_unary = -logf(inactive);
    std::vector<float> u((size_t)C * N, inactive_unary);
    for (int i = 0; i < N; i++) u[(size_t)N * h_classes[i] + i] = active_unary;
    return crf_put_unary(c, s, u.data());
}

// SimpleCRFFrame::set_proba (simple-crf.cpp:53-55): unary = -logf(p), p float [C][N]
extern "C" int fslic_b200_crf_set_proba(fslic_crf* c, int time, const float* h_proba) {
    CRF_FRAME(c, time, s);
    const size_t CN = (size_t)c->C * c->N;
    std::vector<float> u(CN);
    for (size_t k = 0; k < CN; k++) u[k] = -logf(h_proba[k]);
    return crf_put_unary(c, s, u.data());
}

// SimpleCRFFrame::get_inferred: q float [C][N]
extern "C" int fslic_b200_crf_get_inferred(fslic_crf* c, int time, float* h_out) {
    CRF_FRAME(c, time, s);
    const size_t CN = (size_t)c->C * c->N;
    if (CN) CK(cudaMemcpyAsync(h_out, c->cur ? s->q1 : s->q0, sizeof(float) * CN, cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    return FSLIC_OK;
}

// The unaries and current q buffer of a frame, for the per-frame kernels
static CrfFrameQ crf_frame_q(const fslic_crf* c, const CrfSlot* s) { return CrfFrameQ{s->unary, c->cur ? s->q1 : s->q0}; }

// reset_inferred of the frames of `set` (n <= CRF_GROUP_MAX, C * N values each) in one launch
static int crf_reset_set(const CrfFrameQSet& set, int n, long long CN, int device, cudaStream_t st) {
    if (!CN || !n) return FSLIC_OK;
    k_crf_reset<<<dim3((unsigned)grid_for(CN, device), (unsigned)n), 256, 0, st>>>(set, CN);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

static int crf_reset(fslic_crf* c, CrfSlot* s) {
    CrfFrameQSet set;
    set.f[0] = crf_frame_q(c, s);
    return crf_reset_set(set, 1, (long long)c->C * c->N, c->device, c->st);
}

// SimpleCRFFrame::reset_inferred (simple-crf.cpp:57-59): q = expf(-unary), asynchronous on the CRF's stream
extern "C" int fslic_b200_crf_reset_inferred(fslic_crf* c, int time) {
    CrfSlot* s = nullptr;
    int rc = crf_frame(c, time, &s);
    if (rc) return rc;
    USE_DEVICE(c->device);
    return crf_reset(c, s);
}

// SimpleCRF::initialize (simple-crf.cpp:153-157): reset_inferred on every frame
extern "C" int fslic_b200_crf_initialize(fslic_crf* c) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    USE_DEVICE(c->device);
    const long long CN = (long long)c->C * c->N;
    for (size_t t0 = 0; t0 < c->frames.size(); t0 += CRF_GROUP_MAX) {
        const int n = (int)std::min(c->frames.size() - t0, (size_t)CRF_GROUP_MAX);
        CrfFrameQSet set;
        for (int k = 0; k < n; k++) set.f[k] = crf_frame_q(c, c->frames[t0 + k]);
        int rc = crf_reset_set(set, n, CN, c->device, c->st);
        if (rc) return rc;
    }
    return FSLIC_OK;
}

// max_iter Jacobi steps of the chains of crfs[0 .. n) (n <= CRF_GROUP_MAX; one device, C and N; each with frames) on
// `st`: 1 + 2 max_iter launches; each CRF's cur flips once per step.  With N or C zero there is nothing to compute and
// cur stays.
static int crf_run_chains(fslic_crf* const* crfs, int n, unsigned long long max_iter, cudaStream_t st) {
    const int C = crfs[0]->C, N = crfs[0]->N;
    if (!n || !max_iter || !N || !C) return FSLIC_OK;
    CrfChainSet set;
    long long Tmax = 0;
    for (int k = 0; k < n; k++) {
        const fslic_crf* c = crfs[k];
        set.ch[k] = CrfChain{c->d_table, (int)c->frames.size(), c->cur, c->p};
        Tmax = std::max(Tmax, (long long)c->frames.size());
    }
    const long long TN = Tmax * N, TCN = TN * C;
    const dim3 node_grid((unsigned)((TN + 127) / 128), (unsigned)n), msg_grid((unsigned)((TCN + 127) / 128), (unsigned)n);
    k_crf_pairwise<<<node_grid, 128, 0, st>>>(set, N);
    CK(cudaGetLastError());
    for (unsigned long long it = 0; it < max_iter; it++) {
        k_crf_msg<<<msg_grid, 128, 0, st>>>(set, N, C, (int)(it & 1));
        k_crf_compat<<<node_grid, 128, 0, st>>>(set, N, C, (int)(it & 1));
        CK(cudaGetLastError());
    }
    for (int k = 0; k < n; k++) crfs[k]->cur ^= (int)(max_iter & 1);
    return FSLIC_OK;
}

// SimpleCRF::inference (simple-crf.cpp:159-163): max_iter Jacobi steps over all frames.  1 + 2 max_iter launches on
// `stream`, no host synchronisation.  With no frames the reference's infer_once looks up time -1 and throws
// std::out_of_range; here that is FSLIC_ENOFRAME.
extern "C" int fslic_b200_crf_inference(fslic_crf* c, unsigned long long max_iter, void* stream) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    if (max_iter == 0) return FSLIC_OK;
    if (c->frames.empty()) return set_err(FSLIC_ENOFRAME, "Time out of range");
    USE_DEVICE(c->device);
    if ((cudaStream_t)stream != c->st) {
        CK(cudaStreamSynchronize(c->st));
        c->st = (cudaStream_t)stream;
    }
    return crf_run_chains(&c, 1, max_iter, c->st);
}

// SimpleCRFFrame::calc_spatial_pairwise_energy(node_i, node_j) of frame `time` (simple-crf.hpp:149-174)
extern "C" int fslic_b200_crf_spatial_pairwise_energy(fslic_crf* c, int time, int node_i, int node_j, float* out) {
    CRF_FRAME(c, time, s);
    if (node_i < 0 || node_j < 0 || node_i >= c->N || node_j >= c->N) return set_err(FSLIC_EINVAL, "node number is out of range");
    { int rc = crf_refresh_host(c, s); if (rc) return rc; }
    if (node_i == node_j) {
        *out = 0.0f;
        return FSLIC_OK;
    }
    k_crf_energy<<<1, 1, 0, c->st>>>(s->h_clusters[node_i], s->h_clusters[node_j], 1, c->p, c->d_scalar);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, c->d_scalar, sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    return FSLIC_OK;
}

// SimpleCRFFrame::calc_temporal_pairwise_energy(node, other) of frame `time` of `c` against frame `other_time` of `other`
// (simple-crf.hpp:135-147), with c's params; 0 when both are the same frame.
extern "C" int fslic_b200_crf_temporal_pairwise_energy(fslic_crf* c, int time, int node, fslic_crf* other, int other_time,
                                                       float* out) {
    CrfSlot* o = nullptr;
    int rc = crf_frame(other, other_time, &o);
    if (rc) return rc;
    CRF_FRAME(c, time, s);
    if (node < 0 || node >= c->N || node >= other->N) return set_err(FSLIC_EINVAL, "node number is out of range");
    rc = crf_refresh_host(c, s);
    if (!rc) rc = crf_refresh_host(other, o);
    if (rc) return rc;
    if (s == o) {
        *out = 0.0f;
        return FSLIC_OK;
    }
    k_crf_energy<<<1, 1, 0, c->st>>>(s->h_clusters[node], o->h_clusters[node], 0, c->p, c->d_scalar);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, c->d_scalar, sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    return FSLIC_OK;
}

// A glibc clone (glibc_expf.cuh, glibc_logf.cuh) over the bit patterns first .. first + n - 1 (wrapping) on the host,
// with the FMA instruction where the CPU has it.  Both compiles are exact (libm's fma is correctly rounded); the FMA
// instruction is only faster.
template <float (*fn)(float)>
static inline __attribute__((always_inline)) void host_over_bits(uint32_t first, long long n, float* out) {
    for (long long i = 0; i < n; i++) out[i] = fn(gexpf::u2f(first + (uint32_t)i));
}
template <float (*fn)(float)>
__attribute__((target("fma"))) static void host_over_bits_fma(uint32_t first, long long n, float* out) {
    host_over_bits<fn>(first, n, out);
}
template <float (*fn)(float)>
static int debug_host_over_bits(uint32_t first, long long n, float* h_out) {
    if (n < 0 || (n && !h_out)) return set_err(FSLIC_EINVAL, "bad buffer");
    if (__builtin_cpu_supports("fma")) host_over_bits_fma<fn>(first, n, h_out);
    else host_over_bits<fn>(first, n, h_out);
    return FSLIC_OK;
}

extern "C" int fslic_b200_debug_expf_host(uint32_t first, long long n, float* h_out) {
    return debug_host_over_bits<gexpf::expf>(first, n, h_out);
}

extern "C" int fslic_b200_debug_expf_device(int device, uint32_t first, long long n, float* d_out, void* stream) {
    if (n < 0 || (n && !d_out)) return set_err(FSLIC_EINVAL, "bad buffer");
    if (!n) return FSLIC_OK;
    USE_DEVICE(device);
    k_expf_debug<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(first, n, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// The CRF fed from device memory (crf_feed.cuh).  Each entry point adopts `stream` the way inference does (waiting for
// the CRF's previous stream if it differs) and only enqueues: labels, clusters, graphs and unaries never pass through
// the host.  The host waits left are the frame-table upload every push makes and set_mask's 4-byte validity flag.
// A device push marks the frame's host copies stale; crf_refresh_host brings them back for the host-side readers.

// Switch the CRF to `stream`, waiting for the old one if it differs (as fslic_b200_crf_inference does)
static int crf_adopt_stream(fslic_crf* c, void* stream) {
    if ((cudaStream_t)stream != c->st) {
        CK(cudaStreamSynchronize(c->st));
        c->st = (cudaStream_t)stream;
    }
    return FSLIC_OK;
}

// The graph of `batch` label maps (fslic_b200_get_connectivity_batch's scratch) followed by their counts [batch][K] and
// neighbour lists [batch][K][12].
extern "C" size_t fslic_b200_crfdev_push_scratch_bytes(int K, int batch) {
    const size_t graph = fslic_b200_connectivity_batch_scratch_bytes(K, batch);
    if (graph == (size_t)-1) return graph;
    if (K <= 0 || batch <= 0) return 256;
    return align_up(graph, 256) + align_up((size_t)batch * K * 4, 256) + align_up((size_t)batch * K * CONN_MAX * 4, 256);
}

// A slot for a device push: from the pool or newly allocated, with room for 12 * N edges (the graph's cap), so the
// steady state never reallocates.  The slot is not in the deque yet.
static int crfdev_take_slot(fslic_crf* c, CrfSlot** out) {
    const size_t N = (size_t)c->N, E = N * CONN_MAX;
    CrfSlot* s;
    { int rc = crf_take_slot(c, &s); if (rc) return rc; }
    if (s->edge_cap < E) {
        cudaFree(s->nbr); cudaFree(s->e_sp); cudaFree(s->r_sp);
        s->nbr = nullptr; s->e_sp = s->r_sp = nullptr; s->edge_cap = 0;
        cudaError_t e = cudaMalloc(&s->nbr, sizeof(int32_t) * E);
        if (e == cudaSuccess) e = cudaMalloc(&s->e_sp, sizeof(float) * E);
        if (e == cudaSuccess) e = cudaMalloc(&s->r_sp, sizeof(float) * E);
        if (e != cudaSuccess) {
            c->pool.push_back(s);  // keeps its node buffers; edge_cap 0 makes the next push retry
            return set_err(e == cudaErrorMemoryAllocation ? FSLIC_ENOMEM : FSLIC_ECUDA,
                           std::string("cudaMalloc: ") + cudaGetErrorString(e));
        }
        s->edge_cap = E;
    }
    s->h_clusters.resize(N);  // sizes the host readers rely on; the contents are stale until refreshed
    s->h_off.resize(N + 1);
    s->h_stale = true;
    *out = s;
    return FSLIC_OK;
}

// The argument checks of a device push of `batch` label maps into CRFs with N == K nodes.
static int crfdev_check_push(int batch, int H, int W, int K, const uint16_t* d_labels, const fslic_cluster* d_clusters,
                             void* d_scratch, size_t scratch_bytes) {
    if (batch < 0 || H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    if (batch == 0) return FSLIC_OK;
    if (!d_labels || !d_clusters || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_crfdev_push_scratch_bytes(K, batch);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    const int obits = bit_length(3ull * (unsigned long long)H * (unsigned long long)W);
    if (obits + bit_length(batch - 1) > 64) return set_err(FSLIC_EINVAL, "batch * H * W too large");
    return FSLIC_OK;
}

// Appends frame b, built from d_labels[b] and d_clusters[b], to owners[b] (all on one device with the same C and
// N == K, all already on `stream`; a CRF may own several frames, which it receives in order).  Arguments are checked
// by the caller.  The new frames join their tables first, so the one host wait (after the table uploads) does not
// include this push's kernels.  On failure every owner is left as it was.
static int crfdev_push(fslic_crf* const* owners, int batch, int H, int W, int K, const uint16_t* d_labels,
                       const fslic_cluster* d_clusters, void* d_scratch, cudaStream_t st, int* times_out) {
    std::vector<CrfSlot*> slots;
    for (int b = 0; b < batch; b++) {
        CrfSlot* s = nullptr;
        int rc = crfdev_take_slot(owners[b], &s);
        if (rc) {
            for (int k = 0; k < b; k++) owners[k]->pool.push_back(slots[k]);
            return rc;
        }
        slots.push_back(s);
    }
    std::vector<fslic_crf*> distinct;
    for (int b = 0; b < batch; b++) {
        fslic_crf* c = owners[b];
        if (std::find(distinct.begin(), distinct.end(), c) == distinct.end()) distinct.push_back(c);
        slots[b]->time = c->next_time++;
        c->frames.push_back(slots[b]);
    }
    int rc = FSLIC_OK;
    {
        std::vector<std::vector<CrfFrameDev>> tables(distinct.size());
        for (size_t k = 0; k < distinct.size() && !rc; k++) rc = crf_stage_table(distinct[k], tables[k]);
        const cudaError_t e = cudaStreamSynchronize(st);
        if (!rc && e != cudaSuccess) rc = set_err(FSLIC_ECUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e));
    }
    const fslic_crf* c0 = owners[0];
    if (!rc) {
        const size_t graph_bytes = align_up(fslic_b200_connectivity_batch_scratch_bytes(K, batch), 256);
        unsigned char* p = static_cast<unsigned char*>(d_scratch);
        int32_t* counts = reinterpret_cast<int32_t*>(p + graph_bytes);
        uint32_t* nbrs = reinterpret_cast<uint32_t*>(p + graph_bytes + align_up((size_t)batch * K * 4, 256));
        rc = fslic_b200_get_connectivity_batch(c0->device, batch, H, W, K, d_labels, counts, nbrs, nullptr, d_scratch,
                                               graph_bytes, st);
        const long long CN = (long long)c0->C * K;
        const float unbiased = logf((float)c0->C);  // set_unbiased's constant, glibc's logf as on the host path
        const unsigned node_blocks = (unsigned)grid_for(CN > K ? CN : K, c0->device);
        for (int b0 = 0; b0 < batch && !rc; b0 += CRF_GROUP_MAX) {
            const int n = std::min(batch - b0, CRF_GROUP_MAX);
            FeedFrameSet dst;
            for (int k = 0; k < n; k++) {
                const CrfSlot* s = slots[b0 + k];
                dst.f[k] = FeedFramePtrs{s->clusters, s->unary, s->q0, s->q1, s->offsets, s->nbr};
            }
            k_feed_nodes<<<dim3(node_blocks, (unsigned)n), 256, 0, st>>>(d_clusters + (size_t)b0 * K, dst, K, c0->C,
                                                                         unbiased);
            k_feed_csr<<<dim3(1, (unsigned)n), FEED_CSR_THREADS, 0, st>>>(counts + (size_t)b0 * K,
                                                                          nbrs + (size_t)b0 * K * CONN_MAX, K, dst);
            const cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) rc = set_err(FSLIC_ECUDA, std::string("feed kernels: ") + cudaGetErrorString(e));
        }
    }
    if (rc) {  // take the frames back out, newest first
        for (int b = batch - 1; b >= 0; b--) {
            fslic_crf* c = owners[b];
            c->pool.push_back(c->frames.back());
            c->frames.pop_back();
            c->next_time--;
        }
        for (fslic_crf* c : distinct) crf_upload_table(c);
        return rc;
    }
    if (times_out)
        for (int b = 0; b < batch; b++) times_out[b] = slots[b]->time;
    return FSLIC_OK;
}

// Pushes `batch` frames; frame b is what push_slic_frame gives for label map d_labels[b] (int16 [H][W], labels outside
// [0, K) ignored) and records d_clusters[b] ([K]): its records, its adjacency graph and unbiased unaries.  K must equal
// the CRF's num_nodes.  Every argument is checked before anything is pushed (the host push_slic_frame pushes a blank
// frame first and only then fails on a K mismatch).  times_out (host, [batch], may be NULL) receives the new times.
extern "C" int fslic_b200_crfdev_push_label_frames(fslic_crf* c, int batch, int H, int W, int K, const uint16_t* d_labels,
                                                   const fslic_cluster* d_clusters, void* d_scratch, size_t scratch_bytes,
                                                   void* stream, int* times_out) {
    if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
    if (K != c->N) return set_err(FSLIC_EINVAL, "K must equal the CRF's num_nodes");
    { int rc = crfdev_check_push(batch, H, W, K, d_labels, d_clusters, d_scratch, scratch_bytes); if (rc) return rc; }
    if (batch == 0) return FSLIC_OK;
    USE_DEVICE(c->device);
    { int rc = crf_adopt_stream(c, stream); if (rc) return rc; }
    const std::vector<fslic_crf*> owners(batch, c);
    return crfdev_push(owners.data(), batch, H, W, K, d_labels, d_clusters, d_scratch, c->st, times_out);
}

// Look up frame `time`, switch to the CRF's device and adopt `stream`: the device setters never wait for it.
#define CRFDEV_FRAME(c, time, s, stream)                                                              \
    CrfSlot* s = nullptr;                                                                             \
    { int rc__ = crf_frame(c, time, &s); if (rc__) return rc__; }                                     \
    USE_DEVICE((c)->device);                                                                          \
    { int rc__ = crf_adopt_stream(c, stream); if (rc__) return rc__; }

// set_unary from device memory: float [C][N], copied on the stream
extern "C" int fslic_b200_crfdev_set_unary(fslic_crf* c, int time, const float* d_unary, void* stream) {
    CRFDEV_FRAME(c, time, s, stream);
    const size_t CN = (size_t)c->C * c->N;
    if (CN && !d_unary) return set_err(FSLIC_EINVAL, "NULL argument");
    if (CN) CK(cudaMemcpyAsync(s->unary, d_unary, sizeof(float) * CN, cudaMemcpyDeviceToDevice, c->st));
    return FSLIC_OK;
}

// set_proba from device memory: unary = -logf(p) with glibc's logf (glibc_logf.cuh), p float [C][N]
extern "C" int fslic_b200_crfdev_set_proba(fslic_crf* c, int time, const float* d_proba, void* stream) {
    CRFDEV_FRAME(c, time, s, stream);
    const long long CN = (long long)c->C * c->N;
    if (!CN) return FSLIC_OK;
    if (!d_proba) return set_err(FSLIC_EINVAL, "NULL argument");
    CrfFrameQSet set;
    set.f[0] = crf_frame_q(c, s);
    k_feed_proba<<<(unsigned)grid_for(CN, c->device), 256, 0, c->st>>>(d_proba, set, CN);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// set_mask from device memory: classes int32 [N], each in [0, C), checked on the device; the call waits for that one
// flag and changes nothing if any class is out of range.  The two unary values are the host path's: fmaf, division
// and glibc's logf in its order, on the host.
extern "C" int fslic_b200_crfdev_set_mask(fslic_crf* c, int time, const int32_t* d_classes, float confidence, void* stream) {
    CRFDEV_FRAME(c, time, s, stream);
    const int C = c->C, N = c->N;
    if (!N) return FSLIC_OK;
    if (!d_classes) return set_err(FSLIC_EINVAL, "NULL argument");
    int* d_bad = reinterpret_cast<int*>(c->d_scalar);
    CK(cudaMemsetAsync(d_bad, 0, sizeof(int), c->st));
    k_feed_mask_check<<<(int)grid_for(N, c->device), 256, 0, c->st>>>(d_classes, N, C, d_bad);
    CK(cudaGetLastError());
    int bad = 0;
    CK(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    if (bad) return set_err(FSLIC_EINVAL, "class index out of range");
    const float lowest = 1.0f / (float)C;
    const float active = fmaf(1.0f - lowest, confidence, lowest);
    const float inactive = (1.0f - active) / (float)(C - 1);
    const float active_unary = glogf::neg_logf(active), inactive_unary = glogf::neg_logf(inactive);
    const long long CN = (long long)C * N;
    k_feed_mask<<<(int)grid_for(CN, c->device), 256, 0, c->st>>>(d_classes, N, C, active_unary, inactive_unary, s->unary);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// get_inferred into device memory: q float [C][N], copied on the stream
extern "C" int fslic_b200_crfdev_get_inferred(fslic_crf* c, int time, float* d_out, void* stream) {
    CRFDEV_FRAME(c, time, s, stream);
    const size_t CN = (size_t)c->C * c->N;
    if (CN && !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    if (CN) CK(cudaMemcpyAsync(d_out, c->cur ? s->q1 : s->q0, sizeof(float) * CN, cudaMemcpyDeviceToDevice, c->st));
    return FSLIC_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Groups: crfs[0 .. n) are distinct CRFs on one device with the same C and N, typically one per video stream, driven
// in the same launches (CRF_GROUP_MAX members per launch set).  Every call checks all members before it enqueues
// anything, so a refused call changes none of them; it adopts `stream` for every member like crf_adopt_stream, with one
// wait per different stream the members were on; and it leaves each member in the state (cur, stream, frame table,
// stale host copies) its own entry points would have left it in.

static int crf_group_check(fslic_crf* const* crfs, int n, bool need_frames) {
    if (n < 0 || (n && !crfs)) return set_err(FSLIC_EINVAL, "bad group");
    std::unordered_set<const fslic_crf*> seen;
    for (int k = 0; k < n; k++) {
        const fslic_crf* c = crfs[k];
        if (!c) return set_err(FSLIC_EINVAL, "crf is NULL");
        if (!seen.insert(c).second) return set_err(FSLIC_EINVAL, "a CRF is in the group twice");
        if (c->device != crfs[0]->device || c->C != crfs[0]->C || c->N != crfs[0]->N)
            return set_err(FSLIC_EINVAL, "group members differ in device, num_classes or num_nodes");
    }
    if (need_frames)
        for (int k = 0; k < n; k++)
            if (crfs[k]->frames.empty()) return set_err(FSLIC_ENOFRAME, "Time out of range");
    return FSLIC_OK;
}

static int crf_group_adopt(fslic_crf* const* crfs, int n, void* stream) {
    std::vector<cudaStream_t> waited;
    for (int k = 0; k < n; k++) {
        fslic_crf* c = crfs[k];
        if (c->st == (cudaStream_t)stream) continue;
        if (std::find(waited.begin(), waited.end(), c->st) == waited.end()) {
            CK(cudaStreamSynchronize(c->st));
            waited.push_back(c->st);
        }
        c->st = (cudaStream_t)stream;
    }
    return FSLIC_OK;
}

// The newest frame of each of crfs[0 .. n), n <= CRF_GROUP_MAX
static CrfFrameQSet crf_group_newest(fslic_crf* const* crfs, int n) {
    CrfFrameQSet set;
    for (int k = 0; k < n; k++) set.f[k] = crf_frame_q(crfs[k], crfs[k]->frames.back());
    return set;
}

extern "C" int fslic_b200_crfgroup_inference(fslic_crf* const* crfs, int n, unsigned long long max_iter, void* stream) {
    { int rc = crf_group_check(crfs, n, max_iter > 0); if (rc) return rc; }
    if (!n || !max_iter) return FSLIC_OK;
    USE_DEVICE(crfs[0]->device);
    { int rc = crf_group_adopt(crfs, n, stream); if (rc) return rc; }
    for (int k0 = 0; k0 < n; k0 += CRF_GROUP_MAX) {
        int rc = crf_run_chains(crfs + k0, std::min(n - k0, CRF_GROUP_MAX), max_iter, (cudaStream_t)stream);
        if (rc) return rc;
    }
    return FSLIC_OK;
}

extern "C" int fslic_b200_crfdev_group_push_label_frames(fslic_crf* const* crfs, int n, int H, int W, int K,
                                                         const uint16_t* d_labels, const fslic_cluster* d_clusters,
                                                         void* d_scratch, size_t scratch_bytes, void* stream,
                                                         int* times_out) {
    { int rc = crf_group_check(crfs, n, false); if (rc) return rc; }
    if (n && K != crfs[0]->N) return set_err(FSLIC_EINVAL, "K must equal the CRFs' num_nodes");
    { int rc = crfdev_check_push(n, H, W, K, d_labels, d_clusters, d_scratch, scratch_bytes); if (rc) return rc; }
    if (!n) return FSLIC_OK;
    USE_DEVICE(crfs[0]->device);
    { int rc = crf_group_adopt(crfs, n, stream); if (rc) return rc; }
    return crfdev_push(crfs, n, H, W, K, d_labels, d_clusters, d_scratch, (cudaStream_t)stream, times_out);
}

extern "C" int fslic_b200_crfdev_group_set_proba(fslic_crf* const* crfs, int n, const float* d_proba, void* stream) {
    { int rc = crf_group_check(crfs, n, true); if (rc) return rc; }
    if (!n) return FSLIC_OK;
    const long long CN = (long long)crfs[0]->C * crfs[0]->N;
    if (CN && !d_proba) return set_err(FSLIC_EINVAL, "NULL argument");
    const int device = crfs[0]->device;
    USE_DEVICE(device);
    { int rc = crf_group_adopt(crfs, n, stream); if (rc) return rc; }
    if (!CN) return FSLIC_OK;
    for (int k0 = 0; k0 < n; k0 += CRF_GROUP_MAX) {
        const int m = std::min(n - k0, CRF_GROUP_MAX);
        k_feed_proba<<<dim3((unsigned)grid_for(CN, device), (unsigned)m), 256, 0, (cudaStream_t)stream>>>(
            d_proba + (size_t)k0 * CN, crf_group_newest(crfs + k0, m), CN);
        CK(cudaGetLastError());
    }
    return FSLIC_OK;
}

extern "C" int fslic_b200_crfdev_group_reset_inferred(fslic_crf* const* crfs, int n, void* stream) {
    { int rc = crf_group_check(crfs, n, true); if (rc) return rc; }
    if (!n) return FSLIC_OK;
    const int device = crfs[0]->device;
    USE_DEVICE(device);
    { int rc = crf_group_adopt(crfs, n, stream); if (rc) return rc; }
    const long long CN = (long long)crfs[0]->C * crfs[0]->N;
    for (int k0 = 0; k0 < n; k0 += CRF_GROUP_MAX) {
        const int m = std::min(n - k0, CRF_GROUP_MAX);
        int rc = crf_reset_set(crf_group_newest(crfs + k0, m), m, CN, device, (cudaStream_t)stream);
        if (rc) return rc;
    }
    return FSLIC_OK;
}

extern "C" int fslic_b200_crfdev_group_get_inferred(fslic_crf* const* crfs, int n, float* d_out, void* stream) {
    { int rc = crf_group_check(crfs, n, true); if (rc) return rc; }
    if (!n) return FSLIC_OK;
    const long long CN = (long long)crfs[0]->C * crfs[0]->N;
    if (CN && !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    const int device = crfs[0]->device;
    USE_DEVICE(device);
    { int rc = crf_group_adopt(crfs, n, stream); if (rc) return rc; }
    if (!CN) return FSLIC_OK;
    for (int k0 = 0; k0 < n; k0 += CRF_GROUP_MAX) {
        const int m = std::min(n - k0, CRF_GROUP_MAX);
        k_crf_get_q<<<dim3((unsigned)grid_for(CN, device), (unsigned)m), 256, 0, (cudaStream_t)stream>>>(
            crf_group_newest(crfs + k0, m), d_out + (size_t)k0 * CN, CN);
        CK(cudaGetLastError());
    }
    return FSLIC_OK;
}

// pop_frame of every member: the table uploads of all of them, then one wait per stream the members are on.
extern "C" int fslic_b200_crfgroup_pop_frame(fslic_crf* const* crfs, int n, int* times_out) {
    { int rc = crf_group_check(crfs, n, false); if (rc) return rc; }
    if (!n) return FSLIC_OK;
    USE_DEVICE(crfs[0]->device);
    std::vector<std::vector<CrfFrameDev>> tables(n);
    std::vector<cudaStream_t> streams;
    int rc = FSLIC_OK;
    for (int k = 0; k < n; k++) {
        fslic_crf* c = crfs[k];
        if (c->frames.empty()) {
            if (times_out) times_out[k] = -1;
            continue;
        }
        CrfSlot* s = c->frames.front();
        c->frames.pop_front();
        c->pool.push_back(s);
        if (times_out) times_out[k] = s->time;
        if (!rc) rc = crf_stage_table(c, tables[k]);
        if (std::find(streams.begin(), streams.end(), c->st) == streams.end()) streams.push_back(c->st);
    }
    for (cudaStream_t st : streams) CK(cudaStreamSynchronize(st));
    return rc;
}

extern "C" int fslic_b200_debug_logf_host(uint32_t first, long long n, float* h_out) {
    return debug_host_over_bits<glogf::logf>(first, n, h_out);
}

extern "C" int fslic_b200_debug_logf_device(int device, uint32_t first, long long n, float* d_out, void* stream) {
    if (n < 0 || (n && !d_out)) return set_err(FSLIC_EINVAL, "bad buffer");
    if (!n) return FSLIC_OK;
    USE_DEVICE(device);
    k_logf_debug<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(first, n, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
