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
#include <string>
#include <vector>

#include "assign.cuh"
#include "assign5.cuh"
#include "capi_common.h"
#include "realdist.cuh"
#include "lsc.cuh"
#include "preempt.cuh"
#include "cca_stage.h"
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
    CcaDispatch cca;         // the connectivity stage, recorded when enqueued
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
    CcaStage cca;  // connectivity enforcement (cca_stage.cu)
    // staging for the host entry points
    uint8_t* d_img = nullptr;
    fslic_cluster* d_cl = nullptr;
    uint16_t* d_lab = nullptr;
    cudaStream_t own_stream = nullptr, in_stream = nullptr, out_stream = nullptr;
    // second lane of the blocking host path (the two halves of a batch overlap on the device)
    cudaStream_t own_stream2 = nullptr;
    cudaEvent_t front_done = nullptr;
    // the `preemptive` option (preempt.cuh), allocated at the first such call
    uint8_t* pre_cellmap = nullptr;     // [B][ceil(H/2S) * ceil(W/2S)] active 2S x 2S cells
    int* pre_nactive = nullptr;         // [B] active clusters
    float preempt_l1 = 0.f;             // max(roundf(2 S thres), 1) of the call in progress
    std::vector<cudaEvent_t> pipe_ev;  // [2 * chunks]: input-ready / compute-done events of iterate_host
    // timing
    cudaEvent_t ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    float stage_ms[FSLIC_T_COUNT] = {0, 0, 0, 0, 0, 0, 0, 0};
    int last_launches = 0;
    int max_smem_optin = 0;
    // per-launch timing of the dominant kernel (k_assign_tiles on the subsampled passes)
    std::vector<cudaEvent_t> kev;
    int kev_used = 0;
    bool kev_on = false;
    bool pending = false;  // an iterate_host_async batch is in flight on this context's streams
    cudaEvent_t last_work = nullptr;  // end of the last call's device work on this context (CtxOrder)
    // small host batches replay one captured CUDA graph per call instead of ~45 launches
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
    cca_read_dispatch(ctx->disp.cca, out, count);
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
    if (c->last_work) cudaEventSynchronize(c->last_work);  // the last call may still be running on a caller's stream
    void* ptrs[] = {c->d_gamma, c->d_labtbl, c->quad,   c->labels,  c->cinfo,  c->acc,    c->cell_start,
                    c->cinfo_tmp, c->cell_cnt, c->prep_tickets, c->sptable, c->d_img, c->d_cl, c->d_lab};
    for (void* p : ptrs)
        if (p) cudaFree(p);
    cca_stage_destroy(c->cca);
    for (auto& e : c->ev)
        if (e) cudaEventDestroy(e);
    for (auto& e : c->kev) cudaEventDestroy(e);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    if (c->in_stream) cudaStreamDestroy(c->in_stream);
    if (c->out_stream) cudaStreamDestroy(c->out_stream);
    if (c->own_stream2) cudaStreamDestroy(c->own_stream2);
    for (cudaEvent_t e : {c->front_done, c->last_work})
        if (e) cudaEventDestroy(e);
    if (c->gexec) cudaGraphExecDestroy(c->gexec);
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

    CKC(cca_stage_create(c->cca, H, W, max_batch, device_bytes, c->num_sms, c->max_smem_optin));
    for (auto& e : c->ev) CKC(cudaEventCreate(&e));
    CKC(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->in_stream, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->out_stream, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&c->own_stream2, cudaStreamNonBlocking));
    CKC(cudaEventCreateWithFlags(&c->front_done, cudaEventDisableTiming));
    CKC(cudaEventCreateWithFlags(&c->last_work, cudaEventDisableTiming));

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

// ---- order between calls on one context ----------------------------------------------------------------------
// The scratch above belongs to the context, not to a call, and calls may come on any stream: the device entry points
// enqueue on the caller's, the host ones on the context's own non-blocking streams.  So every entry point that touches
// the scratch first makes each stream it computes on wait for `last_work`, and records its own end there: consecutive
// calls on one context run one after the other on the device, whatever streams they use.  A stream that is being
// captured into a CUDA graph neither waits nor records (the capture cannot depend on outside work); fslic_b200_iterate
// waits before iterate_graphed begins its capture and records after the graph's launch.
static bool stream_capturing(cudaStream_t st) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    return cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap != cudaStreamCaptureStatusNone;
}

// Waits for the context's last work on `st` when constructed and, when the call returns, records the call's end on
// `join` (the stream where all of its work comes together; `st` for the device entry points), on every return path:
// work enqueued before an error is ordered too.
struct CtxOrder {
    fslic_ctx* c;
    cudaStream_t join;
    bool on;
    cudaError_t err = cudaSuccess;
    CtxOrder(fslic_ctx* c_, cudaStream_t st, cudaStream_t join_) : c(c_), join(join_), on(!stream_capturing(st)) {
        if (on) err = cudaStreamWaitEvent(st, c->last_work, 0);
    }
    ~CtxOrder() {
        if (on && err == cudaSuccess && cudaEventRecord(c->last_work, join) != cudaSuccess) cudaGetLastError();
    }
};
#define ORDER_CALL_JOIN(c, st, join)                                                                  \
    CtxOrder ctx_order__(c, st, join);                                                                \
    if (ctx_order__.err != cudaSuccess)                                                               \
        return set_err(FSLIC_ECUDA, std::string("cudaStreamWaitEvent: ") + cudaGetErrorString(ctx_order__.err))
#define ORDER_CALL(c, st) ORDER_CALL_JOIN(c, st, st)

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

// ---- connectivity enforcement (cca_stage.cu) ------------------------------------------------------------------
extern "C" int fslic_b200_enforce_connectivity(fslic_ctx* c, uint16_t* d_labels, int batch, int K, int min_threshold,
                                               void* stream) {
    int rc = check_batch(c, batch, false);
    if (rc) return rc;
    if (K <= 0) return FSLIC_OK;  // context.cpp:17
    if (K > 65535) return set_err(FSLIC_EINVAL, "K must fit the u16 label type");
    USE_DEVICE(c->device);
    ORDER_CALL(c, (cudaStream_t)stream);
    c->disp = DispatchRecord();
    return cca_run(c->cca, c->disp.cca, d_labels, d_labels, batch, K, min_threshold, (cudaStream_t)stream, nullptr);
}

extern "C" int fslic_b200_debug_heap_select(fslic_ctx* c, const int32_t* d_area, int n, int middle, uint8_t* d_kept,
                                            void* stream) {
    if (!c) return set_err(FSLIC_EINVAL, "ctx is NULL");
    if (middle + 2 > CCA_HEAP_K || middle < 1 || n < 1) return set_err(FSLIC_EINVAL, "bad n/middle");
    USE_DEVICE(c->device);
    ORDER_CALL(c, (cudaStream_t)stream);
    return cca_heap_select(c->cca, d_area, n, middle, d_kept, (cudaStream_t)stream);
}

// The assign path of an iterate call.  The values are the template arguments of k_assign_real<V> (0..2) and
// k_trace_pass<KIND> (-1, 0..2, 4), and 10 + path is the dispatch record's kernel number of the per-pixel paths.
enum AssignPath {
    PATH_U16 = -1,        // u16 distances: the warp-tile kernels over the spatial patches, or k_assign_generic
    PATH_REAL = 0,        // float-distance contexts (realdist.cuh): ContextRealDist ("standard"),
    PATH_REAL_L2 = 1,     //   ContextRealDistL2,
    PATH_REAL_NOQ = 2,    //   ContextRealDistNoQ
    PATH_PREEMPTIVE = 3,  // the `preemptive` option (preempt.cuh) on the u16 distances
    PATH_LSC = 4,         // ContextLSC (lsc.cuh)
};
static bool float_distances(AssignPath path) { return path != PATH_U16 && path != PATH_PREEMPTIVE; }
static bool uses_patches(AssignPath path) { return !float_distances(path); }
static bool is_preemptive(AssignPath path) { return path == PATH_PREEMPTIVE; }

// Images [first, first + batch) of the context's batched buffers: the front half of an iterate works on one slice
struct Slice {
    int first;
    uint32_t* quad;
    uint16_t* labels;
    CInfo* cinfo;
    int* cell_start;
    unsigned long long* acc;
    CInfo* cinfo_tmp;
    int* cell_cnt;
    unsigned int* prep_tickets;
    uint8_t* pre_cellmap;  // the `preemptive` scratch; null until the first such call
    int* pre_nactive;
};

// Active-cell grid of the `preemptive` option: 2S x 2S cells (preemptive.h:37-38)
static int preempt_cols(const fslic_ctx* c) { return ceil_div(c->W, 2 * c->S); }
static int preempt_cells(const fslic_ctx* c) { return preempt_cols(c) * ceil_div(c->H, 2 * c->S); }

static Slice slice_at(const fslic_ctx* c, int first) {
    const size_t b = (size_t)first, N = (size_t)c->N, K = (size_t)c->K, cells = (size_t)c->ncell + 1;
    Slice s;
    s.first = first;
    s.quad = c->quad + b * N;
    s.labels = c->labels + b * N;
    s.cinfo = c->cinfo + b * K;
    s.cell_start = c->cell_start + b * cells;
    s.acc = c->acc + b * K * 4;
    s.cinfo_tmp = c->cinfo_tmp + b * K;
    s.cell_cnt = c->cell_cnt + b * cells;
    s.prep_tickets = c->prep_tickets + b;
    s.pre_cellmap = c->pre_cellmap ? c->pre_cellmap + b * preempt_cells(c) : nullptr;
    s.pre_nactive = c->pre_nactive ? c->pre_nactive + b : nullptr;
    return s;
}

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
    c->spt_stream = st;  // a call on another stream rebuilds (ordered after this build by CtxOrder all the same)
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

// The fields every assign and trace kernel shares: geometry, the rows of the pass, the freshness test, the cell grid and
// the spatial term.  Everything else is zero.
static AssignParams base_params(const fslic_ctx* c, int batch, int stride, int rem, int cfg_stride, int fresh_from,
                                float coef) {
    AssignParams ap;
    memset(&ap, 0, sizeof(ap));
    ap.H = c->H; ap.W = c->W; ap.K = c->K; ap.S = c->S; ap.B = batch;
    ap.stride = stride; ap.rem = rem;
    ap.nsub = (c->H - rem + stride - 1) / stride;
    ap.cfg_stride = cfg_stride; ap.fresh_from = fresh_from;
    ap.G = c->G; ap.cellW = c->cellW; ap.cellH = c->cellH; ap.ncell = c->ncell;
    ap.coef = coef;
    ap.manhattan = c->manhattan;
    return ap;
}

// CTAs of 256 threads for a per-pixel grid-stride kernel: one per 256 pixels, at most `per_sm` per SM
static long pixel_grid(const fslic_ctx* c, long px, int per_sm = 32) {
    const long grid = (px + 255) / 256, cap = (long)c->num_sms * per_sm;
    return grid > cap ? cap : grid;
}

// Grows an event pool to at least n events
static int ensure_events(std::vector<cudaEvent_t>& ev, int n, unsigned flags) {
    while ((int)ev.size() < n) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, flags));
        ev.push_back(e);
    }
    return FSLIC_OK;
}

// Records the start of a timed launch on `st` when `on`, and hands out the event that marks its end (null when off).
static int timed_launch(std::vector<cudaEvent_t>& ev, int& used, bool on, cudaStream_t st, cudaEvent_t* end) {
    *end = nullptr;
    if (!on) return FSLIC_OK;
    int rc = ensure_events(ev, used + 2, cudaEventDefault);
    if (rc) return rc;
    CK(cudaEventRecord(ev[used++], st));
    *end = ev[used++];
    return FSLIC_OK;
}

// ---- the per-pixel kernels: one thread per pixel of the pass over the cell grid ----
static void launch_preempt(fslic_ctx* c, const Slice& sl, const AssignParams& ap, const fslic_cluster* cl, cudaStream_t st) {
    const long px = (long)ap.nsub * c->W * ap.B, grid = pixel_grid(c, px);
    k_assign_preempt<true><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, cl, sl.acc,
                                                      sl.pre_cellmap, preempt_cols(c), preempt_cells(c), sl.pre_nactive);
    record_pass(c, true, 10 + PATH_PREEMPTIVE, 1, grid, 256, px);
}

static void launch_lsc(fslic_ctx* c, const Slice& sl, const AssignParams& ap, bool update, cudaStream_t st) {
    const long px = (long)ap.nsub * c->W * ap.B, grid = pixel_grid(c, px);
    if (update)
        k_assign_lsc<true><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, c->lsc_feat, c->lsc_cf,
                                                      sl.acc, c->lsc_box);
    else
        k_assign_lsc<false><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, c->lsc_feat, c->lsc_cf,
                                                       sl.acc, c->lsc_box);
    record_pass(c, update, 10 + PATH_LSC, 1, grid, 256, px);
}

// The NoQ variant reads its float centroids from the cluster records `cl` themselves
template <int V>
static void launch_real_v(const Slice& sl, const AssignParams& ap, bool update, const fslic_cluster* cl, long grid,
                          cudaStream_t st) {
    if (update)
        k_assign_real<V, true><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, cl, sl.acc);
    else
        k_assign_real<V, false><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, cl, sl.acc);
}
static void launch_real(fslic_ctx* c, const Slice& sl, const AssignParams& ap, AssignPath path, bool update,
                        const fslic_cluster* cl, cudaStream_t st) {
    const long px = (long)ap.nsub * c->W * ap.B, grid = pixel_grid(c, px);
    if (path == PATH_REAL) launch_real_v<PATH_REAL>(sl, ap, update, cl, grid, st);
    else if (path == PATH_REAL_L2) launch_real_v<PATH_REAL_L2>(sl, ap, update, cl, grid, st);
    else launch_real_v<PATH_REAL_NOQ>(sl, ap, update, cl, grid, st);
    record_pass(c, update, 10 + path, 1, grid, 256, px);
}

static void launch_generic(fslic_ctx* c, const Slice& sl, const AssignParams& ap, bool update, cudaStream_t st) {
    const long px = (long)ap.nsub * c->W * ap.B, grid = pixel_grid(c, px, 64);
    record_pass(c, update, 0, 1, grid, 256, px);
    if (update)
        k_assign_generic<true><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, sl.acc);
    else
        k_assign_generic<false><<<(int)grid, 256, 0, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, sl.acc);
}

// ---- the warp-tile kernels over the spatial patch in shared memory ----
// The TMA-staged kernel.  Sets *launched = false and launches nothing where it does not apply: row strides of the tensor
// maps must be multiples of 16 bytes (W % 8 == 0 for the u16 labels), the sub-row pitch is an immediate of its patch
// loads (stride 3 with the update, 1 without), and its per-warp shared blocks must fit beside the patch.
// fuse_clusters / fused_out: when it takes an update pass of a small batch, its last CTA also does the bookkeeping for
// the NEXT pass (prepare_in_tail) on these cluster records; *fused_out tells the caller to skip k_prepare.
static int launch_tma_tiles(fslic_ctx* c, const Slice& sl, AssignParams ap, const PassGeom& g, bool update, cudaStream_t st,
                            fslic_cluster* fuse_clusters, bool* fused_out, bool* launched) {
    *launched = false;
    const int batch = ap.B, stride = ap.stride;
    if (!((c->W % 8) == 0 && g.TS <= 256 && (update ? stride == 3 : stride == 1) &&
          (long)ceil_div(c->W, 32) * ap.tiles_y * batch < (1L << 30) && tensor_map_encoder() != nullptr))
        return FSLIC_OK;
    const size_t tblb = align_up((size_t)g.tbl_elems * 2, 128);
    int warps5 = 0;
    for (int w : {32, 16, 8}) {
        if (tblb + (size_t)w * A5_WBLK <= (size_t)(c->max_smem_optin - 1024)) {
            warps5 = w;
            break;
        }
    }
    if (!warps5) return FSLIC_OK;
    // super tiles of 4 tiles when that still gives every warp of the grid work and the union list stays well below
    // its 32 slots; single tiles otherwise (single images, small S)
    const double est4 = (double)(2 * c->S + stride * 3 + 1) * (2 * c->S + 128) / ((double)c->S * c->S);
    const long supers4 = (long)ceil_div(ap.tiles_x, 4) * ap.tiles_y * batch;
    const int tps = (est4 <= 24.0 && supers4 >= (long)c->num_sms * warps5) ? 4 : 1;
    ap.tps = tps;
    CUtensorMap tmq, tml;
    if (!make_subrow_map(&tmq, CU_TENSOR_MAP_DATA_TYPE_UINT32, 4, sl.quad, c->H, c->W, batch, stride, ap.rem, ap.nsub, 32 * tps) ||
        !make_subrow_map(&tml, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, sl.labels, c->H, c->W, batch, stride, ap.rem, ap.nsub, 32 * tps))
        return FSLIC_OK;
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
    } else if (supers < (long)c->num_sms * warps5) {
        // not even one super tile per warp (single images): spread them over all SMs instead of filling a few
        warps5 = std::min(warps5, std::max(4, (int)ceil_div((int)supers, c->num_sms)));
    }
    size_t smem5 = tblb + (size_t)warps5 * A5_WBLK;
    const size_t tail_smem = prepare_tail_smem_bytes(c->K, c->ncell);
    if (update && fuse_clusters && fused_out && batch <= 2 && c->K <= 4096 && tail_smem <= (size_t)(c->max_smem_optin - 1024)) {
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
    ap.tbl_bytes = (uint32_t)tblb;
    ap.cinfo_img_bytes = (uint32_t)c->K * (uint32_t)sizeof(CInfo);
    ap.cells_img_bytes = (uint32_t)(c->ncell + 1) * 4u;
    ap.acc_img_bytes = (uint32_t)c->K * 32u;
    const uint16_t* tbl = c->sptable + (update ? 0 : SPT_MAX_ELEMS);
    cudaEvent_t end;
    int rc = timed_launch(c->kev, c->kev_used, c->kev_on && update, st, &end);
    if (rc) return rc;
    fn<<<(int)grid, 32 * warps5, smem5, st>>>(ap, tmq, tml, sl.quad, sl.labels, sl.cinfo, sl.cell_start, sl.acc, tbl,
                                              fuse_clusters, sl.cinfo, sl.cell_start, sl.prep_tickets);
    if (end) CK(cudaEventRecord(end, st));
    record_pass(c, update, 5, tps, grid, warps5, supers);
    *launched = true;
    return FSLIC_OK;
}

// The LDG warp-tile kernel: every pass whose patch fits shared memory but that the TMA-staged kernel does not take
static int launch_ldg_tiles(fslic_ctx* c, const Slice& sl, AssignParams ap, const PassGeom& g, bool update, cudaStream_t st) {
    const uint16_t* tbl = c->sptable + (update ? 0 : SPT_MAX_ELEMS);
    const assign_fn fn = pick_assign(g.TS, ap.stride, update);
    int occ = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, AS_THREADS, g.smem);
    if (occ < 1) occ = 1;
    long grid = (long)c->num_sms * occ;
    // small launches (single images): one tile per warp step so that every SM gets work
    ap.tps = ((long)ap.ntiles * ap.B < (long)c->num_sms * occ * AS_WARPS * AS_T) ? 1 : AS_T;
    const long supers = (long)ceil_div(ap.tiles_x, ap.tps) * ap.tiles_y * ap.B;
    const long need = (supers + AS_WARPS - 1) / AS_WARPS;
    if (grid > need) grid = need;
    cudaEvent_t end;
    int rc = timed_launch(c->kev, c->kev_used, c->kev_on && update, st, &end);
    if (rc) return rc;
    fn<<<(int)grid, AS_THREADS, g.smem, st>>>(ap, sl.quad, sl.labels, sl.cinfo, sl.cell_start, sl.acc, tbl);
    if (end) CK(cudaEventRecord(end, st));
    record_pass(c, update, 4, ap.tps, grid, AS_WARPS, supers);
    return FSLIC_OK;
}

// One assign pass over the rows rem, rem + stride, ... of a slice.  The u16 passes take the warp-tile kernels, or the
// generic kernel when the patch cannot live in shared memory; see launch_tma_tiles for fuse_clusters / fused_out.
static int run_assign_pass(fslic_ctx* c, const Slice& sl, int batch, int stride, int rem, int cfg_stride, int fresh_from,
                           bool update, float coef, cudaStream_t st, int* launches, AssignPath path,
                           const fslic_cluster* d_clusters = nullptr, fslic_cluster* fuse_clusters = nullptr,
                           bool* fused_out = nullptr) {
    if (fused_out) *fused_out = false;
    AssignParams ap = base_params(c, batch, stride, rem, cfg_stride, fresh_from, coef);
    if (ap.nsub <= 0) return FSLIC_OK;
    if (is_preemptive(path) && update) {  // the full assign of the `preemptive` option is the ordinary one
        launch_preempt(c, sl, ap, d_clusters, st);
    } else if (path == PATH_LSC) {
        launch_lsc(c, sl, ap, update, st);
    } else if (float_distances(path)) {
        launch_real(c, sl, ap, path, update, d_clusters, st);
    } else {
        const PassGeom g = pass_geometry(c, stride);
        ap.Ginv = (uint32_t)(((1ull << 32) + (unsigned)c->G - 1) / (unsigned)c->G);
        ap.OY = g.OY; ap.OX = g.OX; ap.TS = g.TS; ap.tbl_elems = g.tbl_elems;
        ap.tiles_x = ceil_div(c->W, 32);
        ap.tiles_y = ceil_div(ap.nsub, g.R);
        ap.ntiles = ap.tiles_x * ap.tiles_y;
        ap.tps = AS_T;
        bool launched = false;
        int rc = FSLIC_OK;
        if (g.fast) rc = launch_tma_tiles(c, sl, ap, g, update, st, fuse_clusters, fused_out, &launched);
        if (!rc && g.fast && !launched) rc = launch_ldg_tiles(c, sl, ap, g, update, st);
        if (rc) return rc;
        if (!g.fast) launch_generic(c, sl, ap, update, st);
    }
    if (launches) *launches += 1;
    CK(cudaGetLastError());
    return FSLIC_OK;
}

static int run_prepare(fslic_ctx* c, const Slice& sl, fslic_cluster* d_clusters, int batch, int first, int finalize,
                       cudaStream_t st, int* launches, int noq = 0, int preempt = 0, int last = 0) {
    PrepParams pp = prep_params(c->H, c->W, c->K, c->S, c->G, c->cellW, c->cellH, c->ncell);
    pp.first = first; pp.finalize = finalize; pp.last = last; pp.noq = noq;
    pp.preempt = preempt; pp.l1_thres = c->preempt_l1; pp.nactive = preempt ? sl.pre_nactive : nullptr;
    const size_t smem = (size_t)(c->ncell + 2) * sizeof(int);
    if (preempt) {  // k_prepare carries the option's bookkeeping; after an update k_preempt_mark derives the active set
        k_prepare<<<batch, 1024, smem, st>>>(pp, d_clusters, sl.acc, sl.quad, sl.cinfo, sl.cell_start, sl.cinfo_tmp);
        c->disp.prepare = 1;
        if (launches) *launches += 1;
        if (finalize && !last) {
            k_preempt_mark<<<batch, 1024, 0, st>>>(c->K, c->S, c->H, c->W, c->G, c->cellW, c->cellH, c->ncell, d_clusters,
                                                   sl.cinfo, sl.cell_start, sl.pre_cellmap, preempt_cols(c),
                                                   preempt_cells(c), sl.pre_nactive);
            if (launches) *launches += 1;
        }
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    // k_prepare2 (one thread per cluster, several CTAs per image) is quicker for a handful of images (single image:
    // 0.412 vs 0.431 ms per blocking call); with a full batch its extra CTAs only contend (18 vs 13 us at 32 images)
    if (c->K <= 1024 * PREP3_PER) {
        k_prepare3<<<batch, 1024, smem, st>>>(pp, d_clusters, sl.acc, sl.quad, sl.cinfo, sl.cell_start);
        c->disp.prepare = 3;
    } else if (batch >= 8) {
        k_prepare<<<batch, 1024, smem, st>>>(pp, d_clusters, sl.acc, sl.quad, sl.cinfo, sl.cell_start, sl.cinfo_tmp);
        c->disp.prepare = 1;
    } else {
        k_prepare2<<<dim3(ceil_div(c->K, 256), batch), 256, smem, st>>>(pp, d_clusters, sl.acc, sl.quad, sl.cinfo,
                                                                         sl.cell_start, sl.cinfo_tmp, sl.cell_cnt,
                                                                         sl.prep_tickets);
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
static int lsc_before_iteration(fslic_ctx* c, const Slice& sl, const fslic_cluster* d_clusters, int batch,
                                const fslic_params* p, cudaStream_t st, int* launches) {
    uint32_t key;
    memcpy(&key, &p->compactness, 4);
    if (!c->lsc_tab_valid || key != c->lsc_tab_key) {
        build_lsc_tables(c->H, c->W, c->S, p->compactness, c->lsc_htab);
        // pageable source: the copy is staged before cudaMemcpyAsync returns, so the vector may change afterwards
        CK(cudaMemcpyAsync(c->lsc_tab, c->lsc_htab.data(), c->lsc_htab.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        c->lsc_tab_key = key;
        c->lsc_tab_valid = true;
    }
    k_lsc_means<<<batch * LSC_NF, 32, 0, st>>>(sl.quad, c->lsc_tab, c->H, c->W, c->lsc_means);
    const long px = (long)c->N * batch, grid = pixel_grid(c, px);
    k_lsc_features<<<(int)grid, 256, 0, st>>>(sl.quad, c->lsc_tab, c->H, c->W, batch, c->lsc_means, c->lsc_feat, c->lsc_w);
    c->disp.lsc_trips = (int)((px + grid * 256 - 1) / (grid * 256));
    k_lsc_centroids<<<ceil_div(batch * c->K, 256), 256, 0, st>>>(c->lsc_feat, c->H, c->W, c->K, c->S, batch, d_clusters,
                                                                 c->lsc_cf, c->lsc_cf_init, c->lsc_box);
    if (launches) *launches += 3;
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// after_update (lsc.cpp:226-307) of the pass just assigned; timed launch by launch when collect_timing is on.
static int lsc_after_update(fslic_ctx* c, const Slice& sl, int batch, int stride, cudaStream_t st, int* launches,
                            bool timing) {
    cudaEvent_t end;
    int rc = timed_launch(c->lev, c->lev_used, timing, st, &end);
    if (rc) return rc;
    k_lsc_after_update<<<ceil_div(batch * c->K, LSC_AU_WARPS), LSC_AU_WARPS * 32, 0, st>>>(
        c->H, c->W, c->K, batch, stride, sl.labels, c->lsc_feat, c->lsc_w, c->lsc_cf, c->lsc_box);
    if (end) CK(cudaEventRecord(end, st));
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
static int trace_begin(fslic_ctx* c, int batch, int max_iter, AssignPath path, cudaStream_t st) {
    c->tr_T = 0;
    const int T = max_iter + 1, db = float_distances(path) ? 4 : 2;
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
static int trace_seed(fslic_ctx* c, const Slice& sl, const fslic_cluster* d_clusters, int batch, cudaStream_t st,
                      int* launches) {
    const size_t N = c->N, T = c->tr_T;
    k_trace_seed<<<ceil_div(batch * c->K, 256), 256, 0, st>>>(c->H, c->W, c->K, batch, sl.quad, d_clusters, tr_clusters(c),
                                                             (long long)T * c->K);
    CK(cudaGetLastError());
    CK(cudaMemset2DAsync(tr_assign(c), T * N * 2, 0xFF, N * 2, batch, st));
    CK(cudaMemset2DAsync(tr_dist(c), T * N * c->tr_dist_bytes, 0, N * c->tr_dist_bytes, batch, st));
    (*launches)++;
    return FSLIC_OK;
}

// Assignment and minimum distances after update pass `it` (slot it + 1), from the records that pass read.  Runs before
// the next prepare rewrites them and, for LSC, before after_update.
template <int KIND>
static void launch_trace(const Slice& sl, const TraceParams& tp, long grid, const fslic_cluster* d_clusters, uint16_t* oa,
                         void* od, unsigned int* bad, cudaStream_t st) {
    k_trace_pass<KIND><<<(int)grid, 256, 0, st>>>(tp, sl.quad, sl.labels, sl.cinfo, sl.cell_start, d_clusters, oa, od, bad);
}
static int trace_pass(fslic_ctx* c, const Slice& sl, int batch, int it, int stride, int rem, float coef, AssignPath path,
                      const fslic_cluster* d_clusters, cudaStream_t st, int* launches) {
    TraceParams tp;
    memset(&tp, 0, sizeof(tp));
    tp.ap = base_params(c, batch, stride, rem, stride, 0, coef);
    tp.fresh_after = it + 1;
    tp.preempt = is_preemptive(path);
    tp.img_pitch = (long long)c->tr_T * c->N;
    tp.feat = c->lsc_feat;
    tp.cf = c->lsc_cf;
    const size_t slot = (size_t)(it + 1) * c->N;
    uint16_t* oa = tr_assign(c) + slot;
    void* od = tr_dist(c) + slot * c->tr_dist_bytes;
    const long grid = pixel_grid(c, (long)c->N * batch);
    if (path == PATH_REAL) launch_trace<PATH_REAL>(sl, tp, grid, d_clusters, oa, od, c->tr_bad, st);
    else if (path == PATH_REAL_L2) launch_trace<PATH_REAL_L2>(sl, tp, grid, d_clusters, oa, od, c->tr_bad, st);
    else if (path == PATH_REAL_NOQ) launch_trace<PATH_REAL_NOQ>(sl, tp, grid, d_clusters, oa, od, c->tr_bad, st);
    else if (path == PATH_LSC) launch_trace<PATH_LSC>(sl, tp, grid, d_clusters, oa, od, c->tr_bad, st);
    else launch_trace<PATH_U16>(sl, tp, grid, d_clusters, oa, od, c->tr_bad, st);  // the preemptive option too
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
                         bool lab_done = false, AssignPath path = PATH_U16) {
    const Slice sl = slice_at(c, b0);
    int rc = FSLIC_OK;
    if (!lab_done) rc = launch_lab(c, d_images, sl.quad, batch, p->convert_to_lab, st);  // else: the caller ran it
    if (rc) return rc;
    (*launches)++;
    if (timing) CK(cudaEventRecord(c->ev[1], st));
    if (path == PATH_LSC) {  // before_iteration (context.cpp:151-154)
        rc = lsc_before_iteration(c, sl, d_clusters, batch, p, st, launches);
        if (rc) return rc;
        if (timing) CK(cudaEventRecord(c->ev[5], st));
    }
    const int stride = p->subsample_stride;
    const int noq = path == PATH_REAL_NOQ ? 1 : 0;
    const int preempt = is_preemptive(path) ? 1 : 0;
    if (uses_patches(path)) {
        rc = build_patches(c, stride, p->max_iter > 0, coef, st, launches);
        if (rc) return rc;
    }
    // debug_mode: snapshots between the stages below; a traced call never fuses the next prepare into an assign tail
    const bool trace = c->trace_on;
    if (trace) {
        rc = trace_seed(c, sl, d_clusters, batch, st, launches);
        if (rc) return rc;
    }
    int rem = 0;
    bool prepared = false;  // the previous assign+update launch already did the bookkeeping in its tail
    for (int it = 0; it < p->max_iter; it++) {
        if (!prepared) {
            rc = run_prepare(c, sl, d_clusters, batch, it == 0, it > 0, st, launches, noq, preempt, 0);
            if (rc) return rc;
            if (trace && it > 0) rc = trace_clusters(c, d_clusters, batch, it, st);
            if (rc) return rc;
        }
        rc = run_assign_pass(c, sl, batch, stride, rem, stride, it, true, coef, st, launches, path, d_clusters,
                             path == PATH_U16 && !trace ? d_clusters : nullptr, &prepared);
        if (rc) return rc;
        if (trace) {
            rc = trace_pass(c, sl, batch, it, stride, rem, coef, path, d_clusters, st, launches);
            if (rc) return rc;
        }
        if (path == PATH_LSC) {  // after_update (context.cpp:169-172); its Cluster update is the next prepare's
            rc = lsc_after_update(c, sl, batch, stride, st, launches, timing);
            if (rc) return rc;
        }
        rem = (rem + 1) % stride;
    }
    if (timing) CK(cudaEventRecord(c->ev[2], st));
    if (!prepared) {
        // The last snapshot precedes PreemptiveGrid::finalize (context.cpp:173-176): a traced `preemptive` call lets this
        // prepare derive the final update's active set like the earlier ones, records it, then sets every is_active.
        const bool hold = trace && preempt && p->max_iter > 0;
        rc = run_prepare(c, sl, d_clusters, batch, p->max_iter == 0, p->max_iter > 0, st, launches, noq, preempt, hold ? 0 : 1);
        if (rc) return rc;
        if (trace && p->max_iter > 0) rc = trace_clusters(c, d_clusters, batch, p->max_iter, st);
        if (rc) return rc;
        if (hold) {
            k_trace_activate<<<ceil_div(batch * c->K, 256), 256, 0, st>>>(d_clusters, batch * c->K);
            CK(cudaGetLastError());
            (*launches)++;
        }
    }
    return run_assign_pass(c, sl, batch, 1, 0, stride, p->max_iter < stride ? p->max_iter : stride, false, coef, st,
                           launches, path, d_clusters);
}

// Back half (context.cpp:191-194): connectivity enforcement of images [0, batch) of c->labels into d_labels.
static int iterate_back(fslic_ctx* c, uint16_t* d_labels, int batch, const fslic_params* p, cudaStream_t st, int* launches,
                        HostOut* ho = nullptr, int slot = 0, int lane = 0) {
    const int thres = (int)round((double)(c->S * c->S) * (double)p->min_size_factor);  // context.cpp:16
    return cca_run(c->cca, c->disp.cca, c->labels + (size_t)slot * c->N, d_labels, batch, c->K, thres, st, launches, ho, slot,
                   lane);
}

static int iterate_plain(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                         int batch, const fslic_params* p, void* stream, bool lab_done = false,
                         AssignPath path = PATH_U16) {
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
    cca_set_timing(c->cca, timing);
    if (c->trace_on) {
        rc = trace_begin(c, batch, p->max_iter, path, st);
        if (rc) return rc;
    }
    if (timing) CK(cudaEventRecord(c->ev[0], st));
    rc = iterate_front(c, 0, d_images, d_clusters, batch, p, coef, st, &launches, timing, lab_done, path);
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
        if (path == PATH_LSC) {  // before_iteration and the after_update launches are their own stages
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
        cca_read_timing(c->cca);
        c->assign_kernel_ms = 0.f;
        c->assign_kernel_launches = 0;
        for (int i = 0; i + 1 < c->kev_used; i += 2) {
            CK(cudaEventElapsedTime(&ms, c->kev[i], c->kev[i + 1]));
            c->assign_kernel_ms += ms;
            c->assign_kernel_launches++;
        }
    }
    c->last_launches = launches;
    cca_set_timing(c->cca, false);
    return FSLIC_OK;
}

extern "C" int fslic_b200_cca_stage_ms(fslic_ctx* c, float* out_ms, int count) {
    if (!c || !out_ms) return set_err(FSLIC_EINVAL, "NULL argument");
    cca_read_ms(c->cca, out_ms, count);
    return FSLIC_OK;
}

// What a captured graph depends on besides the images: the cluster and label buffers, the batch and the parameters
static void graph_key(const fslic_ctx* c, const fslic_cluster* d_clusters, const uint16_t* d_labels, int batch,
                      const fslic_params* p, fslic_ctx::GraphKey* k) {
    memset(k, 0, sizeof(*k));  // memcmp'd: the padding must be zero too
    k->img = nullptr; k->cl = d_clusters; k->lab = d_labels; k->batch = batch; k->p = *p; k->manhattan = c->manhattan;
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
    graph_key(c, d_clusters, d_labels, batch, p, &k);
    {
        USE_DEVICE(c->device);
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

// Public entry.  A small batch is ~45 launches of kernels that each run a few microseconds: when the same buffers,
// batch and parameters come back (second consecutive call) the call is captured into a CUDA graph once and replayed
// from then on.  Needs a capturable stream (not the legacy default stream) and no timing; anything else launches plainly.
extern "C" int fslic_b200_iterate(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                                  int batch, const fslic_params* p, void* stream) {
    if (!c) return set_err(FSLIC_EINVAL, "ctx is NULL");
    // (the wait is enqueued before iterate_graphed begins a capture: the graph's launch waits, the graph itself does not)
    ORDER_CALL(c, (cudaStream_t)stream);
    // A traced call launches plainly and leaves the graph and its key alone: the next untraced call replays as before.
    if (c && p && !c->trace_on && batch > 0 && batch < 4 && p->collect_timing == 0 && stream != nullptr) {
        fslic_ctx::GraphKey k;
        graph_key(c, d_clusters, d_labels, batch, p, &k);
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
    if (!c) return set_err(FSLIC_EINVAL, "ctx is NULL");
    ORDER_CALL(c, (cudaStream_t)stream);
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream, false, (AssignPath)variant);
}

// The reference's ContextLSC (src/lsc.cpp; cfast_slic.pyx:207-214) driven with num_threads = 1 (lsc.cuh).
extern "C" int fslic_b200_iterate_lsc(fslic_ctx* c, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                                      int batch, const fslic_params* p, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    USE_DEVICE(c->device);
    rc = ensure_lsc(c);
    if (rc) return rc;
    ORDER_CALL(c, (cudaStream_t)stream);
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream, false, PATH_LSC);
}

extern "C" int fslic_b200_debug_lsc_stages(fslic_ctx* c, float* d_means_out, float* d_weights_out, float* d_cinit_out,
                                           int batch, void* stream) {
    int rc = check_batch(c, batch);
    if (rc) return rc;
    if (!c->lsc_feat) return set_err(FSLIC_EINVAL, "no LSC iterate has run on this context");
    USE_DEVICE(c->device);
    cudaStream_t st = (cudaStream_t)stream;
    ORDER_CALL(c, st);
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
    ORDER_CALL(c, (cudaStream_t)stream);
    return iterate_plain(c, d_images, d_clusters, d_labels, batch, p, stream, false, PATH_PREEMPTIVE);
}

extern "C" int fslic_b200_assign_kernel_time(fslic_ctx* c, float* total_ms, int* launches) {
    if (!c || !total_ms || !launches) return set_err(FSLIC_EINVAL, "NULL argument");
    *total_ms = c->assign_kernel_ms;
    *launches = c->assign_kernel_launches;
    return FSLIC_OK;
}

extern "C" int fslic_b200_debug_cca_counters(fslic_ctx* c, int32_t* out8, int image) {
    if (!c || !out8 || image < 0 || image >= c->cca.batch) return set_err(FSLIC_EINVAL, "bad argument");
    USE_DEVICE(c->device);
    return cca_read_counters(c->cca, out8, image);
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
    ORDER_CALL(c, st);
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
    ORDER_CALL(c, st);
    const size_t ib = (size_t)batch * c->N * 3, cb = (size_t)batch * c->K * sizeof(fslic_cluster);
    CK(cudaMemcpyAsync(c->d_img, h_images, ib, cudaMemcpyHostToDevice, st));
    rc = fslic_b200_initialize_clusters(c, c->d_img, c->d_cl, batch, st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h_clusters, c->d_cl, cb, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return FSLIC_OK;
}

// H2D of images [s0, s0 + n) and their cluster records into the staging buffers on in_stream; `ready` marks the end
static int upload_slice(fslic_ctx* c, const uint8_t* h_images, const fslic_cluster* h_clusters, int s0, int n,
                        cudaEvent_t ready) {
    const size_t N = (size_t)c->N, K = (size_t)c->K;
    CK(cudaMemcpyAsync(c->d_img + s0 * N * 3, h_images + s0 * N * 3, n * N * 3, cudaMemcpyHostToDevice, c->in_stream));
    CK(cudaMemcpyAsync(c->d_cl + s0 * K, h_clusters + s0 * K, n * K * sizeof(fslic_cluster), cudaMemcpyHostToDevice,
                       c->in_stream));
    CK(cudaEventRecord(ready, c->in_stream));
    return FSLIC_OK;
}

// D2H of the label maps (unless the connectivity stage already copied them) and cluster records of images [s0, s0 + n)
// on out_stream, behind the work enqueued so far on `cs`; `done` is the event that hands over
static int download_slice(fslic_ctx* c, uint16_t* h_labels, fslic_cluster* h_clusters, int s0, int n, bool labels_copied,
                          cudaStream_t cs, cudaEvent_t done) {
    const size_t N = (size_t)c->N, K = (size_t)c->K;
    CK(cudaEventRecord(done, cs));
    CK(cudaStreamWaitEvent(c->out_stream, done, 0));
    if (!labels_copied)
        CK(cudaMemcpyAsync(h_labels + s0 * N, c->d_lab + s0 * N, n * N * 2, cudaMemcpyDeviceToHost, c->out_stream));
    CK(cudaMemcpyAsync(h_clusters + s0 * K, c->d_cl + s0 * K, n * K * sizeof(fslic_cluster), cudaMemcpyDeviceToHost,
                       c->out_stream));
    return FSLIC_OK;
}

// A blocking call of 16..64 images in one chunk: the caller waits anyway, so the two halves run as two independent
// pipelines that overlap on the device -- half A's connectivity stage (incl. the ~0.7 ms std::partial_sort replay of its
// ambiguous images, a handful of SMs) and its label download run while half B is still on the wire / in its assign
// passes.  Each half has its own compute + side stream and its own window of the scratch arrays.
static int iterate_host_lanes(fslic_ctx* c, const uint8_t* h_images, fslic_cluster* h_clusters, uint16_t* h_labels, int nb,
                              const fslic_params* pp, float coef) {
    const size_t N = (size_t)c->N, K = (size_t)c->K;
    const int h0 = nb / 2, s0[2] = {0, h0}, sn[2] = {h0, nb - h0};
    cudaStream_t const cs[2] = {c->own_stream, c->own_stream2};
    cudaEvent_t const up[2] = {c->pipe_ev[2], c->pipe_ev[0]};
    int launches = 0, rc;
    CK(cudaStreamWaitEvent(c->own_stream2, c->last_work, 0));
    for (int h = 0; h < 2; h++) {
        rc = upload_slice(c, h_images, h_clusters, s0[h], sn[h], up[h]);
        if (rc) return rc;
    }
    for (int h = 0; h < 2; h++) {  // both front halves first: nothing in them waits for the host
        CK(cudaStreamWaitEvent(cs[h], up[h], 0));
        // (the second front half starts behind the first: they share the cached spatial patches, which the first
        //  call may still be building, and the first half's data is there earlier anyway)
        if (h) CK(cudaStreamWaitEvent(cs[h], c->front_done, 0));
        rc = iterate_front(c, s0[h], c->d_img + s0[h] * N * 3, c->d_cl + s0[h] * K, sn[h], pp, coef, cs[h], &launches, false);
        if (rc) return rc;
        if (!h) CK(cudaEventRecord(c->front_done, cs[h]));
    }
    for (int h = 0; h < 2; h++) {  // back halves: each reads its per-image decisions back mid-way
        HostOut ho = {h_labels + s0[h] * N, c->out_stream, false};
        rc = iterate_back(c, c->d_lab + s0[h] * N, sn[h], pp, cs[h], &launches, &ho, s0[h], h);
        if (rc) return rc;
        rc = download_slice(c, h_labels, h_clusters, s0[h], sn[h], ho.done, cs[h], c->pipe_ev[1]);
        if (rc) return rc;
    }
    c->last_launches = launches;
    c->pending = true;
    CK(cudaStreamSynchronize(c->out_stream));
    CK(cudaStreamSynchronize(c->own_stream));
    CK(cudaStreamSynchronize(c->own_stream2));
    c->pending = false;
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
    // The compute streams start behind the context's last work (own_stream2 in iterate_host_lanes); the call's work
    // joins on out_stream, behind the label and cluster downloads.  in_stream only fills the staging buffers, which no
    // other call touches while this one runs: host calls wait for a pending one above, device calls never use them.
    ORDER_CALL_JOIN(c, c->own_stream, c->out_stream);
    c->disp = DispatchRecord();
    // Software pipeline over chunks of the batch: H2D(chunk i+1) | compute(chunk i) | D2H(chunk i-1) on three
    // streams, so for batches the PCIe copies hide behind the kernels (and vice versa).  With pinned host
    // buffers the copies are truly asynchronous; pageable buffers still work, just without overlap.
    const size_t N = (size_t)c->N, K = (size_t)c->K;
    // chunks of 32: smaller chunks would pay the fixed latencies of the pipeline (notably the sequential
    // std::partial_sort replay of ambiguous images) once per chunk, which costs more than the overlap wins
    int chunk = batch < 32 ? batch : 32;
    if (const char* e = getenv("FSLIC_HOST_CHUNK")) {  // test hook: force the multi-chunk pipeline
        const int v = atoi(e);
        if (v >= 1 && v < chunk) chunk = v;
    }
    const int nchunks = (batch + chunk - 1) / chunk;
    rc = ensure_events(c->pipe_ev, 3 * nchunks, cudaEventDisableTiming);
    if (rc) return rc;
    fslic_params pp = *p;
    if (nchunks > 1) pp.collect_timing = 0;  // per-stage timings are only meaningful for an unchunked run
    for (int k = 0; k < nchunks; k++) {
        const int b0 = k * chunk, nb = (batch - b0 < chunk) ? (batch - b0) : chunk;
        // pipe_ev[3k]: upload of the chunk (of its second half when split), [3k + 2]: of its first half, [3k + 1]: compute
        cudaEvent_t* const ev = &c->pipe_ev[3 * k];
        bool labels_copied = false;
        if (nb >= 8) {
            // Upload in two halves: the front half of the pipeline (Lab + passes) of the first half runs while the
            // second half is still on the wire; the back half (connectivity enforcement, whose replay latency is per
            // launch, not per image) then runs once over the whole chunk.
            float coef;
            rc = check_params(c, &pp, &coef);
            if (rc) return rc;
            int launches = 0;
            c->kev_on = false;  // per-launch kernel timing belongs to fslic_b200_iterate(collect_timing >= 2) only
            c->kev_used = 0;
            if (may_sync && nchunks == 1 && nb >= 16 && nb <= c->cca.batch && nb <= 64)
                return iterate_host_lanes(c, h_images, h_clusters, h_labels, nb, &pp, coef);
            const int h0 = nb / 2, s0[2] = {b0, b0 + h0}, sn[2] = {h0, nb - h0};
            cudaEvent_t const up[2] = {ev[2], ev[0]};
            for (int h = 0; h < 2; h++) {
                rc = upload_slice(c, h_images, h_clusters, s0[h], sn[h], up[h]);
                if (rc) return rc;
                CK(cudaStreamWaitEvent(c->own_stream, up[h], 0));
                // slice s0 - b0 of the context buffers <-> images s0 .. s0+sn of this chunk
                rc = iterate_front(c, s0[h] - b0, c->d_img + s0[h] * N * 3, c->d_cl + s0[h] * K, sn[h], &pp, coef,
                                   c->own_stream, &launches, false);
                if (rc) return rc;
            }
            HostOut ho = {h_labels + b0 * N, c->out_stream, false};
            rc = iterate_back(c, c->d_lab + b0 * N, nb, &pp, c->own_stream, &launches, may_sync ? &ho : nullptr);
            if (rc) return rc;
            labels_copied = ho.done;
            c->last_launches = launches;
        } else {
            rc = upload_slice(c, h_images, h_clusters, b0, nb, ev[0]);
            if (rc) return rc;
            CK(cudaStreamWaitEvent(c->own_stream, ev[0], 0));
            if (nb < 4 && nchunks == 1 && pp.collect_timing == 0)  // nb < 4: one stream, no host sync inside
                rc = iterate_graphed(c, c->d_img, c->d_cl, c->d_lab, nb, &pp, c->own_stream);
            else
                rc = iterate_plain(c, c->d_img + b0 * N * 3, c->d_cl + b0 * K, c->d_lab + b0 * N, nb, &pp, c->own_stream);
            if (rc) return rc;
        }
        rc = download_slice(c, h_labels, h_clusters, b0, nb, labels_copied, c->own_stream, ev[1]);
        if (rc) return rc;
    }
    c->pending = true;
    if (!may_sync) return FSLIC_OK;
    CK(cudaStreamSynchronize(c->out_stream));
    CK(cudaStreamSynchronize(c->own_stream));
    c->pending = false;
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
        if (c->own_stream2) cudaStreamSynchronize(c->own_stream2);
        cca_sync_lanes(c->cca);
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
