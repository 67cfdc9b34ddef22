// fast_slic_b200/csrc/capi_crf.cu -- the extern "C" entry points of the temporal CRF (crf.cuh, crf_feed.cuh): frames fed
// from the host (fslic_b200_crf_*) and from device memory (fslic_b200_crfdev_*), groups of CRFs stepped together
// (fslic_b200_crfgroup_*), and the glibc expf / logf clones the CRF kernels use, exposed for testing.
#include <algorithm>
#include <cstring>
#include <deque>
#include <new>
#include <string>
#include <unordered_set>
#include <vector>

#include "capi_common.h"
#include "common.cuh"
#include "crf.cuh"
#include "crf_feed.cuh"

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
struct PushScratch {
    void* graph;
    int32_t* counts;
    uint32_t* nbrs;
    size_t graph_bytes, total;
};

static PushScratch crfdev_push_layout(int K, int batch, void* base) {
    PushScratch s;
    Carve c(base);
    s.graph_bytes = align_up(fslic_b200_connectivity_batch_scratch_bytes(K, batch), 256);
    s.graph = c.take<void>(s.graph_bytes);
    s.counts = c.take<int32_t>((size_t)batch * K * 4);
    s.nbrs = c.take<uint32_t>((size_t)batch * K * CONN_MAX * 4);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_crfdev_push_scratch_bytes(int K, int batch) {
    const size_t graph = fslic_b200_connectivity_batch_scratch_bytes(K, batch);
    if (graph == (size_t)-1) return graph;
    if (K <= 0 || batch <= 0) return 256;
    return crfdev_push_layout(K, batch, nullptr).total;
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
        const PushScratch g = crfdev_push_layout(K, batch, d_scratch);
        rc = fslic_b200_get_connectivity_batch(c0->device, batch, H, W, K, d_labels, g.counts, g.nbrs, nullptr, g.graph,
                                               g.graph_bytes, st);
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
            k_feed_csr<<<dim3(1, (unsigned)n), FEED_CSR_THREADS, 0, st>>>(g.counts + (size_t)b0 * K,
                                                                          g.nbrs + (size_t)b0 * K * CONN_MAX, K, dst);
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
