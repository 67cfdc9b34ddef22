// fast_slic_b200/csrc/capi_float_slic.cu -- the extern "C" entry points of SLIC over float32 data (float_slic.cuh):
// feature maps [B,C,H,W], and volumes [B,C,D,H,W] with their 3-D connectivity enforcement (sv_cca.cuh).  Stateless
// (device pointers, caller-provided scratch), asynchronous on the caller's stream, never synchronise.  Feature maps
// leave connectivity enforcement to the caller (fslic_b200_enforce_connectivity).
#include <limits.h>
#include <math.h>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "float_slic.cuh"
#include "pool_stage.h"
#include "sv_cca.cuh"

#define FLOAT_SLIC_MAX_C 1024
#define FLOAT_SLIC_MAX_SIDE 32767
#define FLOAT_SLIC_MAX_NODES (1LL << 30)
#define FLOAT_SLIC_MAX_STRIDE 255
// k_float_slic_grid keeps one counter per cell in shared memory.  Cell pitches start at the window radii; above this
// cap they grow (fs_geom, sv_geom) until the grid fits, so a cell holds a few centres more and the tile and fallback
// kernels scan a little longer.
#define FLOAT_SLIC_MAX_CELLS 8192

// ---- the passes, shared by feature maps and volumes -----------------------------------------------------------------

// The tiles per image of a pass with npr rows along axis NA - 2, and along each axis
template <class G>
static int pass_tiles(FloatSlicParams& p, int npr) {
    p.tiles = 1;
    for (int a = 0; a < G::NA; a++) {
        p.ntiles[a] = ceil_div(a == G::NA - 2 ? npr : p.L[a], tile_extent<G>(a));
        p.tiles *= p.ntiles[a];
    }
    return p.tiles;
}

// pool's sort for the keys of the largest pass (the rows 0, s, 2s, .. of every slice), the pooled means [B,C,K], the
// cell grid (records and starts), per pass the count of tiles that overflowed, and the list of those tiles
struct FloatSlicScratch {
    PoolScratch pool;
    float* means;
    uint32_t* rec;
    int *cell_start, *ovf_count, *ovf_list;
    size_t total;
};

template <class G>
static FloatSlicScratch float_slic_layout(int batch, FloatSlicParams p, int stride, int max_iter, void* base) {
    FloatSlicScratch s;
    Carve c(base);
    const int rows = p.L[G::NA - 2];
    const long long nkeys = (long long)batch * (image_size<G::NA>(p) / rows) * ceil_div(rows, stride);
    const long long nk = (long long)batch * p.K;
    s.pool = pool_layout(nkeys, nk, c.take<void>(pool_layout(nkeys, nk, nullptr).total));
    s.means = c.take<float>((size_t)nk * p.C * 4);
    s.rec = c.take<uint32_t>((size_t)nk * 4);
    s.cell_start = c.take<int>((size_t)batch * (p.ncell + 1) * 4);
    s.ovf_count = c.take<int>(((size_t)max_iter + 1) * 4);
    s.ovf_list = c.take<int>((size_t)batch * pass_tiles<G>(p, rows) * 4);
    s.total = c.total;
    return s;
}

// The passes of `batch` images from the seeds in pos / feat: pass t < max_iter assigns the rows r = t % stride,
// r + stride, .. (of every slice) and updates, pass max_iter assigns every row.  labels u16 [batch, image]; the
// per-pass count of overflowed tiles goes to d_overflow when given.
template <class G>
static int float_slic_passes(int device, int batch, FloatSlicParams p, int stride, int max_iter, const float* d_x,
                             uint16_t* labels, float* pos, float* feat, int32_t* count, int32_t* d_overflow,
                             void* d_scratch, cudaStream_t st) {
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    const FloatSlicScratch s = float_slic_layout<G>(batch, p, stride, max_iter, d_scratch);
    const int rows = p.L[G::NA - 2];
    const long n = image_size<G::NA>(p), nk = (long)batch * p.K;
    const size_t grid_smem = ((size_t)p.ncell + 1) * 4;

    CK(cudaMemsetAsync(s.ovf_count, 0, ((size_t)max_iter + 1) * 4, st));
    CK(cudaMemsetAsync(labels, 0xff, (size_t)batch * n * 2, st));
    k_float_slic_grid<G><<<batch, 1024, grid_smem, st>>>(p, pos, s.cell_start, s.rec);
    for (int t = 0; t <= max_iter; t++) {
        p.r = t < max_iter ? t % stride : 0;
        p.s = t < max_iter ? stride : 1;
        p.npr = p.r < rows ? (rows - 1 - p.r) / p.s + 1 : 0;
        pass_tiles<G>(p, p.npr);
        if (p.npr > 0) {
            const dim3 grid((unsigned)p.tiles, (unsigned)batch);
            k_float_slic_assign_tiles<G><<<grid, tile_threads<G>, 0, st>>>(p, d_x, feat, pos, s.cell_start, s.rec,
                                                                           labels, s.ovf_count + t, s.ovf_list);
            const long fb = (long)batch * p.tiles < 4L * sms ? (long)batch * p.tiles : 4L * sms;
            k_float_slic_assign_fallback<G><<<(int)fb, tile_threads<G>, 0, st>>>(p, d_x, feat, pos, s.cell_start,
                                                                                 s.rec, labels, s.ovf_count + t,
                                                                                 s.ovf_list);
        }
        if (t == max_iter) break;
        const long nkeys = (long)batch * (n / rows) * p.npr;
        if (nkeys > 0)
            k_float_slic_keys<G><<<(int)grid_for(nkeys, device), 256, 0, st>>>(p, labels, nkeys, s.pool.key,
                                                                                s.pool.val);
        const int rc = pool_sorted_segments(s.pool, nkeys, batch, p.K, p.C, n, d_x, 1, s.means, count, device, st);
        if (rc) return rc;
        k_float_slic_update<G><<<(unsigned)((nk + 7) / 8), 256, 0, st>>>(p, nk, s.pool.seg_start, s.pool.seg_end,
                                                                         s.pool.sval, s.means, pos, feat);
        k_float_slic_grid<G><<<batch, 1024, grid_smem, st>>>(p, pos, s.cell_start, s.rec);
    }
    if (d_overflow)
        CK(cudaMemcpyAsync(d_overflow, s.ovf_count, ((size_t)max_iter + 1) * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// ---- feature maps ---------------------------------------------------------------------------------------------------

static bool fs_args_ok(int batch, int H, int W, int C, int K, int stride, int max_iter) {
    return batch >= 0 && H >= 1 && W >= 1 && H <= FLOAT_SLIC_MAX_SIDE && W <= FLOAT_SLIC_MAX_SIDE &&
           (long long)H * W <= MAX_IMAGE_PIXELS && C >= 1 && C <= FLOAT_SLIC_MAX_C && K >= 1 && K <= MAX_K &&
           K <= (long long)H * W && (long long)batch * K <= FLOAT_SLIC_MAX_NODES && stride >= 1 &&
           stride <= FLOAT_SLIC_MAX_STRIDE && max_iter >= 0;
}

// The window S on both axes as the u16 context computes it (capi.cu, context.h:60), and the cell pitch G >= S on both
// axes with at most FLOAT_SLIC_MAX_CELLS cells
static FloatSlicParams fs_geom(int H, int W, int C, int K) {
    FloatSlicParams p = {};
    const int S = (int)(int16_t)sqrt((double)(H * W / K));
    int G = S;
    while ((long long)ceil_div(H, G) * ceil_div(W, G) > FLOAT_SLIC_MAX_CELLS) G++;
    const int L[2] = {H, W};
    for (int a = 0; a < 2; a++) {
        p.L[a] = L[a];
        p.R[a] = S;
        p.G[a] = G;
        p.cells[a] = ceil_div(L[a], G);
    }
    p.ncell = p.cells[0] * p.cells[1];
    p.C = C;
    p.K = K;
    return p;
}

extern "C" size_t fslic_b200_feature_slic_scratch_bytes(int batch, int H, int W, int C, int K, int stride,
                                                        int max_iter) {
    if (!fs_args_ok(batch, H, W, C, K, stride, max_iter)) return (size_t)-1;
    if (batch == 0) return 256;
    if ((long long)batch * H * W > INT_MAX || batch > 65535) return (size_t)-1;  // one radix sort: split the batch
    return float_slic_layout<MapSlic>(batch, fs_geom(H, W, C, K), stride, max_iter, nullptr).total;
}

extern "C" int fslic_b200_feature_slic(int device, int batch, int H, int W, int C, int K, float compactness, int stride,
                                       int max_iter, const float* d_features, const float* d_init_position,
                                       const float* d_init_features, uint16_t* d_labels, float* d_position,
                                       float* d_centroids, int32_t* d_count, int32_t* d_overflow, void* d_scratch,
                                       size_t scratch_bytes, void* stream) {
    if (!fs_args_ok(batch, H, W, C, K, stride, max_iter) || !(compactness > 0.f) || !isfinite(compactness))
        return set_err(FSLIC_EINVAL, "bad batch, H, W, C, K, compactness, stride or max_iter");
    if (batch == 0) return FSLIC_OK;
    if (!d_features || !d_labels || !d_position || !d_centroids || !d_count || !d_scratch)
        return set_err(FSLIC_EINVAL, "NULL argument");
    if (!d_init_position != !d_init_features) return set_err(FSLIC_EINVAL, "init needs both positions and features");
    const size_t need = fslic_b200_feature_slic_scratch_bytes(batch, H, W, C, K, stride, max_iter);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    FloatSlicParams p = fs_geom(H, W, C, K);
    const float w = compactness / (float)p.R[0];
    p.w2[0] = w * w;
    const long nk = (long)batch * K;
    k_fs_seed<<<(int)grid_for(nk * C, device), 256, 0, st>>>(d_features, d_init_position, d_init_features, nk * C, H,
                                                             W, C, K, d_position, d_centroids, d_count);
    return float_slic_passes<MapSlic>(device, batch, p, stride, max_iter, d_features, d_labels, d_position,
                                      d_centroids, d_count, d_overflow, d_scratch, st);
}

// ---- volumes: connectivity enforcement ------------------------------------------------------------------------------

static bool sv_volume_ok(int batch, int D, int H, int W) {
    return batch >= 0 && D >= 1 && H >= 1 && W >= 1 && D <= FLOAT_SLIC_MAX_SIDE && H <= FLOAT_SLIC_MAX_SIDE &&
           W <= FLOAT_SLIC_MAX_SIDE && (long long)D * H * W <= MAX_IMAGE_PIXELS;
}

// One call takes at most 65535 volumes (pool's keys hold the volume in 16 bits) and a batch whose voxels and one more
// fit an int (the scan that numbers the components)
static bool sv_call_ok(int batch, int D, int H, int W) {
    return batch <= 65535 && (long long)batch * D * H * W < INT_MAX;
}

// Per voxel of the batch: parents, component numbers (one more for the scan's total), and, indexed by component,
// areas, predecessors and final labels -- sized for every voxel its own component
struct SvcScratch {
    int *par, *cid, *area, *pred, *fin;
    void* temp;
    size_t temp_bytes, total;
};

static SvcScratch svc_layout(long long voxels, void* base) {
    SvcScratch s;
    Carve c(base);
    s.par = c.take<int>((size_t)voxels * 4);
    s.cid = c.take<int>(((size_t)voxels + 1) * 4);
    s.area = c.take<int>((size_t)voxels * 4);
    s.pred = c.take<int>((size_t)voxels * 4);
    s.fin = c.take<int>((size_t)voxels * 4);
    s.temp_bytes = align_up(exclusive_sum_temp_bytes<int>(voxels + 1), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

// Enforcement of `batch` label volumes d_in u16 [batch, D, H, W] into d_out (d_out may be d_in)
static int svc_run(int device, int batch, int D, int H, int W, int K, int min_size, const uint16_t* d_in,
                   int16_t* d_out, void* d_scratch, cudaStream_t st) {
    const long n = (long)D * H * W, total = (long)batch * n;
    const SvcScratch s = svc_layout(total, d_scratch);
    const int nseg = ceil_div(W, 32);
    const long rows = (long)batch * D * H;
    k_svc_runs<<<(int)grid_for(rows * nseg * 32, device), 256, 0, st>>>(d_in, rows, W, nseg, n, s.par);
    k_svc_union<<<(int)grid_for(total, device), 256, 0, st>>>(d_in, total, D, H, W, s.par);
    k_svc_flatten<<<(int)grid_for(total, device), 256, 0, st>>>(total, n, s.par, s.cid);
    CK(cudaMemsetAsync(s.cid + total, 0, 4, st));
    size_t temp_bytes = s.temp_bytes;
    CK(cub::DeviceScan::ExclusiveSum(s.temp, temp_bytes, s.cid, s.cid, (int)(total + 1), st));
    CK(cudaMemsetAsync(s.area, 0, (size_t)total * 4, st));
    k_svc_comp<<<(int)grid_for(total, device), 256, 0, st>>>(total, D, H, W, s.par, s.cid, s.area, s.pred);
    k_svc_select<<<batch, SVC_SELECT_THREADS, 0, st>>>(n, K, min_size, s.cid, s.area, s.fin);
    k_svc_absorb<<<image_grid(batch, n, device), 256, 0, st>>>(n, s.cid, s.pred, s.fin);
    k_svc_output<<<(int)grid_for(total, device), 256, 0, st>>>(total, n, s.par, s.cid, s.fin, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" size_t fslic_b200_sv_enforce_scratch_bytes(int batch, int D, int H, int W) {
    if (!sv_volume_ok(batch, D, H, W)) return (size_t)-1;
    if (batch == 0) return 256;
    if (!sv_call_ok(batch, D, H, W)) return (size_t)-1;
    return svc_layout((long long)batch * D * H * W, nullptr).total;
}

extern "C" int fslic_b200_sv_enforce(int device, int batch, int D, int H, int W, int K, int min_size,
                                     const uint16_t* d_labels, int16_t* d_out, void* d_scratch, size_t scratch_bytes,
                                     void* stream) {
    if (!sv_volume_ok(batch, D, H, W) || K < 1 || K > MAX_K || min_size < 0)
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, K or min_size");
    if (batch == 0) return FSLIC_OK;
    if (!d_labels || !d_out || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_sv_enforce_scratch_bytes(batch, D, H, W);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    return svc_run(device, batch, D, H, W, K, min_size, d_labels, d_out, d_scratch, (cudaStream_t)stream);
}

// ---- volumes: SLIC --------------------------------------------------------------------------------------------------

static bool sv_args_ok(int batch, int D, int H, int W, int C, int nd, int nh, int nw, int stride, int max_iter) {
    return sv_volume_ok(batch, D, H, W) && C >= 1 && C <= FLOAT_SLIC_MAX_C && nd >= 1 && nh >= 1 && nw >= 1 &&
           nd <= D && nh <= H && nw <= W && (long long)nd * nh * nw <= MAX_K &&
           (long long)batch * nd * nh * nw <= FLOAT_SLIC_MAX_NODES && stride >= 1 && stride <= FLOAT_SLIC_MAX_STRIDE &&
           max_iter >= 0;
}

// The window radii R_a = ceil(L_a / n_a) and the cell pitches G_a >= R_a: the axis with the most cells, z first on a
// tie, grows until at most FLOAT_SLIC_MAX_CELLS cells remain
static FloatSlicParams sv_geom(int D, int H, int W, int C, int nd, int nh, int nw) {
    FloatSlicParams p = {};
    const int L[3] = {D, H, W}, nn[3] = {nd, nh, nw};
    for (int a = 0; a < 3; a++) {
        p.L[a] = L[a];
        p.R[a] = ceil_div(L[a], nn[a]);
        p.G[a] = p.R[a];
        p.cells[a] = ceil_div(L[a], p.G[a]);
    }
    while ((long long)p.cells[0] * p.cells[1] * p.cells[2] > FLOAT_SLIC_MAX_CELLS) {
        int a = 0;
        for (int e = 1; e < 3; e++)
            if (p.cells[e] > p.cells[a]) a = e;
        p.G[a]++;
        p.cells[a] = ceil_div(L[a], p.G[a]);
    }
    p.ncell = p.cells[0] * p.cells[1] * p.cells[2];
    p.C = C;
    p.K = nd * nh * nw;
    return p;
}

// The SLIC passes and the enforcement run one after the other on one stream, so they share the scratch
extern "C" size_t fslic_b200_sv_slic_scratch_bytes(int batch, int D, int H, int W, int C, int nd, int nh, int nw,
                                                   int stride, int max_iter) {
    if (!sv_args_ok(batch, D, H, W, C, nd, nh, nw, stride, max_iter)) return (size_t)-1;
    if (batch == 0) return 256;
    if (!sv_call_ok(batch, D, H, W)) return (size_t)-1;
    const size_t slic =
        float_slic_layout<VolumeSlic>(batch, sv_geom(D, H, W, C, nd, nh, nw), stride, max_iter, nullptr).total;
    const size_t cca = svc_layout((long long)batch * D * H * W, nullptr).total;
    return slic > cca ? slic : cca;
}

extern "C" int fslic_b200_sv_slic(int device, int batch, int D, int H, int W, int C, int nd, int nh, int nw, float w2z,
                                  float w2y, float w2x, int stride, int max_iter, int min_size, const float* d_volumes,
                                  int16_t* d_labels, float* d_position, float* d_centroids, int32_t* d_count,
                                  int32_t* d_overflow, void* d_scratch, size_t scratch_bytes, void* stream) {
    if (!sv_args_ok(batch, D, H, W, C, nd, nh, nw, stride, max_iter) || min_size < 0 || !(w2z >= 0.f) ||
        !(w2y >= 0.f) || !(w2x >= 0.f) || !isfinite(w2z) || !isfinite(w2y) || !isfinite(w2x))
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, C, grid, weights, stride, max_iter or min_size");
    if (batch == 0) return FSLIC_OK;
    if (!d_volumes || !d_labels || !d_position || !d_centroids || !d_count || !d_scratch)
        return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_sv_slic_scratch_bytes(batch, D, H, W, C, nd, nh, nw, stride, max_iter);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    FloatSlicParams p = sv_geom(D, H, W, C, nd, nh, nw);
    p.w2[0] = w2z;
    p.w2[1] = w2y;
    p.w2[2] = w2x;
    const long nkc = (long)batch * p.K * C;
    uint16_t* labels = reinterpret_cast<uint16_t*>(d_labels);
    k_sv_seed<<<(int)grid_for(nkc, device), 256, 0, st>>>(d_volumes, nkc, D, H, W, C, nd, nh, nw, d_position,
                                                          d_centroids, d_count);
    const int rc = float_slic_passes<VolumeSlic>(device, batch, p, stride, max_iter, d_volumes, labels, d_position,
                                                 d_centroids, d_count, d_overflow, d_scratch, st);
    if (rc) return rc;
    return svc_run(device, batch, D, H, W, p.K, min_size, labels, d_labels, d_scratch, st);
}
