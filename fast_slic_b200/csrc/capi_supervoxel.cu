// fast_slic_b200/csrc/capi_supervoxel.cu -- the extern "C" entry points of supervoxels: SLIC over float32 volumes
// (supervoxel.cuh) and 3-D connectivity enforcement (sv_cca.cuh).  Stateless (device pointers, caller-provided
// scratch), asynchronous on the caller's stream, never synchronise.
#include <limits.h>
#include <math.h>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "pool_stage.h"
#include "supervoxel.cuh"
#include "sv_cca.cuh"

#define SV_MAX_C 1024
#define SV_MAX_SIDE 32767
#define SV_MAX_NODES (1LL << 30)
#define SV_MAX_STRIDE 255
// k_sv_grid keeps one counter per bucket in shared memory.  Bucket pitches start at the window radii, which gives
// about one bucket per cluster (up to 65534); above this cap the pitch of the axis with the most buckets grows until
// the grid fits, so a bucket holds a few centres more and the tile and fallback kernels scan a little longer.
#define SV_MAX_CELLS 8192

static bool sv_volume_ok(int batch, int D, int H, int W) {
    return batch >= 0 && D >= 1 && H >= 1 && W >= 1 && D <= SV_MAX_SIDE && H <= SV_MAX_SIDE && W <= SV_MAX_SIDE &&
           (long long)D * H * W <= MAX_IMAGE_PIXELS;
}

// One call takes at most 65535 volumes (pool's keys hold the volume in 16 bits) and a batch whose voxels and one more
// fit an int (the scan that numbers the components)
static bool sv_call_ok(int batch, int D, int H, int W) {
    return batch <= 65535 && (long long)batch * D * H * W < INT_MAX;
}

// ---- connectivity enforcement ----------------------------------------------------------------------------------------

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

// ---- SLIC ----------------------------------------------------------------------------------------------------------

static bool sv_args_ok(int batch, int D, int H, int W, int C, int nd, int nh, int nw, int stride, int max_iter) {
    return sv_volume_ok(batch, D, H, W) && C >= 1 && C <= SV_MAX_C && nd >= 1 && nh >= 1 && nw >= 1 && nd <= D &&
           nh <= H && nw <= W && (long long)nd * nh * nw <= MAX_K &&
           (long long)batch * nd * nh * nw <= SV_MAX_NODES && stride >= 1 && stride <= SV_MAX_STRIDE && max_iter >= 0;
}

// The window radii R_a = ceil(L_a / n_a), the bucket pitches G_a >= R_a (the axis with the most buckets, z first on a
// tie, grows until at most SV_MAX_CELLS buckets remain) and the tiles of the full pass
struct SvGeom {
    int R[3], G[3], cells[3], ncell, tiles_x, tiles_z, full_tiles;
};

static SvGeom sv_geom(int D, int H, int W, int nd, int nh, int nw) {
    SvGeom g;
    const int L[3] = {D, H, W}, nn[3] = {nd, nh, nw};
    for (int a = 0; a < 3; a++) {
        g.R[a] = ceil_div(L[a], nn[a]);
        g.G[a] = g.R[a];
        g.cells[a] = ceil_div(L[a], g.G[a]);
    }
    while ((long long)g.cells[0] * g.cells[1] * g.cells[2] > SV_MAX_CELLS) {
        int a = 0;
        for (int e = 1; e < 3; e++)
            if (g.cells[e] > g.cells[a]) a = e;
        g.G[a]++;
        g.cells[a] = ceil_div(L[a], g.G[a]);
    }
    g.ncell = g.cells[0] * g.cells[1] * g.cells[2];
    g.tiles_x = ceil_div(W, SV_TILE_W);
    g.tiles_z = ceil_div(D, SV_TILE_D);
    g.full_tiles = g.tiles_x * ceil_div(H, SV_TILE_R) * g.tiles_z;
    return g;
}

// pool's sort for the keys of the largest pass (the rows 0, s, 2s, .. of every slice), the pooled means [B,C,K], the
// buckets (records and starts), per pass the count of tiles that overflowed, and the list of those tiles
struct SvScratch {
    PoolScratch pool;
    float* means;
    uint32_t* rec;
    int *cell_start, *ovf_count, *ovf_list;
    size_t total;
};

static SvScratch sv_layout(int batch, int D, int H, int W, int C, int K, int stride, int max_iter, const SvGeom& g,
                           void* base) {
    SvScratch s;
    Carve c(base);
    const long long nkeys = (long long)batch * D * ceil_div(H, stride) * W, nk = (long long)batch * K;
    s.pool = pool_layout(nkeys, nk, c.take<void>(pool_layout(nkeys, nk, nullptr).total));
    s.means = c.take<float>((size_t)nk * C * 4);
    s.rec = c.take<uint32_t>((size_t)nk * 4);
    s.cell_start = c.take<int>((size_t)batch * (g.ncell + 1) * 4);
    s.ovf_count = c.take<int>(((size_t)max_iter + 1) * 4);
    s.ovf_list = c.take<int>((size_t)batch * g.full_tiles * 4);
    s.total = c.total;
    return s;
}

// The SLIC passes and the enforcement run one after the other on one stream, so they share the scratch
extern "C" size_t fslic_b200_sv_slic_scratch_bytes(int batch, int D, int H, int W, int C, int nd, int nh, int nw,
                                                   int stride, int max_iter) {
    if (!sv_args_ok(batch, D, H, W, C, nd, nh, nw, stride, max_iter)) return (size_t)-1;
    if (batch == 0) return 256;
    if (!sv_call_ok(batch, D, H, W)) return (size_t)-1;
    const size_t slic = sv_layout(batch, D, H, W, C, nd * nh * nw, stride, max_iter, sv_geom(D, H, W, nd, nh, nw),
                                  nullptr).total;
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
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    const int K = nd * nh * nw;
    const SvGeom g = sv_geom(D, H, W, nd, nh, nw);
    const SvScratch s = sv_layout(batch, D, H, W, C, K, stride, max_iter, g, d_scratch);
    const long n = (long)D * H * W, nk = (long)batch * K;
    uint16_t* labels = reinterpret_cast<uint16_t*>(d_labels);
    SvParams p = {D, H, W, C, K, nd, nh, nw, g.R[0], g.R[1], g.R[2], g.G[0], g.G[1], g.G[2], g.cells[1], g.cells[2],
                  g.ncell, w2z, w2y, w2x, 0, 1, H, g.tiles_x, 0, 0};

    CK(cudaMemsetAsync(s.ovf_count, 0, ((size_t)max_iter + 1) * 4, st));
    CK(cudaMemsetAsync(labels, 0xff, (size_t)batch * n * 2, st));
    k_sv_seed<<<(int)grid_for(nk * C, device), 256, 0, st>>>(p, d_volumes, nk * C, d_position, d_centroids, d_count);
    const size_t grid_smem = ((size_t)g.ncell + 1) * 4;
    k_sv_grid<<<batch, 1024, grid_smem, st>>>(p, d_position, s.cell_start, s.rec);
    // pass t < max_iter visits the rows r = t % stride, r + stride, .. of every slice; pass max_iter is the full assign
    for (int t = 0; t <= max_iter; t++) {
        p.r = t < max_iter ? t % stride : 0;
        p.s = t < max_iter ? stride : 1;
        p.npr = p.r < H ? (H - 1 - p.r) / p.s + 1 : 0;
        p.tiles_y = ceil_div(p.npr, SV_TILE_R);
        p.tiles = g.tiles_x * p.tiles_y * g.tiles_z;
        if (p.npr > 0) {
            const dim3 grid((unsigned)p.tiles, (unsigned)batch);
            k_sv_assign_tiles<<<grid, SV_THREADS, 0, st>>>(p, d_volumes, d_centroids, d_position, s.cell_start, s.rec,
                                                           labels, s.ovf_count + t, s.ovf_list);
            const long fb = (long)batch * p.tiles < 4L * sms ? (long)batch * p.tiles : 4L * sms;
            k_sv_assign_fallback<<<(int)fb, SV_THREADS, 0, st>>>(p, d_volumes, d_centroids, d_position, s.cell_start,
                                                                 s.rec, labels, s.ovf_count + t, s.ovf_list);
        }
        if (t == max_iter) break;
        const long nkeys = (long)batch * D * p.npr * W;
        if (nkeys > 0)
            k_sv_keys<<<(int)grid_for(nkeys, device), 256, 0, st>>>(p, labels, nkeys, s.pool.key, s.pool.val);
        const int rc = pool_sorted_segments(s.pool, nkeys, batch, K, C, n, d_volumes, 1, s.means, d_count, device, st);
        if (rc) return rc;
        k_sv_update<<<(unsigned)((nk + 7) / 8), 256, 0, st>>>(p, nk, s.pool.seg_start, s.pool.seg_end, s.pool.sval,
                                                             s.means, d_position, d_centroids);
        k_sv_grid<<<batch, 1024, grid_smem, st>>>(p, d_position, s.cell_start, s.rec);
    }
    if (d_overflow)
        CK(cudaMemcpyAsync(d_overflow, s.ovf_count, ((size_t)max_iter + 1) * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return svc_run(device, batch, D, H, W, K, min_size, labels, d_labels, d_scratch, st);
}
