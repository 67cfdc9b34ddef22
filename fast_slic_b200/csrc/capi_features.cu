// fast_slic_b200/csrc/capi_features.cu -- the extern "C" entry points of SLIC over float feature maps
// (feature_slic.cuh).  Stateless (device pointers, caller-provided scratch), asynchronous on the caller's stream,
// never synchronise.  Connectivity enforcement is the caller's next step (fslic_b200_enforce_connectivity).
#include <limits.h>
#include <math.h>

#include "capi_common.h"
#include "feature_slic.cuh"
#include "pool_stage.h"

#define FS_MAX_C 1024
#define FS_MAX_SIDE 32767
#define FS_MAX_NODES (1LL << 30)
#define FS_MAX_STRIDE 255
#define FS_MAX_CELLS 8192  // k_fs_grid keeps one counter per cell in shared memory

static bool fs_args_ok(int batch, int H, int W, int C, int K, int stride, int max_iter) {
    return batch >= 0 && H >= 1 && W >= 1 && H <= FS_MAX_SIDE && W <= FS_MAX_SIDE &&
           (long long)H * W <= MAX_IMAGE_PIXELS && C >= 1 && C <= FS_MAX_C && K >= 1 && K <= MAX_K &&
           K <= (long long)H * W && (long long)batch * K <= FS_MAX_NODES && stride >= 1 && stride <= FS_MAX_STRIDE &&
           max_iter >= 0;
}

// S as the u16 context computes it (capi.cu, context.h:60), the cell pitch G >= S with at most FS_MAX_CELLS cells, and
// the tiles of the full pass
struct FsGeom {
    int S, G, cellW, ncell, tiles_x, full_tiles;
};

static FsGeom fs_geom(int H, int W, int K) {
    FsGeom g;
    g.S = (int)(int16_t)sqrt((double)(H * W / K));
    g.G = g.S;
    while ((long long)ceil_div(H, g.G) * ceil_div(W, g.G) > FS_MAX_CELLS) g.G++;
    g.cellW = ceil_div(W, g.G);
    g.ncell = g.cellW * ceil_div(H, g.G);
    g.tiles_x = ceil_div(W, FS_TILE_W);
    g.full_tiles = g.tiles_x * ceil_div(H, FS_TILE_R);
    return g;
}

// pool's sort for the keys of the largest pass (the rows 0, s, 2s, ..), the pooled means [B,C,K], the cell grid
// (records and starts), per pass the count of tiles that overflowed, and the list of those tiles
struct FsScratch {
    PoolScratch pool;
    float* means;
    uint32_t* rec;
    int *cell_start, *ovf_count, *ovf_list;
    size_t total;
};

static FsScratch fs_layout(int batch, int H, int W, int C, int K, int stride, int max_iter, const FsGeom& g,
                           void* base) {
    FsScratch s;
    Carve c(base);
    const long long nkeys = (long long)batch * ceil_div(H, stride) * W, nk = (long long)batch * K;
    s.pool = pool_layout(nkeys, nk, c.take<void>(pool_layout(nkeys, nk, nullptr).total));
    s.means = c.take<float>((size_t)nk * C * 4);
    s.rec = c.take<uint32_t>((size_t)nk * 4);
    s.cell_start = c.take<int>((size_t)batch * (g.ncell + 1) * 4);
    s.ovf_count = c.take<int>(((size_t)max_iter + 1) * 4);
    s.ovf_list = c.take<int>((size_t)batch * g.full_tiles * 4);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_feature_slic_scratch_bytes(int batch, int H, int W, int C, int K, int stride,
                                                        int max_iter) {
    if (!fs_args_ok(batch, H, W, C, K, stride, max_iter)) return (size_t)-1;
    if (batch == 0) return 256;
    if ((long long)batch * H * W > INT_MAX || batch > 65535) return (size_t)-1;  // one radix sort: split the batch
    return fs_layout(batch, H, W, C, K, stride, max_iter, fs_geom(H, W, K), nullptr).total;
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
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    const FsGeom g = fs_geom(H, W, K);
    const FsScratch s = fs_layout(batch, H, W, C, K, stride, max_iter, g, d_scratch);
    const long hw = (long)H * W, nk = (long)batch * K;
    const float w = compactness / (float)g.S;
    FsParams p = {H, W, C, K, g.S, g.G, g.cellW, g.ncell, w * w, 0, 1, H, g.tiles_x, 0};

    CK(cudaMemsetAsync(s.ovf_count, 0, ((size_t)max_iter + 1) * 4, st));
    CK(cudaMemsetAsync(d_labels, 0xff, (size_t)batch * hw * 2, st));
    k_fs_seed<<<(int)grid_for(nk * C, device), 256, 0, st>>>(d_features, d_init_position, d_init_features, nk * C, H,
                                                             W, C, K, d_position, d_centroids, d_count);
    const size_t grid_smem = ((size_t)g.ncell + 1) * 4;
    k_fs_grid<<<batch, 1024, grid_smem, st>>>(p, d_position, s.cell_start, s.rec);
    // pass t < max_iter visits the rows r = t % stride, r + stride, ..; pass max_iter is the full assign
    for (int t = 0; t <= max_iter; t++) {
        p.r = t < max_iter ? t % stride : 0;
        p.s = t < max_iter ? stride : 1;
        p.npr = p.r < H ? (H - 1 - p.r) / p.s + 1 : 0;
        p.tiles = g.tiles_x * ceil_div(p.npr, FS_TILE_R);
        if (p.npr > 0) {
            const dim3 grid((unsigned)p.tiles, (unsigned)batch);
            k_fs_assign_tiles<<<grid, FS_TILE_W * FS_TILE_R, 0, st>>>(p, d_features, d_centroids, d_position,
                                                                      s.cell_start, s.rec, d_labels, s.ovf_count + t,
                                                                      s.ovf_list);
            const long fb = (long)batch * p.tiles < 4L * sms ? (long)batch * p.tiles : 4L * sms;
            k_fs_assign_fallback<<<(int)fb, FS_TILE_W * FS_TILE_R, 0, st>>>(
                p, d_features, d_centroids, d_position, s.cell_start, s.rec, d_labels, s.ovf_count + t, s.ovf_list);
        }
        if (t == max_iter) break;
        const long n = (long)batch * p.npr * W;
        if (n > 0) k_fs_keys<<<(int)grid_for(n, device), 256, 0, st>>>(p, d_labels, n, s.pool.key, s.pool.val);
        const int rc = pool_sorted_segments(s.pool, n, batch, K, C, hw, d_features, 1, s.means, d_count, device, st);
        if (rc) return rc;
        k_fs_update<<<(unsigned)((nk + 7) / 8), 256, 0, st>>>(p, nk, s.pool.seg_start, s.pool.seg_end, s.pool.sval,
                                                             s.means, d_position, d_centroids);
        k_fs_grid<<<batch, 1024, grid_smem, st>>>(p, d_position, s.cell_start, s.rec);
    }
    if (d_overflow)
        CK(cudaMemcpyAsync(d_overflow, s.ovf_count, ((size_t)max_iter + 1) * 4, cudaMemcpyDeviceToDevice, st));
    CK(cudaGetLastError());
    return FSLIC_OK;
}
