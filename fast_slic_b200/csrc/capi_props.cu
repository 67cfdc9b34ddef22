// fast_slic_b200/csrc/capi_props.cu -- the extern "C" entry points of superpixel shapes (props.cuh) over a batch of
// label maps and of supervoxel shapes (props3d.cuh) over a batch of label volumes.  Stateless (device pointers, no scratch), asynchronous on the caller's stream, never synchronises: a CUDA
// graph can capture it.
#include "capi_common.h"
#include "props.cuh"
#include "props3d.cuh"

#define PROPS_MAX_SIDE 65535  // with MAX_IMAGE_PIXELS every sum fits int64 and the perimeter int32
#define PROPS3D_MAX_SIDE 32767  // supervoxels' side limit; with MAX_IMAGE_PIXELS every sum fits int64 (N D^2 < 2^59)

extern "C" int fslic_b200_props_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                      int32_t* d_area, int32_t* d_bbox, long long* d_moments, int32_t* d_perimeter,
                                      int32_t* d_border, double* d_centroid, double* d_covariance, void* stream) {
    if (!labels_shape_ok(batch, H, W, K) || H > PROPS_MAX_SIDE || W > PROPS_MAX_SIDE ||
        (long long)H * W > MAX_IMAGE_PIXELS)
        return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    if (batch == 0) return FSLIC_OK;
    if (!d_area || !d_bbox || !d_moments || !d_perimeter || !d_border || !d_centroid || !d_covariance ||
        (!d_labels && (long long)H * W > 0))
        return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long nodes = (long)batch * K;
    PropsOut o{d_area, d_bbox, reinterpret_cast<unsigned long long*>(d_moments), d_perimeter, d_border};
    if ((long long)H * W == 0) {  // no pixel: every field 0
        CK(cudaMemsetAsync(d_area, 0, (size_t)nodes * 4, st));
        CK(cudaMemsetAsync(d_bbox, 0, (size_t)nodes * 16, st));
        CK(cudaMemsetAsync(d_moments, 0, (size_t)nodes * 8 * PROPS_MOMENTS, st));
        CK(cudaMemsetAsync(d_perimeter, 0, (size_t)nodes * 4, st));
        CK(cudaMemsetAsync(d_border, 0, (size_t)nodes * 4, st));
        CK(cudaMemsetAsync(d_centroid, 0, (size_t)nodes * 16, st));
        CK(cudaMemsetAsync(d_covariance, 0, (size_t)nodes * 24, st));
        return FSLIC_OK;
    }
    const int node_grid = (int)grid_for(nodes, device);
    k_props_init<<<node_grid, 256, 0, st>>>(nodes, o);
    const long Wd = (W + 31) / 32;
    const long tiles = (long)ceil_div(H, PROPS_TILE_ROWS) * ((Wd + PROPS_TILE_WORDS - 1) / PROPS_TILE_WORDS);
    // one CTA per tile
    k_props_tiles<<<image_grid(batch, tiles * 256, device), 256, 0, st>>>(d_labels, batch, H, W, K, o);
    k_props_finish<<<node_grid, 256, 0, st>>>(nodes, o, d_centroid, d_covariance);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_props3d_batch(int device, int batch, int D, int H, int W, int K, const uint16_t* d_labels,
                                        int32_t* d_area, int32_t* d_bbox, long long* d_moments, long long* d_surface,
                                        int32_t* d_border, double* d_centroid, double* d_covariance, void* stream) {
    if (!labels_shape_ok(batch, H, W, K) || D < 0 || D > PROPS3D_MAX_SIDE || H > PROPS3D_MAX_SIDE ||
        W > PROPS3D_MAX_SIDE || (long long)D * H * W > MAX_IMAGE_PIXELS)
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W or K");
    if (batch == 0) return FSLIC_OK;
    const long long dhw = (long long)D * H * W;
    if (!d_area || !d_bbox || !d_moments || !d_surface || !d_border || !d_centroid || !d_covariance ||
        (!d_labels && dhw > 0))
        return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long nodes = (long)batch * K;
    Props3dOut o{d_area, d_bbox, reinterpret_cast<unsigned long long*>(d_moments),
                 reinterpret_cast<unsigned long long*>(d_surface), d_border};
    if (dhw == 0) {  // no voxel: every field 0
        CK(cudaMemsetAsync(d_area, 0, (size_t)nodes * 4, st));
        CK(cudaMemsetAsync(d_bbox, 0, (size_t)nodes * 24, st));
        CK(cudaMemsetAsync(d_moments, 0, (size_t)nodes * 8 * PROPS3D_MOMENTS, st));
        CK(cudaMemsetAsync(d_surface, 0, (size_t)nodes * 8, st));
        CK(cudaMemsetAsync(d_border, 0, (size_t)nodes * 4, st));
        CK(cudaMemsetAsync(d_centroid, 0, (size_t)nodes * 24, st));
        CK(cudaMemsetAsync(d_covariance, 0, (size_t)nodes * 48, st));
        return FSLIC_OK;
    }
    const int node_grid = (int)grid_for(nodes, device);
    k_props3d_init<<<node_grid, 256, 0, st>>>(nodes, o);
    const long Wd = (W + 31) / 32;
    const long tiles =
        (long)D * ceil_div(H, PROPS3D_TILE_ROWS) * ((Wd + PROPS3D_TILE_WORDS - 1) / PROPS3D_TILE_WORDS);
    // one CTA per tile
    k_props3d_tiles<<<image_grid(batch, tiles * 256, device), 256, 0, st>>>(d_labels, batch, D, H, W, K, o);
    k_props3d_finish<<<node_grid, 256, 0, st>>>(nodes, o, d_centroid, d_covariance);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
