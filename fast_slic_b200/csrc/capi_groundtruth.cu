// fast_slic_b200/csrc/capi_groundtruth.cu -- the extern "C" entry points of ground-truth scores (groundtruth.cuh): class
// histograms, segmentation scores and boundary maps over a batch of label maps.  Stateless (device pointers,
// caller-provided scratch), asynchronous on the caller's stream, never synchronise: a CUDA graph can capture them.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>

#include "capi_common.h"
#include "groundtruth.cuh"

#define GT_MAX_BATCH (1 << 17)  // image bits of a key: 17 + 16 label bits + 31 gt bits

// K = 1 for the boundary map, which takes any label
static bool gt_shape_ok(int batch, int H, int W, int K) {
    return labels_shape_ok(batch, H, W, K) && (long long)H * W <= MAX_IMAGE_PIXELS;
}

static bool gt_dtype_ok(int dtype) {
    return dtype == FSLIC_GT_UINT8 || dtype == FSLIC_GT_INT16 || dtype == FSLIC_GT_INT32 || dtype == FSLIC_GT_INT64;
}

// Bits of the gt field of a key: every valid value of the dtype
static int gt_bits(int dtype) { return dtype == FSLIC_GT_UINT8 ? 8 : dtype == FSLIC_GT_INT16 ? 15 : 31; }

extern "C" int fslic_b200_gt_histogram_batch(int device, int batch, int H, int W, int K, int num_classes, int dtype,
                                             const void* d_classes, const uint16_t* d_labels, int32_t* d_out,
                                             void* stream) {
    if (!gt_shape_ok(batch, H, W, K) || num_classes < 1 || num_classes > 65536 || !gt_dtype_ok(dtype))
        return set_err(FSLIC_EINVAL, "bad batch, H, W, K, num_classes or dtype");
    const long hw = (long)H * W, n = (long)batch * hw;
    if (n == 0) return FSLIC_OK;
    if (!d_classes || !d_labels || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemsetAsync(d_out, 0, (size_t)batch * K * num_classes * 4, st));
    const int grid = (int)grid_for(n, device);
    switch (dtype) {
        case FSLIC_GT_UINT8:
            k_gt_histogram<<<grid, 256, 0, st>>>(d_labels, (const uint8_t*)d_classes, hw, n, K, num_classes, d_out);
            break;
        case FSLIC_GT_INT16:
            k_gt_histogram<<<grid, 256, 0, st>>>(d_labels, (const int16_t*)d_classes, hw, n, K, num_classes, d_out);
            break;
        case FSLIC_GT_INT32:
            k_gt_histogram<<<grid, 256, 0, st>>>(d_labels, (const int32_t*)d_classes, hw, n, K, num_classes, d_out);
            break;
        default:
            k_gt_histogram<<<grid, 256, 0, st>>>(d_labels, (const int64_t*)d_classes, hw, n, K, num_classes, d_out);
    }
    CK(cudaGetLastError());
    return FSLIC_OK;
}

static size_t gt_sort_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DoubleBuffer<unsigned long long> keys(nullptr, nullptr);
    cub::DeviceRadixSort::SortKeys(nullptr, bytes, keys, (int)items, 0, 64);
    return bytes;
}

static size_t gt_rle_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceRunLengthEncode::Encode(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                       (int*)nullptr, (int*)nullptr, (int)items);
    return bytes;
}

// The scratch of one scores call: the keys and their sort buffer (the run-length encoding writes the unique keys into
// whichever of the two the sort left free), the run counts (8 + 8 + 4 bytes per pixel), the run total, n_k, max_g n_kg
// and the UE sums per (image, label) (4 + 4 + 8 bytes), `nbits` boundary bitmaps (1/8 byte per pixel each: three for
// maps, five for volumes, whose windows are dilated in two steps) and the temporary storage of the sort or the
// encoding, whichever is larger.  Volumes take it with H = D * H.
struct GtScratch {
    unsigned long long* key[2];
    int *cnt, *nruns;
    uint32_t *nk, *mx;
    unsigned long long* ue;
    uint32_t* bits[5];
    void* temp;
    size_t temp_bytes, total;
};

static GtScratch gt_layout(int batch, int H, int W, int K, int nbits, void* base) {
    const size_t n = (size_t)batch * H * W, nk = (size_t)batch * K, words = (size_t)batch * H * ((W + 31) / 32);
    const size_t sort = gt_sort_temp_bytes((long long)n), rle = gt_rle_temp_bytes((long long)n);
    GtScratch s;
    Carve c(base);
    for (auto& k : s.key) k = c.take<unsigned long long>(n * 8);
    s.cnt = c.take<int>(n * 4);
    s.nruns = c.take<int>(4);
    s.nk = c.take<uint32_t>(nk * 4);
    s.mx = c.take<uint32_t>(nk * 4);
    s.ue = c.take<unsigned long long>(nk * 8);
    for (int i = 0; i < 5; i++) s.bits[i] = i < nbits ? c.take<uint32_t>(words * 4) : nullptr;
    s.temp_bytes = align_up(sort > rle ? sort : rle, 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_gt_scores_scratch_bytes(int batch, int H, int W, int K) {
    if (!gt_shape_ok(batch, H, W, K)) return (size_t)-1;
    const long long n = (long long)batch * H * W;
    if (n == 0) return 256;
    if (n > INT_MAX || batch > GT_MAX_BATCH) return (size_t)-1;  // one sort of 64-bit keys: split the batch
    return gt_layout(batch, H, W, K, 3, nullptr).total;
}

// The two per-pixel passes over the gt of one dtype: the overlap keys into s.key[0] and the three boundary bitmaps
template <typename T>
static void gt_pixel_passes(int batch, int H, int W, int K, int gbits, const void* d_gt, const uint16_t* lab,
                            int has_ignore, long long ignore, unsigned long long none, const GtScratch& s, int device,
                            cudaStream_t st) {
    const T* gt = static_cast<const T*>(d_gt);
    const long hw = (long)H * W, n = (long)batch * hw;
    const int Wd = (W + 31) / 32;
    k_gt_keys<<<(int)grid_for(n, device), 256, 0, st>>>(lab, gt, hw, n, K, gbits, has_ignore, ignore, none, s.key[0]);
    k_gt_bitmaps<<<image_grid(batch, (long)H * Wd * 32, device), 256, 0, st>>>(lab, gt, batch, H, W, Wd, has_ignore, ignore,
                                                                             s.bits[0], s.bits[1], s.bits[2]);
}

// The overlap table of a scores call whose keys are in s.key[0]: the keys sorted, one run per (image, label, gt), then
// n_k, max_g n_kg and the UE sums per (image, label) and their sums per image into d_out
static int gt_overlap(int batch, long n, int K, int gbits, int bits, unsigned long long none, const GtScratch& s,
                      long long* d_out, int device, cudaStream_t st) {
    const long nk = (long)batch * K;
    cub::DoubleBuffer<unsigned long long> keys(s.key[0], s.key[1]);
    size_t temp_used = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, temp_used, keys, (int)n, 0, bits, st);
    if (temp_used > s.temp_bytes) return set_err(FSLIC_ECUDA, "radix sort temporary storage");
    if (cub::DeviceRadixSort::SortKeys(s.temp, temp_used, keys, (int)n, 0, bits, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the overlap keys failed");
    const unsigned long long* sorted = keys.Current();
    unsigned long long* unique = keys.Alternate();
    temp_used = 0;
    cub::DeviceRunLengthEncode::Encode(nullptr, temp_used, sorted, unique, s.cnt, s.nruns, (int)n, st);
    if (temp_used > s.temp_bytes) return set_err(FSLIC_ECUDA, "run-length encoding temporary storage");
    if (cub::DeviceRunLengthEncode::Encode(s.temp, temp_used, sorted, unique, s.cnt, s.nruns, (int)n, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "run-length encoding of the overlap keys failed");
    CK(cudaMemsetAsync(s.nk, 0, (size_t)nk * 4, st));
    CK(cudaMemsetAsync(s.mx, 0, (size_t)nk * 4, st));
    CK(cudaMemsetAsync(s.ue, 0, (size_t)nk * 8, st));
    const int grid = (int)grid_for(n, device);
    k_gt_run_totals<<<grid, 256, 0, st>>>(unique, s.cnt, s.nruns, none, gbits, K, s.nk, s.mx);
    k_gt_run_ue<<<grid, 256, 0, st>>>(unique, s.cnt, s.nruns, none, gbits, K, s.nk, s.ue);
    k_gt_reduce<<<batch, 256, 0, st>>>(s.nk, s.mx, s.ue, K, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_gt_scores_batch(int device, int batch, int H, int W, int K, int tolerance, int dtype,
                                          const void* d_gt, const uint16_t* d_labels, int has_ignore, long long ignore,
                                          long long* d_out, void* d_scratch, size_t scratch_bytes, void* stream) {
    if (!gt_shape_ok(batch, H, W, K) || tolerance < 0 || tolerance > 32 || !gt_dtype_ok(dtype))
        return set_err(FSLIC_EINVAL, "bad batch, H, W, K, tolerance or dtype");
    const long hw = (long)H * W, n = (long)batch * hw;
    if (batch == 0) return FSLIC_OK;
    if (!d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemsetAsync(d_out, 0, (size_t)batch * GT_FIELDS * 8, st));
    if (n == 0) return FSLIC_OK;
    if (!d_gt || !d_labels || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_gt_scores_scratch_bytes(batch, H, W, K);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    const GtScratch s = gt_layout(batch, H, W, K, 3, d_scratch);
    const int gbits = gt_bits(dtype), bits = bit_length((unsigned long long)(batch - 1)) + 16 + gbits;
    const unsigned long long none = bits >= 64 ? ~0ull : (1ull << bits) - 1;
    switch (dtype) {
        case FSLIC_GT_UINT8:
            gt_pixel_passes<uint8_t>(batch, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
            break;
        case FSLIC_GT_INT16:
            gt_pixel_passes<int16_t>(batch, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
            break;
        case FSLIC_GT_INT32:
            gt_pixel_passes<int32_t>(batch, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
            break;
        default:
            gt_pixel_passes<int64_t>(batch, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
    }
    const int Wd = (W + 31) / 32;
    k_gt_boundary_counts<<<image_grid(batch, (long)H * Wd, device), 256, 0, st>>>(s.bits[0], s.bits[1], s.bits[2], batch, H,
                                                                                Wd, tolerance, d_out);
    return gt_overlap(batch, n, K, gbits, bits, none, s, d_out, device, st);
}

extern "C" int fslic_b200_gt_boundaries_batch(int device, int batch, int H, int W, const uint16_t* d_labels, uint8_t* d_out,
                                              void* stream) {
    if (!gt_shape_ok(batch, H, W, 1)) return set_err(FSLIC_EINVAL, "bad batch, H or W");
    const long hw = (long)H * W, n = (long)batch * hw;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    k_gt_boundaries<<<(int)grid_for(n, device), 256, 0, (cudaStream_t)stream>>>(d_labels, hw, H, W, n, d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// ---- Volumes (DESIGN.md section 4.24)

// A volume of at most MAX_IMAGE_PIXELS voxels (no overflow: H W <= 2^29 before D multiplies it)
static bool gt3d_shape_ok(int batch, int D, int H, int W, int K) {
    if (!labels_shape_ok(batch, H, W, K) || D < 0) return false;
    const long long hw = (long long)H * W;
    return D == 0 || hw == 0 || (hw <= MAX_IMAGE_PIXELS && (long long)D * hw <= MAX_IMAGE_PIXELS);
}

static bool gt_tolerance_ok(int r) { return r >= 0 && r <= 32; }

extern "C" size_t fslic_b200_gt_scores3d_scratch_bytes(int batch, int D, int H, int W, int K) {
    if (!gt3d_shape_ok(batch, D, H, W, K)) return (size_t)-1;
    const long long n = (long long)batch * D * H * W;
    if (n == 0) return 256;
    if (n > INT_MAX || batch > GT_MAX_BATCH) return (size_t)-1;  // one sort of 64-bit keys: split the batch
    return gt_layout(batch, D * H, W, K, 5, nullptr).total;
}

// The per-voxel passes over the gt of one dtype: the overlap keys into s.key[0] (k_gt_keys over D * H * W voxels per
// volume) and the three boundary bitmaps
template <typename T>
static void gt_voxel_passes(int batch, int D, int H, int W, int K, int gbits, const void* d_gt, const uint16_t* lab,
                            int has_ignore, long long ignore, unsigned long long none, const GtScratch& s, int device,
                            cudaStream_t st) {
    const T* gt = static_cast<const T*>(d_gt);
    const long dhw = (long)D * H * W, n = (long)batch * dhw;
    const int Wd = (W + 31) / 32;
    k_gt_keys<<<(int)grid_for(n, device), 256, 0, st>>>(lab, gt, dhw, n, K, gbits, has_ignore, ignore, none, s.key[0]);
    k_gt_bitmaps3d<<<image_grid(batch, (long)D * H * Wd * 32, device), 256, 0, st>>>(
        lab, gt, batch, D, H, W, Wd, has_ignore, ignore, s.bits[0], s.bits[1], s.bits[2]);
}

extern "C" int fslic_b200_gt_scores3d_batch(int device, int batch, int D, int H, int W, int K, int rz, int ry, int rx,
                                            int dtype, const void* d_gt, const uint16_t* d_labels, int has_ignore,
                                            long long ignore, long long* d_out, void* d_scratch, size_t scratch_bytes,
                                            void* stream) {
    if (!gt3d_shape_ok(batch, D, H, W, K) || !gt_tolerance_ok(rz) || !gt_tolerance_ok(ry) || !gt_tolerance_ok(rx) ||
        !gt_dtype_ok(dtype))
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, K, tolerance or dtype");
    const long dhw = (long)D * H * W, n = (long)batch * dhw;
    if (batch == 0) return FSLIC_OK;
    if (!d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemsetAsync(d_out, 0, (size_t)batch * GT_FIELDS * 8, st));
    if (n == 0) return FSLIC_OK;
    if (!d_gt || !d_labels || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_gt_scores3d_scratch_bytes(batch, D, H, W, K);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "batch too large for one call: split it");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    const GtScratch s = gt_layout(batch, D * H, W, K, 5, d_scratch);
    const int gbits = gt_bits(dtype), bits = bit_length((unsigned long long)(batch - 1)) + 16 + gbits;
    const unsigned long long none = bits >= 64 ? ~0ull : (1ull << bits) - 1;
    switch (dtype) {
        case FSLIC_GT_UINT8:
            gt_voxel_passes<uint8_t>(batch, D, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
            break;
        case FSLIC_GT_INT16:
            gt_voxel_passes<int16_t>(batch, D, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
            break;
        case FSLIC_GT_INT32:
            gt_voxel_passes<int32_t>(batch, D, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
            break;
        default:
            gt_voxel_passes<int64_t>(batch, D, H, W, K, gbits, d_gt, d_labels, has_ignore, ignore, none, s, device, st);
    }
    const int Wd = (W + 31) / 32;
    const dim3 grid = image_grid(batch, (long)D * H * Wd, device);
    k_gt_dilate_yx<<<grid, 256, 0, st>>>(s.bits[0], s.bits[1], batch, D, H, Wd, ry, rx, s.bits[3], s.bits[4]);
    k_gt_boundary_counts3d<<<grid, 256, 0, st>>>(s.bits[0], s.bits[1], s.bits[2], s.bits[3], s.bits[4], batch, D, H, Wd,
                                                 rz, d_out);
    return gt_overlap(batch, n, K, gbits, bits, none, s, d_out, device, st);
}

extern "C" int fslic_b200_gt_boundaries3d_batch(int device, int batch, int D, int H, int W, const uint16_t* d_labels,
                                                uint8_t* d_out, void* stream) {
    if (!gt3d_shape_ok(batch, D, H, W, 1)) return set_err(FSLIC_EINVAL, "bad batch, D, H or W");
    const long dhw = (long)D * H * W, n = (long)batch * dhw;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_out) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    k_gt_boundaries3d<<<(int)grid_for(n, device), 256, 0, (cudaStream_t)stream>>>(d_labels, (uint32_t)dhw, D, H, W, n,
                                                                                  d_out);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
