// fast_slic_b200/csrc/capi_boundary.cu -- the extern "C" entry points of boundary statistics (boundary.cuh).
// Stateless (device pointers, caller-provided scratch), asynchronous on the caller's stream, never synchronise: the
// caller reads the boundary pair count back between the select and the stats.
#include <limits.h>

#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "boundary.cuh"
#include "capi_common.h"
#include "cub_temp.cuh"

static bool boundary_args_ok(int batch, int H, int W, int K, int connectivity) {
    return labels_shape_ok(batch, H, W, K) && (connectivity == 4 || connectivity == 8);
}

// Pixel-pair slots of a call: D per pixel, -1 when they do not fit one select (int items, uint32 slots)
static long long boundary_slots(int batch, int H, int W, int connectivity) {
    if ((long long)H * W > MAX_IMAGE_PIXELS) return -1;
    const long long slots = (long long)batch * H * W * (connectivity == 8 ? 4 : 2);
    return slots > INT_MAX ? -1 : slots;
}

static size_t boundary_select_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceSelect::If(nullptr, bytes, thrust::counting_iterator<uint32_t>(0), (uint32_t*)nullptr, (int*)nullptr,
                          (int)items, BoundaryPair{});
    return bytes;
}

static size_t boundary_starts_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceSelect::Flagged(nullptr, bytes, thrust::counting_iterator<uint32_t>(0), (const uint8_t*)nullptr,
                               (uint32_t*)nullptr, (int*)nullptr, (int)items);
    return bytes;
}

// The select's scratch, which the stats read: the selected slots (4 bytes per slot) and the select's temporary storage
struct SelectScratch {
    uint32_t* sel;
    void* temp;
    size_t temp_bytes, total;
};

static SelectScratch select_layout(long long slots, const void* base) {
    SelectScratch s;
    Carve c(const_cast<void*>(base));
    s.sel = c.take<uint32_t>((size_t)slots * 4);
    s.temp_bytes = align_up(boundary_select_temp_bytes(slots), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_boundary_select_scratch_bytes(int batch, int H, int W, int K, int connectivity) {
    if (!boundary_args_ok(batch, H, W, K, connectivity)) return (size_t)-1;
    const long long slots = boundary_slots(batch, H, W, connectivity);
    if (slots < 0) return (size_t)-1;
    if (slots == 0) return 256;
    return select_layout(slots, nullptr).total;
}

extern "C" int fslic_b200_boundary_select_batch(int device, int batch, int H, int W, int K, int connectivity,
                                                const uint16_t* d_labels, int32_t* d_pairs, void* d_scratch,
                                                size_t scratch_bytes, void* stream) {
    if (!boundary_args_ok(batch, H, W, K, connectivity)) return set_err(FSLIC_EINVAL, "bad batch, H, W, K or connectivity");
    const size_t need = fslic_b200_boundary_select_scratch_bytes(batch, H, W, K, connectivity);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "image or batch too large for one call");
    const long long slots = boundary_slots(batch, H, W, connectivity);
    if (!d_pairs) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    if (slots == 0) {
        CK(cudaMemsetAsync(d_pairs, 0, 4, st));
        return FSLIC_OK;
    }
    if (!d_labels || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    const SelectScratch s = select_layout(slots, d_scratch);
    size_t temp_bytes = s.temp_bytes;
    const BoundaryPair op{d_labels, (uint32_t)((long long)H * W), (uint32_t)W, (uint32_t)H, (uint32_t)K,
                          connectivity == 8 ? 2 : 1};
    if (cub::DeviceSelect::If(s.temp, temp_bytes, thrust::counting_iterator<uint32_t>(0), s.sel, d_pairs, (int)slots, op,
                              st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "selection of the boundary pairs failed");
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// The stats' scratch for `pairs` boundary pairs and `edges` graph entries: pair keys, sorted keys, sorted slots and run
// starts (24 bytes per pair) and the run-head flags (1 byte per pair), entry keys and indices and their sorted copies (24 bytes per entry), the run count and
// the largest temporary storage of the two sorts and the run select
struct BoundaryScratch {
    unsigned long long *key, *skey, *ekey, *sekey;
    uint32_t *sslot, *start, *eidx, *seidx;
    uint8_t* head;
    int* runs;
    void* temp;
    size_t temp_bytes, total;
};

static BoundaryScratch boundary_layout(long long pairs, long long edges, void* base) {
    BoundaryScratch s;
    Carve c(base);
    s.key = c.take<unsigned long long>((size_t)pairs * 8);
    s.skey = c.take<unsigned long long>((size_t)pairs * 8);
    s.sslot = c.take<uint32_t>((size_t)pairs * 4);
    s.start = c.take<uint32_t>((size_t)pairs * 4);
    s.head = c.take<uint8_t>((size_t)pairs);
    s.ekey = c.take<unsigned long long>((size_t)edges * 8);
    s.sekey = c.take<unsigned long long>((size_t)edges * 8);
    s.eidx = c.take<uint32_t>((size_t)edges * 4);
    s.seidx = c.take<uint32_t>((size_t)edges * 4);
    s.runs = c.take<int>(4);
    size_t temp = radix_pairs_temp_bytes<unsigned long long, uint32_t>(pairs, 64),
           t2 = radix_pairs_temp_bytes<unsigned long long, uint32_t>(edges, 64), t3 = boundary_starts_temp_bytes(pairs);
    if (t2 > temp) temp = t2;
    if (t3 > temp) temp = t3;
    s.temp_bytes = align_up(temp, 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_boundary_stats_scratch_bytes(long long pairs, long long edges) {
    if (pairs < 0 || edges < 0 || pairs > INT_MAX || edges > INT_MAX) return (size_t)-1;
    return boundary_layout(pairs, edges, nullptr).total;
}

extern "C" int fslic_b200_boundary_stats_batch(int device, int batch, int H, int W, int K, int C, int connectivity,
                                               const uint16_t* d_labels, const float* d_values, long long pairs,
                                               const void* d_select_scratch, size_t select_bytes,
                                               long long image_base, long long nodes, long long edges,
                                               const long long* d_src, const long long* d_dst, int first,
                                               float* d_mean, float* d_min, float* d_max, int32_t* d_count,
                                               void* d_scratch, size_t scratch_bytes, void* stream) {
    if (!boundary_args_ok(batch, H, W, K, connectivity) || C < 1 || image_base < 0 || nodes < 0)
        return set_err(FSLIC_EINVAL, "bad batch, H, W, K, C, connectivity, image base or nodes");
    const size_t select_need = fslic_b200_boundary_select_scratch_bytes(batch, H, W, K, connectivity);
    const size_t need = fslic_b200_boundary_stats_scratch_bytes(pairs, edges);
    if (select_need == (size_t)-1 || need == (size_t)-1) return set_err(FSLIC_EINVAL, "image, batch, pairs or edges too large");
    const long long slots = boundary_slots(batch, H, W, connectivity);
    if (pairs > slots) return set_err(FSLIC_EINVAL, "more boundary pairs than pixel pairs");
    if ((long long)C * edges > LLONG_MAX / 4) return set_err(FSLIC_EINVAL, "edges * C too large");
    if (edges == 0) return FSLIC_OK;
    if (!d_src || !d_dst || !d_mean || !d_min || !d_max || !d_count || !d_scratch ||
        (pairs && (!d_labels || !d_values || !d_select_scratch)))
        return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < need || (pairs && select_bytes < select_need)) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    if (first)
        k_boundary_init<<<(int)grid_for((long)(edges * C), device), 256, 0, st>>>(edges, C, d_mean, d_min, d_max, d_count);
    if (pairs == 0) {
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    const BoundaryScratch s = boundary_layout(pairs, edges, d_scratch);
    const uint32_t* sel = select_layout(slots, d_select_scratch).sel;
    const uint32_t hw = (uint32_t)((long long)H * W);
    const int shift = connectivity == 8 ? 2 : 1;
    const int bits = 32 + bit_length((unsigned long long)(batch - 1));  // image << 32 | lo << 16 | hi
    k_boundary_keys<<<(int)grid_for((long)pairs, device), 256, 0, st>>>(sel, (long)pairs, d_labels, hw, W, shift, s.key);
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.key, s.skey, sel, s.sslot, (int)pairs, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the boundary pairs failed");
    temp_bytes = s.temp_bytes;
    k_boundary_heads<<<(int)grid_for((long)pairs, device), 256, 0, st>>>(s.skey, (long)pairs, s.head);
    if (cub::DeviceSelect::Flagged(s.temp, temp_bytes, thrust::counting_iterator<uint32_t>(0), s.head, s.start, s.runs,
                                   (int)pairs, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "selection of the run starts failed");
    k_boundary_entry_keys<<<(int)grid_for((long)edges, device), 256, 0, st>>>(d_src, d_dst, edges, nodes, K, image_base,
                                                                              batch, s.ekey, s.eidx);
    temp_bytes = s.temp_bytes;
    if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.ekey, s.sekey, s.eidx, s.seidx, (int)edges, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the graph entries failed");
    // persistent warps: 8 per CTA, at most 16 CTAs per SM
    k_boundary_runs<<<(int)grid_for((long)pairs, device), 256, 0, st>>>(s.skey, s.sslot, s.start, s.runs, (int)pairs,
                                                                        s.sekey, s.seidx, (int)edges, d_values, C, hw, W,
                                                                        shift, d_mean, d_min, d_max, d_count);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// ---- Volumes (DESIGN.md section 4.24)

static bool boundary3d_args_ok(int batch, int D, int H, int W, int K, int connectivity) {
    return labels_shape_ok(batch, H, W, K) && D >= 0 && (connectivity == 6 || connectivity == 18 || connectivity == 26);
}

// RAG3D_OFFSETS: the forward half of the 3x3x3 neighbourhood, (dz, dy, dx), in k_boundary3d_mask's order
static const int boundary3d_host_dirs[13][3] = {{0, 0, 1}, {0, 1, 0},  {1, 0, 0},  {0, 1, 1},  {0, 1, -1},
                                                {1, 1, 0}, {1, -1, 0}, {1, 0, 1},  {1, 0, -1}, {1, 1, 1},
                                                {1, 1, -1}, {1, -1, 1}, {1, -1, -1}};

static int boundary3d_ndir(int connectivity) { return connectivity == 6 ? 3 : (connectivity == 18 ? 9 : 13); }

// Voxels of a call, -1 when a volume exceeds 2^29 voxels or has more than 2^31 - 1 voxel pairs (a boundary count must
// fit int32), or the call has more than 2^31 - 1 voxels (one select); the per-volume limits are region_adjacency_3d's
static long long boundary3d_voxels(int batch, int D, int H, int W, int connectivity) {
    const long long hw = (long long)H * W;
    if (D == 0 || hw == 0) return 0;
    if (hw > MAX_IMAGE_PIXELS || (long long)D * hw > MAX_IMAGE_PIXELS) return -1;
    const long long L[3][2] = {{D, D - 1}, {H, H - 1}, {W, W - 1}};
    long long pairs = 0;
    for (int d = 0; d < boundary3d_ndir(connectivity); d++) {
        const int o[3] = {boundary3d_host_dirs[d][0], boundary3d_host_dirs[d][1], boundary3d_host_dirs[d][2]};
        pairs += L[0][o[0] != 0] * L[1][o[1] != 0] * L[2][o[2] != 0];
    }
    if (pairs > INT_MAX) return -1;
    const long long n = (long long)batch * D * hw;
    return n > INT_MAX ? -1 : n;
}

static Boundary3dDirs boundary3d_dirs(int H, int W) {
    Boundary3dDirs d;
    for (int k = 0; k < 13; k++)
        d.off[k] = boundary3d_host_dirs[k][0] * H * W + boundary3d_host_dirs[k][1] * W + boundary3d_host_dirs[k][2];
    return d;
}

static size_t boundary3d_select_temp_bytes(long long voxels) {
    size_t a = 0, b = 0;
    cub::DeviceSelect::Flagged(nullptr, a, thrust::counting_iterator<uint32_t>(0), (const uint16_t*)nullptr,
                               (uint32_t*)nullptr, (int*)nullptr, (int)voxels);
    cub::DeviceReduce::Sum(nullptr, b,
                           thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), Boundary3dPopc64{}),
                           (unsigned long long*)nullptr, (int)voxels);
    return a > b ? a : b;
}

// The select's scratch, which the stats read: the direction masks (2 bytes per voxel), the selected voxels (4 bytes
// per voxel), their count and the larger temporary storage of the select and the pair sum
struct Select3dScratch {
    uint16_t* mask;
    uint32_t* sel;
    int* nsel;
    void* temp;
    size_t temp_bytes, total;
};

static Select3dScratch select3d_layout(long long voxels, const void* base) {
    Select3dScratch s;
    Carve c(const_cast<void*>(base));
    s.mask = c.take<uint16_t>((size_t)voxels * 2);
    s.sel = c.take<uint32_t>((size_t)voxels * 4);
    s.nsel = c.take<int>(4);
    s.temp_bytes = align_up(boundary3d_select_temp_bytes(voxels), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_boundary3d_select_scratch_bytes(int batch, int D, int H, int W, int K, int connectivity) {
    if (!boundary3d_args_ok(batch, D, H, W, K, connectivity)) return (size_t)-1;
    const long long n = boundary3d_voxels(batch, D, H, W, connectivity);
    if (n < 0) return (size_t)-1;
    if (n == 0) return 256;
    return select3d_layout(n, nullptr).total;
}

extern "C" int fslic_b200_boundary3d_select_batch(int device, int batch, int D, int H, int W, int K, int connectivity,
                                                  const uint16_t* d_labels, long long* d_counts, void* d_scratch,
                                                  size_t scratch_bytes, void* stream) {
    if (!boundary3d_args_ok(batch, D, H, W, K, connectivity))
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, K or connectivity");
    const size_t need = fslic_b200_boundary3d_select_scratch_bytes(batch, D, H, W, K, connectivity);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "volume or batch too large for one call");
    const long long n = boundary3d_voxels(batch, D, H, W, connectivity);
    if (!d_counts) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        CK(cudaMemsetAsync(d_counts, 0, 16, st));
        return FSLIC_OK;
    }
    if (!d_labels || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    const Select3dScratch s = select3d_layout(n, d_scratch);
    const uint32_t dhw = (uint32_t)((long long)D * H * W);
    const int grid = (int)grid_for((long)n, device);
    const Boundary3dDirs dirs = boundary3d_dirs(H, W);
    if (connectivity == 6)
        k_boundary3d_mask<3><<<grid, 256, 0, st>>>(d_labels, dhw, D, H, W, (uint32_t)n, K, dirs, s.mask);
    else if (connectivity == 18)
        k_boundary3d_mask<9><<<grid, 256, 0, st>>>(d_labels, dhw, D, H, W, (uint32_t)n, K, dirs, s.mask);
    else
        k_boundary3d_mask<13><<<grid, 256, 0, st>>>(d_labels, dhw, D, H, W, (uint32_t)n, K, dirs, s.mask);
    size_t temp_bytes = s.temp_bytes;
    // the mask is the flag: a voxel is selected when it has a boundary direction
    if (cub::DeviceSelect::Flagged(s.temp, temp_bytes, thrust::counting_iterator<uint32_t>(0), (const uint16_t*)s.mask,
                                   s.sel, s.nsel, (int)n, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "selection of the boundary voxels failed");
    k_boundary3d_count<<<1, 1, 0, st>>>(s.nsel, d_counts);
    temp_bytes = s.temp_bytes;
    if (cub::DeviceReduce::Sum(s.temp, temp_bytes,
                               thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0),
                                                               Boundary3dPopc64{s.mask}),
                               reinterpret_cast<unsigned long long*>(d_counts + 1), (int)n, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "sum of the boundary pairs failed");
    CK(cudaGetLastError());
    return FSLIC_OK;
}

static size_t boundary3d_scan_temp_bytes(long long voxels) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes,
                                  thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0),
                                                                  Boundary3dPopc{}),
                                  (uint32_t*)nullptr, (int)voxels);
    return bytes;
}

// The stats' scratch for `voxels` boundary voxels, `pairs` boundary pairs and `edges` graph entries: the first pair of
// each voxel (4 bytes per voxel); pair keys, sorted keys, positions, sorted positions, anchors and run starts (32 bytes
// per pair), directions and run-head flags (2 bytes per pair); entry keys and indices and their sorted copies (24 bytes
// per entry), the run count and the largest temporary storage of the scan, the two sorts and the run select
struct Boundary3dScratch {
    uint32_t* first;
    unsigned long long *key, *skey, *ekey, *sekey;
    uint32_t *pos, *spos, *anchor, *start, *eidx, *seidx;
    uint8_t *dir, *head;
    int* runs;
    void* temp;
    size_t temp_bytes, total;
};

static Boundary3dScratch boundary3d_layout(long long voxels, long long pairs, long long edges, void* base) {
    Boundary3dScratch s;
    Carve c(base);
    s.first = c.take<uint32_t>((size_t)voxels * 4);
    s.key = c.take<unsigned long long>((size_t)pairs * 8);
    s.skey = c.take<unsigned long long>((size_t)pairs * 8);
    s.pos = c.take<uint32_t>((size_t)pairs * 4);
    s.spos = c.take<uint32_t>((size_t)pairs * 4);
    s.anchor = c.take<uint32_t>((size_t)pairs * 4);
    s.start = c.take<uint32_t>((size_t)pairs * 4);
    s.dir = c.take<uint8_t>((size_t)pairs);
    s.head = c.take<uint8_t>((size_t)pairs);
    s.ekey = c.take<unsigned long long>((size_t)edges * 8);
    s.sekey = c.take<unsigned long long>((size_t)edges * 8);
    s.eidx = c.take<uint32_t>((size_t)edges * 4);
    s.seidx = c.take<uint32_t>((size_t)edges * 4);
    s.runs = c.take<int>(4);
    size_t temp = radix_pairs_temp_bytes<unsigned long long, uint32_t>(pairs, 64);
    const size_t t2 = radix_pairs_temp_bytes<unsigned long long, uint32_t>(edges, 64),
                 t3 = boundary_starts_temp_bytes(pairs), t4 = boundary3d_scan_temp_bytes(voxels);
    if (t2 > temp) temp = t2;
    if (t3 > temp) temp = t3;
    if (t4 > temp) temp = t4;
    s.temp_bytes = align_up(temp, 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_boundary3d_stats_scratch_bytes(long long voxels, long long pairs, long long edges) {
    if (voxels < 0 || pairs < 0 || edges < 0 || voxels > INT_MAX || pairs > INT_MAX || edges > INT_MAX ||
        voxels > pairs || pairs > 13 * voxels)
        return (size_t)-1;
    return boundary3d_layout(voxels, pairs, edges, nullptr).total;
}

extern "C" int fslic_b200_boundary3d_stats_batch(int device, int batch, int D, int H, int W, int K, int C,
                                                 int connectivity, const uint16_t* d_labels, const float* d_values,
                                                 long long voxels, long long pairs, const void* d_select_scratch,
                                                 size_t select_bytes, long long image_base, long long nodes,
                                                 long long edges, const long long* d_src, const long long* d_dst,
                                                 int first, float* d_mean, float* d_min, float* d_max,
                                                 int32_t* d_count, void* d_scratch, size_t scratch_bytes,
                                                 void* stream) {
    if (!boundary3d_args_ok(batch, D, H, W, K, connectivity) || C < 1 || image_base < 0 || nodes < 0)
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, K, C, connectivity, image base or nodes");
    const size_t select_need = fslic_b200_boundary3d_select_scratch_bytes(batch, D, H, W, K, connectivity);
    const size_t need = fslic_b200_boundary3d_stats_scratch_bytes(voxels, pairs, edges);
    if (select_need == (size_t)-1 || need == (size_t)-1)
        return set_err(FSLIC_EINVAL, "volume, batch, voxels, pairs or edges too large or inconsistent");
    const long long n = boundary3d_voxels(batch, D, H, W, connectivity);
    if (voxels > n || pairs > (long long)boundary3d_ndir(connectivity) * voxels)
        return set_err(FSLIC_EINVAL, "more boundary voxels or pairs than the volumes have");
    if ((long long)C * edges > LLONG_MAX / 4) return set_err(FSLIC_EINVAL, "edges * C too large");
    if (edges == 0) return FSLIC_OK;
    if (!d_src || !d_dst || !d_mean || !d_min || !d_max || !d_count || !d_scratch ||
        (pairs && (!d_labels || !d_values || !d_select_scratch)))
        return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < need || (pairs && select_bytes < select_need)) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    if (first)
        k_boundary_init<<<(int)grid_for((long)(edges * C), device), 256, 0, st>>>(edges, C, d_mean, d_min, d_max, d_count);
    if (pairs == 0) {
        CK(cudaGetLastError());
        return FSLIC_OK;
    }
    const Boundary3dScratch s = boundary3d_layout(voxels, pairs, edges, d_scratch);
    const Select3dScratch sel = select3d_layout(n, d_select_scratch);
    const uint32_t dhw = (uint32_t)((long long)D * H * W);
    const Boundary3dDirs dirs = boundary3d_dirs(H, W);
    const int bits = 32 + bit_length((unsigned long long)(batch - 1));  // image << 32 | lo << 16 | hi
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceScan::ExclusiveSum(s.temp, temp_bytes,
                                      thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0),
                                                                      Boundary3dPopc{sel.mask, sel.sel}),
                                      s.first, (int)voxels, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "scan of the boundary voxels failed");
    k_boundary3d_expand<<<(int)grid_for((long)voxels, device), 256, 0, st>>>(sel.sel, (uint32_t)voxels, sel.mask, s.first,
                                                                            d_labels, dhw, dirs, s.key, s.pos, s.anchor,
                                                                            s.dir);
    temp_bytes = s.temp_bytes;
    if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.key, s.skey, s.pos, s.spos, (int)pairs, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the boundary pairs failed");
    k_boundary_heads<<<(int)grid_for((long)pairs, device), 256, 0, st>>>(s.skey, (long)pairs, s.head);
    temp_bytes = s.temp_bytes;
    if (cub::DeviceSelect::Flagged(s.temp, temp_bytes, thrust::counting_iterator<uint32_t>(0), s.head, s.start, s.runs,
                                   (int)pairs, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "selection of the run starts failed");
    k_boundary_entry_keys<<<(int)grid_for((long)edges, device), 256, 0, st>>>(d_src, d_dst, edges, nodes, K, image_base,
                                                                              batch, s.ekey, s.eidx);
    temp_bytes = s.temp_bytes;
    if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.ekey, s.sekey, s.eidx, s.seidx, (int)edges, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the graph entries failed");
    k_boundary3d_runs<<<(int)grid_for((long)pairs, device), 256, 0, st>>>(
        s.skey, s.spos, s.anchor, s.dir, s.start, s.runs, (int)pairs, s.sekey, s.seidx, (int)edges, d_values, C, dhw, dirs,
        d_mean, d_min, d_max, d_count);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
