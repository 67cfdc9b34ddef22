// fast_slic_b200/csrc/capi_boundary.cu -- the extern "C" entry points of boundary statistics (boundary.cuh).
// Stateless (device pointers, caller-provided scratch), asynchronous on the caller's stream, never synchronise: the
// caller reads the boundary pair count back between the select and the stats.
#include <limits.h>

#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

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
