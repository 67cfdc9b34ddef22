// fast_slic_b200/csrc/capi_merge.cu -- the extern "C" entry points of superpixel merging (merge.cuh): single-linkage
// threshold and region-count cuts of a batch's region adjacency graph.  Stateless (device pointers, caller-provided
// scratch), asynchronous on the caller's stream, never synchronise and read nothing back: a CUDA graph can capture them.
#include <cub/device/device_segmented_radix_sort.cuh>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "merge.cuh"

#define MERGE_MAX_NODES (1LL << 30)

static size_t merge_sort_temp_bytes(int batch, int K) {
    const int nodes = batch * K;
    size_t sort = 0;
    cub::DeviceSegmentedRadixSort::SortKeys(nullptr, sort, (const unsigned long long*)nullptr,
                                            (unsigned long long*)nullptr, nodes, batch, (const int*)nullptr,
                                            (const int*)nullptr);
    const size_t scan = exclusive_sum_temp_bytes<int>(nodes + 1);
    return sort > scan ? sort : scan;
}

// Per node: the parent, the presence flag, the chosen key, the forest table and its sorted copy, the root flags and
// their scan (4 + 4 + 8 + 8 + 8 + 4 + 4 bytes); per image: the forest edge count, the present count and the two
// segment bounds; the Boruvka round flags; the larger temporary storage of the sort and the scan.
struct MergeScratch {
    int *parent, *present, *count, *P, *seg_begin, *seg_end, *linked, *flag, *pos;
    unsigned long long *best, *table, *sorted;
    void* temp;
    size_t temp_bytes, total;
};

static MergeScratch merge_layout(int batch, int K, void* base) {
    MergeScratch s;
    const size_t n = (size_t)batch * K;
    Carve c(base);
    s.parent = c.take<int>(n * 4);
    s.present = c.take<int>(n * 4);
    s.best = c.take<unsigned long long>(n * 8);
    s.table = c.take<unsigned long long>(n * 8);
    s.sorted = c.take<unsigned long long>(n * 8);
    s.flag = c.take<int>((n + 1) * 4);
    s.pos = c.take<int>((n + 1) * 4);
    s.count = c.take<int>((size_t)batch * 4);
    s.P = c.take<int>((size_t)batch * 4);
    s.seg_begin = c.take<int>((size_t)batch * 4);
    s.seg_end = c.take<int>((size_t)batch * 4);
    s.linked = c.take<int>(MERGE_ROUNDS * 4);
    s.temp_bytes = align_up(merge_sort_temp_bytes(batch, K), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_merge_scratch_bytes(int batch, int K) {
    if (batch < 0 || K < 1 || K > MAX_K || (long long)batch * K > MERGE_MAX_NODES) return (size_t)-1;
    if (batch == 0) return 256;
    return merge_layout(batch, K, nullptr).total;
}

extern "C" int fslic_b200_merge_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                      long long edges, const long long* d_src, const long long* d_dst,
                                      const float* d_weight, int mode, double threshold, int num_regions,
                                      int32_t* d_region, int32_t* d_num_regions, int16_t* d_out, void* d_scratch,
                                      size_t scratch_bytes, void* stream) {
    if (!labels_shape_ok(batch, H, W, K) || (long long)batch * K > MERGE_MAX_NODES || edges < 0)
        return set_err(FSLIC_EINVAL, "bad batch, H, W, K or edges");
    if (mode != FSLIC_MERGE_THRESHOLD && mode != FSLIC_MERGE_NUM_REGIONS) return set_err(FSLIC_EINVAL, "bad mode");
    if (mode == FSLIC_MERGE_THRESHOLD && threshold != threshold) return set_err(FSLIC_EINVAL, "threshold is NaN");
    if (mode == FSLIC_MERGE_NUM_REGIONS && num_regions < 1) return set_err(FSLIC_EINVAL, "num_regions < 1");
    if (batch == 0) return FSLIC_OK;
    const long hw = (long)H * W, n_pix = (long)batch * hw;
    if (!d_region || !d_num_regions || !d_scratch || (n_pix && (!d_labels || !d_out)) ||
        (edges && (!d_src || !d_dst || !d_weight)))
        return set_err(FSLIC_EINVAL, "NULL argument");
    const MergeScratch s = merge_layout(batch, K, d_scratch);
    if (scratch_bytes < s.total) return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long nodes = (long)batch * K;
    const int node_grid = (int)grid_for(nodes, device);
    CK(cudaMemsetAsync(s.present, 0, (size_t)nodes * 4, st));
    CK(cudaMemsetAsync(s.count, 0, (size_t)batch * 4, st));
    CK(cudaMemsetAsync(s.P, 0, (size_t)batch * 4, st));
    CK(cudaMemsetAsync(s.linked, 0, MERGE_ROUNDS * 4, st));
    if (n_pix) k_merge_presence<<<(int)grid_for(n_pix, device), 256, 0, st>>>(d_labels, hw, n_pix, K, s.present, s.P);
    k_merge_init<<<node_grid, 256, 0, st>>>(nodes, s.parent, s.best);
    if (edges) {
        const int edge_grid = (int)grid_for((long)edges, device);
        for (int r = 0; r < MERGE_ROUNDS; r++) {
            k_merge_choose<<<edge_grid, 256, 0, st>>>(r, s.linked, d_src, d_dst, d_weight, edges, nodes, K, s.present,
                                                      s.parent, s.best);
            k_merge_link<<<node_grid, 256, 0, st>>>(r, s.linked, nodes, K, s.parent, s.best, s.table, s.count);
            k_merge_flatten<<<node_grid, 256, 0, st>>>(r, s.linked, nodes, s.parent, s.best);
        }
    }
    // the cut starts from singletons again; only the region count needs the forest in key order
    const unsigned long long* forest = s.table;
    if (mode == FSLIC_MERGE_NUM_REGIONS && edges) {
        k_merge_segments<<<ceil_div(batch, 256), 256, 0, st>>>(batch, K, s.count, s.seg_begin, s.seg_end);
        size_t temp_bytes = s.temp_bytes;
        if (cub::DeviceSegmentedRadixSort::SortKeys(s.temp, temp_bytes, s.table, s.sorted, (int)nodes, batch,
                                                    (const int*)s.seg_begin, (const int*)s.seg_end, 0, 64,
                                                    st) != cudaSuccess)
            return set_err(FSLIC_ECUDA, "segmented radix sort of the forest edges failed");
        forest = s.sorted;
    }
    k_merge_init<<<node_grid, 256, 0, st>>>(nodes, s.parent, s.best);
    if (edges) {
        k_merge_cut<<<node_grid, 256, 0, st>>>(nodes, K, mode == FSLIC_MERGE_NUM_REGIONS, threshold, num_regions,
                                               forest, s.count, s.P, s.parent);
        k_merge_flatten<<<node_grid, 256, 0, st>>>(0, s.linked, nodes, s.parent, s.best);
    }
    k_merge_roots<<<(int)grid_for(nodes + 1, device), 256, 0, st>>>(nodes, s.present, s.parent, s.flag);
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceScan::ExclusiveSum(s.temp, temp_bytes, (const int*)s.flag, s.pos, (int)nodes + 1, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "scan of the region roots failed");
    k_merge_number<<<node_grid, 256, 0, st>>>(nodes, K, s.present, s.parent, s.pos, d_region, d_num_regions);
    CK(cudaGetLastError());
    return fslic_b200_pool_paint_batch(device, batch, H, W, K, d_labels, d_region, d_out, stream);
}
