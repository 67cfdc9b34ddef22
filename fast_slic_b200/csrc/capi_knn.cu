// fast_slic_b200/csrc/capi_knn.cu -- the extern "C" entry points of the k-nearest-neighbour graph (knn.cuh).
// Stateless (device pointers, caller-provided scratch), asynchronous on the caller's stream, never synchronise: the
// caller reads the edge total back between the count and the fill.
#include <limits.h>

#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "knn.cuh"

#define KNN_MAX_D 64
#define KNN_MAX_NEIGHBORS 32
#define KNN_MAX_NODES (1LL << 30)

static bool knn_args_ok(int batch, int K, int D, int k) {
    return batch >= 0 && K >= 1 && K <= MAX_K && D >= 1 && D <= KNN_MAX_D && k >= 1 && k <= KNN_MAX_NEIGHBORS &&
           (long long)batch * K <= KNN_MAX_NODES &&
           2LL * batch * K * k <= INT_MAX;  // both directions of every slot in one radix sort
}

// Coordinates per packed candidate: D padded to a power of two >= 4
static int knn_padded(int D) {
    int p = 4;
    while (p < D) p <<= 1;
    return p;
}

static size_t knn_flagged_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceSelect::Flagged(nullptr, bytes, thrust::counting_iterator<uint32_t>(0), (const uint8_t*)nullptr,
                               (uint32_t*)nullptr, (int*)nullptr, (int)items);
    return bytes;
}

static size_t knn_unique_temp_bytes(long long items) {
    size_t bytes = 0;
    cub::DeviceSelect::UniqueByKey(nullptr, bytes, (const unsigned long long*)nullptr, (const float*)nullptr,
                                   (unsigned long long*)nullptr, (float*)nullptr, (int*)nullptr, (int)items);
    return bytes;
}

// One call's scratch, which the count writes and the fill reads: per node the candidacy flag, the candidate list, the
// packed coordinates (4 * DP bytes), the row count and offset and the k-slot neighbour table (8 * k bytes); per image
// the candidate starts; with `symmetric` the 2k pair keys and values per node, their sorted and unique copies
// (72 * k bytes per node) and the unique count; the largest temporary storage of the cub calls
struct KnnScratch {
    uint8_t* flags;
    uint32_t *cand, *idx;
    int *ncand, *starts, *count, *offs, *nunique;
    float *packed, *dist, *vals, *svals, *uvals;
    unsigned long long *keys, *skeys, *ukeys;
    void* temp;
    size_t temp_bytes, total;
};

static KnnScratch knn_layout(int batch, int K, int D, int k, int symmetric, void* base) {
    KnnScratch s{};
    Carve c(base);
    const long long nodes = (long long)batch * K, slots = nodes * k, pairs = 2 * slots;
    s.flags = c.take<uint8_t>((size_t)nodes);
    s.cand = c.take<uint32_t>((size_t)nodes * 4);
    s.ncand = c.take<int>(4);
    s.starts = c.take<int>(((size_t)batch + 1) * 4);
    s.packed = c.take<float>((size_t)nodes * knn_padded(D) * 4);
    s.count = c.take<int>(((size_t)nodes + 1) * 4);
    s.offs = c.take<int>(((size_t)nodes + 1) * 4);
    s.idx = c.take<uint32_t>((size_t)slots * 4);
    s.dist = c.take<float>((size_t)slots * 4);
    size_t temp = knn_flagged_temp_bytes(nodes), t2 = exclusive_sum_temp_bytes<int>(nodes + 1);
    if (t2 > temp) temp = t2;
    if (symmetric) {
        s.keys = c.take<unsigned long long>((size_t)pairs * 8);
        s.skeys = c.take<unsigned long long>((size_t)pairs * 8);
        s.ukeys = c.take<unsigned long long>((size_t)pairs * 8);
        s.vals = c.take<float>((size_t)pairs * 4);
        s.svals = c.take<float>((size_t)pairs * 4);
        s.uvals = c.take<float>((size_t)pairs * 4);
        s.nunique = c.take<int>(4);
        const size_t t3 = radix_pairs_temp_bytes<unsigned long long, float>(pairs, 64), t4 = knn_unique_temp_bytes(pairs);
        if (t3 > temp) temp = t3;
        if (t4 > temp) temp = t4;
    }
    s.temp_bytes = align_up(temp, 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_knn_scratch_bytes(int batch, int K, int D, int k, int symmetric) {
    if (!knn_args_ok(batch, K, D, k)) return (size_t)-1;
    return knn_layout(batch, K, D, k, symmetric != 0, nullptr).total;
}

template <int KC, int DP>
static void knn_launch_select(dim3 grid, cudaStream_t st, const KnnScratch& s, int batch, int K, int k) {
    k_knn_select<KC, DP><<<grid, KNN_THREADS, 0, st>>>(s.packed, s.cand, s.starts, batch, K, k, s.count, s.idx, s.dist);
}

template <int KC>
static void knn_select_for_d(int DP, dim3 grid, cudaStream_t st, const KnnScratch& s, int batch, int K, int k) {
    switch (DP) {
        case 4: knn_launch_select<KC, 4>(grid, st, s, batch, K, k); break;
        case 8: knn_launch_select<KC, 8>(grid, st, s, batch, K, k); break;
        case 16: knn_launch_select<KC, 16>(grid, st, s, batch, K, k); break;
        case 32: knn_launch_select<KC, 32>(grid, st, s, batch, K, k); break;
        default: knn_launch_select<KC, 64>(grid, st, s, batch, K, k); break;
    }
}

extern "C" int fslic_b200_knn_count(int device, int batch, int K, int D, int k, int symmetric, const float* d_points,
                                    const uint8_t* d_present, long long edge_base, long long* d_indptr,
                                    long long* d_total, void* d_scratch, size_t scratch_bytes, void* stream) {
    if (!knn_args_ok(batch, K, D, k) || edge_base < 0) return set_err(FSLIC_EINVAL, "bad batch, K, D, k or edge base");
    if (!d_indptr || !d_total) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long nodes = (long)batch * K;
    if (nodes == 0) {  // indptr[0] = edge_base, no edges (pageable source: the copy is staged before the call returns)
        CK(cudaMemcpyAsync(d_indptr, &edge_base, 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_total, 0, 8, st));
        return FSLIC_OK;
    }
    const size_t need = fslic_b200_knn_scratch_bytes(batch, K, D, k, symmetric);
    if (!d_points || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    const KnnScratch s = knn_layout(batch, K, D, k, symmetric != 0, d_scratch);
    const int DP = knn_padded(D);
    k_knn_flags<<<(int)grid_for(nodes, device), 256, 0, st>>>(d_points, d_present, nodes, D, s.flags);
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceSelect::Flagged(s.temp, temp_bytes, thrust::counting_iterator<uint32_t>(0), s.flags, s.cand, s.ncand,
                                   (int)nodes, st) != cudaSuccess)
        return set_err(FSLIC_ECUDA, "selection of the candidates failed");
    k_knn_starts<<<(int)grid_for((long)batch + 1, device), 256, 0, st>>>(s.cand, s.ncand, batch, K, s.starts);
    k_knn_pack<<<(int)grid_for(nodes * DP, device), 256, 0, st>>>(d_points, s.cand, s.ncand, D, DP, s.packed);
    CK(cudaMemsetAsync(s.count, 0, ((size_t)nodes + 1) * 4, st));
    const dim3 grid((unsigned)((K + KNN_THREADS - 1) / KNN_THREADS), batch < 65535 ? (unsigned)batch : 65535u);
    if (k <= 8) knn_select_for_d<8>(DP, grid, st, s, batch, K, k);
    else knn_select_for_d<32>(DP, grid, st, s, batch, K, k);
    const long slots = nodes * k;
    if (!symmetric) {
        temp_bytes = s.temp_bytes;
        if (cub::DeviceScan::ExclusiveSum(s.temp, temp_bytes, s.count, s.offs, (int)(nodes + 1), st) != cudaSuccess)
            return set_err(FSLIC_ECUDA, "scan of the row counts failed");
        k_knn_rows<<<(int)grid_for(nodes + 1, device), 256, 0, st>>>(s.offs, nodes, edge_base, d_indptr, d_total);
    } else {
        k_knn_pairs<<<(int)grid_for(slots, device), 256, 0, st>>>(s.count, s.idx, s.dist, nodes, K, k, s.keys, s.vals);
        const int bits = 16 + bit_length((unsigned long long)(nodes - 1));  // row << 16 | target
        temp_bytes = s.temp_bytes;
        if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.keys, s.skeys, s.vals, s.svals, (int)(2 * slots), 0,
                                            bits, st) != cudaSuccess)
            return set_err(FSLIC_ECUDA, "radix sort of the edge keys failed");
        temp_bytes = s.temp_bytes;
        if (cub::DeviceSelect::UniqueByKey(s.temp, temp_bytes, s.skeys, s.svals, s.ukeys, s.uvals, s.nunique,
                                           (int)(2 * slots), st) != cudaSuccess)
            return set_err(FSLIC_ECUDA, "deduplication of the edge keys failed");
        k_knn_unique_rows<<<(int)grid_for(nodes + 1, device), 256, 0, st>>>(s.ukeys, s.nunique, nodes, edge_base,
                                                                            d_indptr, d_total);
    }
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_knn_fill(int device, int batch, int K, int D, int k, int symmetric, long long node_base,
                                   long long edges, const void* d_scratch, size_t scratch_bytes, long long* d_src,
                                   long long* d_dst, float* d_distance, void* stream) {
    if (!knn_args_ok(batch, K, D, k) || node_base < 0 || edges < 0 || edges > 2LL * batch * K * k)
        return set_err(FSLIC_EINVAL, "bad batch, K, D, k, node base or edges");
    if (edges == 0) return FSLIC_OK;
    if (!d_scratch || !d_src || !d_dst || !d_distance) return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < fslic_b200_knn_scratch_bytes(batch, K, D, k, symmetric))
        return set_err(FSLIC_EINVAL, "scratch too small");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const KnnScratch s = knn_layout(batch, K, D, k, symmetric != 0, const_cast<void*>(d_scratch));
    const long nodes = (long)batch * K;
    if (!symmetric)
        k_knn_emit_directed<<<(int)grid_for(nodes * k, device), 256, 0, st>>>(s.count, s.offs, s.idx, s.dist, nodes, K,
                                                                             k, node_base, d_src, d_dst, d_distance);
    else
        k_knn_emit_symmetric<<<(int)grid_for(edges, device), 256, 0, st>>>(s.ukeys, s.uvals, (long)edges, K, node_base,
                                                                          d_src, d_dst, d_distance);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
