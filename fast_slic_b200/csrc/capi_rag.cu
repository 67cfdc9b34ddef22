// fast_slic_b200/csrc/capi_rag.cu -- the extern "C" entry points of region adjacency graphs (rag.cuh).  Stateless
// (device pointers, caller-provided scratch), asynchronous on the caller's stream, never synchronise: the caller reads
// the edge total back between the count and the fill.
#include <limits.h>

#include "capi_common.h"
#include "cub_temp.cuh"
#include "rag.cuh"

#define RAG_MAX_PROBES 512u

static bool rag_args_ok(int batch, int H, int W, int K, int connectivity) {
    return labels_shape_ok(batch, H, W, K) && (connectivity == 4 || connectivity == 8);
}

// Slots T of one image's pair table (a power of two) and the probe limit.  An image has at most
// m = min(K (K - 1) / 2, its pixel pairs) distinct keys; 2m slots or more hold them at a load of at most 1/2, and with
// no probe limit such a table cannot overflow.  `exact` takes that size (false if it exceeds 2^31 slots).  Otherwise
// the table takes the smaller of that size and the adjacency graph's power of two >= max(4096, 32 K), whose probe
// limit flags the image as overflowed instead.
static bool rag_table(int H, int W, int K, int connectivity, int exact, uint32_t* T, uint32_t* max_probes) {
    const long long h = H, w = W;
    long long pairs = h * (w - 1) + (h - 1) * w;
    if (connectivity == 8) pairs += 2 * (h - 1) * (w - 1);
    const long long keys = (long long)K * (K - 1) / 2;
    const long long need = 2 * (keys < pairs ? keys : pairs);
    long long t_exact = 1;
    while (t_exact < need) t_exact <<= 1;
    uint32_t t_graph = 4096;
    while (t_graph < 32u * (uint32_t)K) t_graph <<= 1;
    if (exact || t_exact <= (long long)t_graph) {
        if (t_exact > (1LL << 31)) return false;
        *T = (uint32_t)t_exact;
        *max_probes = (uint32_t)t_exact;
    } else {
        *T = t_graph;
        *max_probes = RAG_MAX_PROBES;
    }
    return true;
}

// The count's scratch, which the fill reads: pair keys and counts (4 bytes each per slot), the degrees and the
// call-local row offsets (8 bytes each per node, plus one), and the scan's temporary storage.
struct RagScratch {
    uint32_t *key, *cnt;
    unsigned long long* deg;
    long long* local;
    void* temp;
    size_t temp_bytes, total;
};

static RagScratch rag_layout(int batch, uint32_t T, int K, const void* base) {
    const size_t slots = (size_t)T * batch, nk1 = (size_t)batch * K + 1;
    RagScratch s;
    Carve c(const_cast<void*>(base));
    s.key = c.take<uint32_t>(slots * 4);
    s.cnt = c.take<uint32_t>(slots * 4);
    s.deg = c.take<unsigned long long>(nk1 * 8);
    s.local = c.take<long long>(nk1 * 8);
    s.temp_bytes = align_up(exclusive_sum_temp_bytes<long long>((long long)nk1), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

// The fill's own scratch: edge keys and their sorted copy (8 bytes each per edge), the boundary counts (4 bytes per
// edge) and the sort's temporary storage (sized for all 64 key bits)
struct RagFillScratch {
    unsigned long long *ekey, *skey;
    int32_t* val;
    void* temp;
    size_t temp_bytes, total;
};

static RagFillScratch rag_fill_layout(long long edges, void* base) {
    RagFillScratch s;
    Carve c(base);
    s.ekey = c.take<unsigned long long>((size_t)edges * 8);
    s.skey = c.take<unsigned long long>((size_t)edges * 8);
    s.val = c.take<int32_t>((size_t)edges * 4);
    s.temp_bytes = align_up(radix_pairs_temp_bytes<unsigned long long, int32_t>(edges, 64), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_rag_batch_scratch_bytes(int batch, int H, int W, int K, int connectivity, int exact) {
    if (!rag_args_ok(batch, H, W, K, connectivity)) return (size_t)-1;
    if ((long long)H * W > MAX_IMAGE_PIXELS) return (size_t)-1;
    if ((long long)batch * H * W == 0) return 256;
    if ((long long)batch * K + 1 > INT_MAX) return (size_t)-1;  // one scan and one sort: split the batch
    uint32_t T, probes;
    if (!rag_table(H, W, K, connectivity, exact, &T, &probes)) return (size_t)-1;
    return rag_layout(batch, T, K, nullptr).total;
}

extern "C" int fslic_b200_rag_batch_count(int device, int batch, int H, int W, int K, int connectivity, int exact,
                                          const uint16_t* d_labels, long long edge_base, long long* d_indptr,
                                          long long* d_info, void* d_scratch, size_t scratch_bytes, void* stream) {
    if (!rag_args_ok(batch, H, W, K, connectivity) || edge_base < 0)
        return set_err(FSLIC_EINVAL, "bad batch, H, W, K, connectivity or edge base");
    const long hw = (long)H * W, n = (long)batch * hw;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_indptr || !d_info || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_rag_batch_scratch_bytes(batch, H, W, K, connectivity, exact);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "image or batch too large for one call");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    uint32_t T, max_probes;
    rag_table(H, W, K, connectivity, exact, &T, &max_probes);
    const RagScratch s = rag_layout(batch, T, K, d_scratch);
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long slots = (long)T * batch, nk = (long)batch * K;
    CK(cudaMemsetAsync(s.key, 0xff, (size_t)slots * 4, st));
    CK(cudaMemsetAsync(s.cnt, 0, (size_t)slots * 4, st));
    CK(cudaMemsetAsync(s.deg, 0, (size_t)(nk + 1) * 8, st));
    CK(cudaMemsetAsync(d_info, 0, (size_t)batch * 8, st));
    if (connectivity == 4)
        k_rag_discover<4><<<(int)grid_for(n, device), 256, 0, st>>>(d_labels, hw, H, W, n, K, s.key, s.cnt, T, max_probes,
                                                                     d_info);
    else
        k_rag_discover<8><<<(int)grid_for(n, device), 256, 0, st>>>(d_labels, hw, H, W, n, K, s.key, s.cnt, T, max_probes,
                                                                     d_info);
    k_rag_degree<<<(int)grid_for(slots, device), 256, 0, st>>>(s.key, slots, bit_length(T) - 1, K, s.deg);
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceScan::ExclusiveSum(s.temp, temp_bytes, (const long long*)s.deg, s.local, (int)(nk + 1), st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "scan of the degrees failed");
    k_rag_finish<<<(int)grid_for(nk + 1, device), 256, 0, st>>>(s.local, nk, edge_base, d_indptr, d_info + batch);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" size_t fslic_b200_rag_fill_scratch_bytes(int batch, int K, long long edges) {
    if (batch < 0 || K < 1 || K > MAX_K || edges < 0 || edges > INT_MAX || (long long)batch * K + 1 > INT_MAX)
        return (size_t)-1;
    if (edges == 0) return 256;
    return rag_fill_layout(edges, nullptr).total;
}

extern "C" int fslic_b200_rag_batch_fill(int device, int batch, int H, int W, int K, int connectivity, int exact,
                                         long long node_base, long long edges, const void* d_scratch,
                                         size_t scratch_bytes, void* d_fill_scratch, size_t fill_bytes,
                                         long long* d_src, long long* d_dst, int32_t* d_boundary, void* stream) {
    if (!rag_args_ok(batch, H, W, K, connectivity) || node_base < 0)
        return set_err(FSLIC_EINVAL, "bad batch, H, W, K, connectivity or node base");
    const long n = (long)batch * H * W;
    if (n == 0 || edges == 0) return FSLIC_OK;
    if (!d_scratch || !d_fill_scratch || !d_src || !d_dst || !d_boundary) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_rag_batch_scratch_bytes(batch, H, W, K, connectivity, exact);
    const size_t fill_need = fslic_b200_rag_fill_scratch_bytes(batch, K, edges);
    if (need == (size_t)-1 || fill_need == (size_t)-1) return set_err(FSLIC_EINVAL, "image, batch or edge count too large");
    if (scratch_bytes < need || fill_bytes < fill_need) return set_err(FSLIC_EINVAL, "scratch too small");
    uint32_t T, max_probes;
    rag_table(H, W, K, connectivity, exact, &T, &max_probes);
    const RagScratch s = rag_layout(batch, T, K, d_scratch);
    const RagFillScratch f = rag_fill_layout(edges, d_fill_scratch);
    const long slots = (long)T * batch, nk = (long)batch * K;
    size_t temp_bytes = f.temp_bytes;
    const int bits = 16 + bit_length((unsigned long long)(nk - 1));  // row << 16 | target
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaMemsetAsync(s.deg, 0, (size_t)nk * 8, st));  // the row cursors
    k_rag_scatter<<<(int)grid_for(slots, device), 256, 0, st>>>(s.key, s.cnt, slots, bit_length(T) - 1, K, s.local, s.deg,
                                                                f.ekey, f.val);
    if (cub::DeviceRadixSort::SortPairs(f.temp, temp_bytes, f.ekey, f.skey, f.val, d_boundary, (int)edges, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the edges failed");
    k_rag_emit<<<(int)grid_for(edges, device), 256, 0, st>>>(f.skey, edges, K, node_base, d_src, d_dst);
    CK(cudaGetLastError());
    return FSLIC_OK;
}
