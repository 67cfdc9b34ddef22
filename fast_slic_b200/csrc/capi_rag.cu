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

static bool rag3d_args_ok(int batch, int D, int H, int W, int K, int connectivity) {
    return labels_shape_ok(batch, H, W, K) && D >= 0 && (connectivity == 6 || connectivity == 18 || connectivity == 26);
}

// Pixel pairs of one H x W image: right and down, with connectivity 8 both diagonals too
static long long rag_pairs(int H, int W, int connectivity) {
    const long long h = H, w = W;
    long long pairs = h * (w - 1) + (h - 1) * w;
    if (connectivity == 8) pairs += 2 * (h - 1) * (w - 1);
    return pairs;
}

// Voxel pairs of one D x H x W volume: sum over the 3, 9 or 13 forward offsets (dz, dy, dx) of
// (D - |dz|)(H - |dy|)(W - |dx|), offsets with 1, <= 2 or <= 3 non-zero components; 0 for an empty volume
static long long rag3d_pairs(int D, int H, int W, int connectivity) {
    if ((long long)D * H * W == 0) return 0;
    const long long L[3][2] = {{D, D - 1}, {H, H - 1}, {W, W - 1}};  // extent along an axis for offset 0, +-1
    const int most = connectivity == 6 ? 1 : (connectivity == 18 ? 2 : 3);
    long long pairs = 0;
    for (int dz = 0; dz <= 1; dz++)
        for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) {
                const bool forward = dz > 0 || (dz == 0 && (dy > 0 || (dy == 0 && dx > 0)));
                const int nz = (dz != 0) + (dy != 0) + (dx != 0);
                if (forward && nz <= most) pairs += L[0][dz != 0] * L[1][dy != 0] * L[2][dx != 0];
            }
    return pairs;
}

// Slots T of one image's pair table (a power of two) and the probe limit.  An image (or volume) has at most
// m = min(K (K - 1) / 2, its pixel pairs) distinct keys; 2m slots or more hold them at a load of at most 1/2, and with
// no probe limit such a table cannot overflow.  `exact` takes that size (false if it exceeds 2^31 slots).  Otherwise
// the table takes the smaller of that size and the adjacency graph's power of two >= max(4096, 32 K), whose probe
// limit flags the image as overflowed instead.
static bool rag_table(long long pairs, int K, int exact, uint32_t* T, uint32_t* max_probes) {
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

// A volume of at most MAX_IMAGE_PIXELS voxels (no overflow: H W <= 2^29 before D multiplies it)
static bool rag3d_volume_ok(int D, int H, int W) {
    const long long hw = (long long)H * W;
    return D == 0 || hw == 0 || (hw <= MAX_IMAGE_PIXELS && (long long)D * hw <= MAX_IMAGE_PIXELS);
}

// The count's scratch bytes of `batch` images (or volumes) of `pixels` elements and `pairs` element pairs each
static size_t rag_scratch_bytes(int batch, long long pixels, long long pairs, int K, int exact) {
    if ((long long)batch * pixels == 0) return 256;
    if ((long long)batch * K + 1 > INT_MAX) return (size_t)-1;  // one scan and one sort: split the batch
    uint32_t T, probes;
    if (!rag_table(pairs, K, exact, &T, &probes)) return (size_t)-1;
    return rag_layout(batch, T, K, nullptr).total;
}

// Everything of a count but the discover launch, which `discover(key, cnt, T, max_probes, grid, stream)` makes: the
// table and degree resets, the degrees, their scan and the row offsets.  Arguments checked by the caller.
template <typename Discover>
static int rag_count(int device, int batch, long n, long long pairs, int K, int exact, long long edge_base,
                     long long* d_indptr, long long* d_info, void* d_scratch, void* stream, Discover discover) {
    uint32_t T, max_probes;
    rag_table(pairs, K, exact, &T, &max_probes);
    const RagScratch s = rag_layout(batch, T, K, d_scratch);
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long slots = (long)T * batch, nk = (long)batch * K;
    CK(cudaMemsetAsync(s.key, 0xff, (size_t)slots * 4, st));
    CK(cudaMemsetAsync(s.cnt, 0, (size_t)slots * 4, st));
    CK(cudaMemsetAsync(s.deg, 0, (size_t)(nk + 1) * 8, st));
    CK(cudaMemsetAsync(d_info, 0, (size_t)batch * 8, st));
    discover(s.key, s.cnt, T, max_probes, (int)grid_for(n, device), st);
    k_rag_degree<<<(int)grid_for(slots, device), 256, 0, st>>>(s.key, slots, bit_length(T) - 1, K, s.deg);
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceScan::ExclusiveSum(s.temp, temp_bytes, (const long long*)s.deg, s.local, (int)(nk + 1), st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "scan of the degrees failed");
    k_rag_finish<<<(int)grid_for(nk + 1, device), 256, 0, st>>>(s.local, nk, edge_base, d_indptr, d_info + batch);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// The fill after a count of the same tables: scatter, sort and emit.  Arguments checked by the caller.
static int rag_fill(int device, int batch, long long pairs, int K, int exact, long long node_base, long long edges,
                    const void* d_scratch, void* d_fill_scratch, long long* d_src, long long* d_dst, int32_t* d_boundary,
                    void* stream) {
    uint32_t T, max_probes;
    rag_table(pairs, K, exact, &T, &max_probes);
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

extern "C" size_t fslic_b200_rag_batch_scratch_bytes(int batch, int H, int W, int K, int connectivity, int exact) {
    if (!rag_args_ok(batch, H, W, K, connectivity)) return (size_t)-1;
    if ((long long)H * W > MAX_IMAGE_PIXELS) return (size_t)-1;
    return rag_scratch_bytes(batch, (long long)H * W, rag_pairs(H, W, connectivity), K, exact);
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
    return rag_count(device, batch, n, rag_pairs(H, W, connectivity), K, exact, edge_base, d_indptr, d_info, d_scratch,
                     stream, [&](uint32_t* key, uint32_t* cnt, uint32_t T, uint32_t max_probes, int grid, cudaStream_t st) {
                         if (connectivity == 4)
                             k_rag_discover<4><<<grid, 256, 0, st>>>(d_labels, hw, H, W, n, K, key, cnt, T, max_probes,
                                                                     d_info);
                         else
                             k_rag_discover<8><<<grid, 256, 0, st>>>(d_labels, hw, H, W, n, K, key, cnt, T, max_probes,
                                                                     d_info);
                     });
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
    return rag_fill(device, batch, rag_pairs(H, W, connectivity), K, exact, node_base, edges, d_scratch, d_fill_scratch,
                    d_src, d_dst, d_boundary, stream);
}

extern "C" size_t fslic_b200_rag3d_batch_scratch_bytes(int batch, int D, int H, int W, int K, int connectivity,
                                                       int exact) {
    if (!rag3d_args_ok(batch, D, H, W, K, connectivity) || !rag3d_volume_ok(D, H, W)) return (size_t)-1;
    const long long pairs = rag3d_pairs(D, H, W, connectivity);
    if (pairs > INT_MAX) return (size_t)-1;  // a boundary count could exceed int32
    return rag_scratch_bytes(batch, (long long)D * H * W, pairs, K, exact);
}

extern "C" int fslic_b200_rag3d_batch_count(int device, int batch, int D, int H, int W, int K, int connectivity,
                                            int exact, const uint16_t* d_labels, long long edge_base,
                                            long long* d_indptr, long long* d_info, void* d_scratch,
                                            size_t scratch_bytes, void* stream) {
    if (!rag3d_args_ok(batch, D, H, W, K, connectivity) || !rag3d_volume_ok(D, H, W) || edge_base < 0)
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, K, connectivity or edge base");
    const long dhw = (long)D * H * W, n = (long)batch * dhw;
    if (n == 0) return FSLIC_OK;
    if (!d_labels || !d_indptr || !d_info || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_rag3d_batch_scratch_bytes(batch, D, H, W, K, connectivity, exact);
    if (need == (size_t)-1) return set_err(FSLIC_EINVAL, "volume or batch too large for one call");
    if (scratch_bytes < need) return set_err(FSLIC_EINVAL, "scratch too small");
    return rag_count(device, batch, n, rag3d_pairs(D, H, W, connectivity), K, exact, edge_base, d_indptr, d_info,
                     d_scratch, stream,
                     [&](uint32_t* key, uint32_t* cnt, uint32_t T, uint32_t max_probes, int grid, cudaStream_t st) {
                         if (connectivity == 6)
                             k_rag3d_discover<6><<<grid, 256, 0, st>>>(d_labels, dhw, D, H, W, n, K, key, cnt, T,
                                                                       max_probes, d_info);
                         else if (connectivity == 18)
                             k_rag3d_discover<18><<<grid, 256, 0, st>>>(d_labels, dhw, D, H, W, n, K, key, cnt, T,
                                                                        max_probes, d_info);
                         else
                             k_rag3d_discover<26><<<grid, 256, 0, st>>>(d_labels, dhw, D, H, W, n, K, key, cnt, T,
                                                                        max_probes, d_info);
                     });
}

extern "C" int fslic_b200_rag3d_batch_fill(int device, int batch, int D, int H, int W, int K, int connectivity,
                                           int exact, long long node_base, long long edges, const void* d_scratch,
                                           size_t scratch_bytes, void* d_fill_scratch, size_t fill_bytes,
                                           long long* d_src, long long* d_dst, int32_t* d_boundary, void* stream) {
    if (!rag3d_args_ok(batch, D, H, W, K, connectivity) || !rag3d_volume_ok(D, H, W) || node_base < 0)
        return set_err(FSLIC_EINVAL, "bad batch, D, H, W, K, connectivity or node base");
    const long n = (long)batch * D * H * W;
    if (n == 0 || edges == 0) return FSLIC_OK;
    if (!d_scratch || !d_fill_scratch || !d_src || !d_dst || !d_boundary) return set_err(FSLIC_EINVAL, "NULL argument");
    const size_t need = fslic_b200_rag3d_batch_scratch_bytes(batch, D, H, W, K, connectivity, exact);
    const size_t fill_need = fslic_b200_rag_fill_scratch_bytes(batch, K, edges);
    if (need == (size_t)-1 || fill_need == (size_t)-1) return set_err(FSLIC_EINVAL, "volume, batch or edge count too large");
    if (scratch_bytes < need || fill_bytes < fill_need) return set_err(FSLIC_EINVAL, "scratch too small");
    return rag_fill(device, batch, rag3d_pairs(D, H, W, connectivity), K, exact, node_base, edges, d_scratch,
                    d_fill_scratch, d_src, d_dst, d_boundary, stream);
}
