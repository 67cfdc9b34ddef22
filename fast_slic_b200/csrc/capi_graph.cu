// fast_slic_b200/csrc/capi_graph.cu -- the extern "C" entry points of the label-map consumers (graph.cuh): the
// adjacency graph, mask density and density broadcast.  Stateless (device pointers, caller-provided scratch),
// asynchronous on the caller's stream, never synchronise.  A single-image call is the batch call with batch = 1.
#include <limits.h>

#include "capi_common.h"
#include "cub_temp.cuh"  // library sort for the adjacency graph only (not on the hot path)
#include "graph.cuh"

// Slots of one image's pair table: a power of two >= max(4096, 32 K)
static uint32_t conn_table_size(int K) {
    uint32_t t = 4096;
    while (t < 32u * (uint32_t)K) t <<= 1;  // a superpixel map has ~3 distinct adjacent pairs per label
    return t;
}
// Key and order tables, their sorted copies, the sort's temporary storage (sized for all 64 key bits, an upper bound
// of what a call sorts) and the per-image overflow flags.
struct ConnScratch {
    uint32_t *tkey, *skey;
    unsigned long long *tord, *sord;
    void* temp;
    int* overflow;
    size_t temp_bytes, total;
};

static ConnScratch conn_layout(int batch, long long slots, void* base) {
    ConnScratch s;
    Carve c(base);
    s.tkey = c.take<uint32_t>((size_t)slots * 4);
    s.skey = c.take<uint32_t>((size_t)slots * 4);
    s.tord = c.take<unsigned long long>((size_t)slots * 8);
    s.sord = c.take<unsigned long long>((size_t)slots * 8);
    s.temp_bytes = align_up(radix_pairs_temp_bytes<unsigned long long, uint32_t>(slots, 64), 256);
    s.temp = c.take<void>(s.temp_bytes);
    s.overflow = c.take<int>((size_t)batch * 4);
    s.total = c.total;
    return s;
}

extern "C" size_t fslic_b200_connectivity_batch_scratch_bytes(int K, int batch) {
    if (K <= 0 || batch <= 0) return 256;
    if (K > 65535) return (size_t)-1;
    const long long slots = (long long)conn_table_size(K) * batch;
    if (slots > INT_MAX) return (size_t)-1;  // more than one radix sort takes: the call refuses such a batch
    return conn_layout(batch, slots, nullptr).total;
}

extern "C" int fslic_b200_get_connectivity_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                                 int32_t* d_counts, uint32_t* d_neighbors, int32_t* d_replayed,
                                                 void* d_scratch, size_t scratch_bytes, void* stream) {
    if (batch < 0 || H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    if (batch == 0) return FSLIC_OK;
    if (!d_labels || !d_counts || !d_neighbors || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    const uint32_t T = conn_table_size(K);
    const long long slots = (long long)T * batch;
    if (slots > INT_MAX) return set_err(FSLIC_EINVAL, "batch too large for one call: the pair tables exceed 2^31 slots");
    const int obits = bit_length(3ull * (unsigned long long)H * (unsigned long long)W), bits = obits + bit_length(batch - 1);
    if (bits > 64) return set_err(FSLIC_EINVAL, "batch * H * W too large");
    USE_DEVICE(device);
    if (scratch_bytes < fslic_b200_connectivity_batch_scratch_bytes(K, batch)) return set_err(FSLIC_EINVAL, "scratch too small");
    cudaStream_t st = (cudaStream_t)stream;
    const ConnScratch s = conn_layout(batch, slots, d_scratch);
    if (radix_pairs_temp_bytes<unsigned long long, uint32_t>(slots, bits) > s.temp_bytes)
        return set_err(FSLIC_ECUDA, "radix sort temporary storage");
    // the walk's shared memory: u8 counts of the K labels + the staged chunk; opted in once per device for any K
    const int smem = ((K + 15) & ~15) + CONNB_CHUNK * 4, smem_max = 65536 + CONNB_CHUNK * 4;
    static bool walk_smem_set[64] = {};
    if (device < 0 || device >= 64 || !walk_smem_set[device]) {
        CK(cudaFuncSetAttribute(k_connb_walk, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
        if (device >= 0 && device < 64) walk_smem_set[device] = true;
    }
    k_connb_init<<<(int)grid_for(slots, device), 256, 0, st>>>(s.tkey, s.tord, slots, bit_length(T) - 1, obits, batch,
                                                                s.overflow);
    const long n = (long)batch * (H - 1) * (W - 1);
    if (n > 0)
        k_connb_discover<<<(int)grid_for(n, device), 256, 0, st>>>(d_labels, batch, H, W, K, s.tkey, s.tord, T, obits,
                                                                   s.overflow);
    size_t temp_bytes = s.temp_bytes;
    if (cub::DeviceRadixSort::SortPairs(s.temp, temp_bytes, s.tord, s.sord, s.tkey, s.skey, (int)slots, 0, bits, st) !=
        cudaSuccess)
        return set_err(FSLIC_ECUDA, "radix sort of the pair tables failed");
    k_connb_walk<<<batch, 256, smem, st>>>(s.skey, T, d_labels, H, W, K, s.overflow, d_counts, d_neighbors, d_replayed);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_get_mask_density_batch(int device, int batch, int H, int W, int K, const fslic_cluster* d_clusters,
                                                 const uint16_t* d_labels, const uint8_t* d_masks, uint8_t* d_densities,
                                                 int32_t* d_scratch, void* stream) {
    if (batch < 0 || H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    if (batch == 0) return FSLIC_OK;
    if (!d_clusters || !d_labels || !d_masks || !d_densities || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    cudaStream_t st = (cudaStream_t)stream;
    const long n = (long)H * W, nk = (long)batch * K;
    CK(cudaMemsetAsync(d_scratch, 0, (size_t)nk * 4, st));
    k_mask_sum_batch<<<(int)grid_for(n * batch, device), 256, 0, st>>>(d_labels, d_masks, n, batch, K, d_scratch);
    k_density_final_batch<<<(int)grid_for(nk, device), 256, 0, st>>>(d_scratch, d_clusters, nk, d_densities);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

extern "C" int fslic_b200_cluster_density_to_mask_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                                        const uint8_t* d_densities, uint8_t* d_result, void* stream) {
    if (batch < 0 || H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad batch, H, W or K");
    if (batch == 0) return FSLIC_OK;
    if (!d_labels || !d_densities || !d_result) return set_err(FSLIC_EINVAL, "NULL argument");
    USE_DEVICE(device);
    const long n = (long)H * W;
    k_density_broadcast_batch<<<(int)grid_for(n * batch, device), 256, 0, (cudaStream_t)stream>>>(d_labels, d_densities, n,
                                                                                                   batch, K, d_result);
    CK(cudaGetLastError());
    return FSLIC_OK;
}

// ---- single images: batches of one, each with its own argument checks --------------------------------------------
extern "C" size_t fslic_b200_connectivity_scratch_bytes(int K) { return fslic_b200_connectivity_batch_scratch_bytes(K, 1); }

extern "C" int fslic_b200_get_connectivity(int device, int H, int W, int K, const uint16_t* d_labels, int32_t* d_counts,
                                           uint32_t* d_neighbors, void* d_scratch, size_t scratch_bytes, void* stream) {
    if (H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad H, W or K");
    if (!d_labels || !d_counts || !d_neighbors || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    if (scratch_bytes < fslic_b200_connectivity_scratch_bytes(K)) return set_err(FSLIC_EINVAL, "scratch too small");
    return fslic_b200_get_connectivity_batch(device, 1, H, W, K, d_labels, d_counts, d_neighbors, nullptr, d_scratch,
                                             scratch_bytes, stream);
}

extern "C" int fslic_b200_get_mask_density(int device, int H, int W, int K, const fslic_cluster* d_clusters,
                                           const uint16_t* d_labels, const uint8_t* d_mask, uint8_t* d_densities,
                                           int32_t* d_scratch, void* stream) {
    if (H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad H, W or K");
    if (!d_clusters || !d_labels || !d_mask || !d_densities || !d_scratch) return set_err(FSLIC_EINVAL, "NULL argument");
    return fslic_b200_get_mask_density_batch(device, 1, H, W, K, d_clusters, d_labels, d_mask, d_densities, d_scratch,
                                             stream);
}

extern "C" int fslic_b200_cluster_density_to_mask(int device, int H, int W, int K, const uint16_t* d_labels,
                                                  const uint8_t* d_densities, uint8_t* d_result, void* stream) {
    if (H <= 0 || W <= 0 || K <= 0 || K > 65535) return set_err(FSLIC_EINVAL, "bad H, W or K");
    if (!d_labels || !d_densities || !d_result) return set_err(FSLIC_EINVAL, "NULL argument");
    return fslic_b200_cluster_density_to_mask_batch(device, 1, H, W, K, d_labels, d_densities, d_result, stream);
}
