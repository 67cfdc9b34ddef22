/*
 * include/fslic_b200.h -- C ABI of the H100-native (sm_90a) SLIC engine (libfslic_b200.so).
 *
 * This is the drop-in boundary for the reference's hot path.  The reference crosses from
 * Cython into C++ through `fslic::ContextBuilder().build(H, W, K, image, clusters)`,
 * public config fields, `initialize_clusters()` and `iterate(uint16_t*, max_iter)`
 * (fast-slic/src/context.h:24-75,138-150; call sites cfast_slic.pyx:124-147,150-197)
 * and `cca::ConnectivityEnforcer(...).execute()` (src/cca.h:73-81; cfast_slic.pyx:371-396).
 * The entry points below mirror that lifecycle with plain pointers and sizes -- no C++ or
 * torch types -- so any FFI (ctypes, Cython, cgo, JNI) can bind them.  See INTEGRATION.md.
 *
 * Conventions: every function returns 0 on success, a negative FSLIC_E* code otherwise;
 * `fslic_b200_last_error()` gives the message (thread local).  Pointers named d_* are
 * device pointers on the context's device, h_* are host pointers.  `stream` is a
 * cudaStream_t passed as void* (NULL = default stream); device entry points are
 * asynchronous on that stream.
 */
#ifndef FSLIC_B200_H
#define FSLIC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* == `Cluster`, fast-slic/src/fast-slic-common.h:10-23 (32 bytes, align 4). */
typedef struct fslic_cluster {
    float y, x;          /* centre; always integer-valued on this path (context.cpp:368-373) */
    float r, g, b, a;    /* colour; L*2,a,b when convert_to_lab (cielab.h:308-325), `a` unused */
    uint16_t number;     /* == index */
    uint8_t is_active;   /* 1 after iterate (preemptive.h:69-74) */
    uint8_t is_updatable;/* 2 after iterate (preemptive.h:59-67) */
    uint32_t num_members;/* member count of the LAST subsampled update (context.cpp:360-364) */
} fslic_cluster;

/* == the public config fields of fslic::BaseContext (src/context.h:26-36) that the default
 *    Slic path reads; the values SlicModel.iterate() copies in (cfast_slic.pyx:179-187). */
typedef struct fslic_params {
    float compactness;       /* context.h:28 */
    float min_size_factor;   /* context.h:29 */
    int32_t subsample_stride;/* context.h:26 (subsample_stride_config) */
    int32_t convert_to_lab;  /* context.h:30 */
    int32_t max_iter;        /* argument of iterate(), context.h:72 */
    int32_t collect_timing;  /* 1: per-stage CUDA-event timings (fstimer analogue, timer.cpp:4-49); 2: + per-launch assign kernel */
} fslic_params;

enum {
    FSLIC_OK = 0,
    FSLIC_EINVAL = -1,   /* bad argument (reference: ValueError, cfast_slic.pyx:24-27,125,153) */
    FSLIC_ECUDA = -2,    /* CUDA runtime error */
    FSLIC_ENOMEM = -3,
    FSLIC_ERANGE = -4,   /* compactness so large the u16 distance would overflow (UB in the reference) */
    FSLIC_ENOFRAME = -5, /* CRF: no frame with that time (reference: std::out_of_range, IndexError in Python) */
    FSLIC_ECHECK = -6    /* debug_mode: an assign pass disagreed with the trace kernel (fslic_b200_trace_snapshots) */
};

typedef struct fslic_ctx fslic_ctx;

/* Stage ids for fslic_b200_stage_ms(): same section names as the reference's timing report
 * (context.cpp:112-192, cca.cpp:194-259). */
enum {
    FSLIC_T_CIELAB = 0, FSLIC_T_ASSIGN = 1, FSLIC_T_UPDATE = 2, FSLIC_T_FULL_ASSIGN = 3,
    FSLIC_T_CCA = 4, FSLIC_T_TOTAL = 5,
    FSLIC_T_BEFORE_ITERATION = 6, FSLIC_T_AFTER_UPDATE = 7, /* LSC only (zero otherwise), lsc.cpp:12-15,226-307 */
    FSLIC_T_COUNT = 8
};

const char* fslic_b200_last_error(void);
const char* fslic_b200_version(void);
int fslic_b200_sizeof_cluster(void);

/* == ContextBuilder::build + BaseContext ctor (context.h:59-66,149): fixes H, W, K and
 *    S = (int16)sqrt(H*W/K); allocates every scratch buffer for up to max_batch images.
 *    Unlike the reference (which rebuilds a Context per call, cfast_slic.pyx:171-197) the
 *    context is meant to be kept and reused. */
int fslic_b200_create(int device, int H, int W, int K, int max_batch, fslic_ctx** out);
int fslic_b200_destroy(fslic_ctx* ctx);

/* == the scratch of cca::ConnectivityEnforcer alone (cca.cpp:176-192: it needs H, W and nothing of the SLIC
 *    context): a context on which only fslic_b200_enforce_connectivity may be called.  No K is fixed here --
 *    K (max_label_size) is an argument of that call, exactly like the reference's constructor argument. */
int fslic_b200_create_cca(int device, int H, int W, int max_batch, fslic_ctx** out);

/* == BaseContext::initialize_clusters (context.cpp:43-97), for `batch` images [B,H,W,3] u8. */
int fslic_b200_initialize_clusters(fslic_ctx* ctx, const uint8_t* d_images, fslic_cluster* d_clusters, int batch,
                                   void* stream);

/* == BaseContext::iterate (context.cpp:109-197): Lab LUT -> max_iter x (assign + update on a
 *    row subsample) -> full assign -> connectivity enforcement.  d_images [B,H,W,3] u8,
 *    d_clusters [B,K] (read and updated in place), d_labels [B,H,W] u16 (0xFFFF = unassigned). */
int fslic_b200_iterate(fslic_ctx* ctx, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                       int batch, const fslic_params* params, void* stream);

/* == the public field BaseContext::manhattan_spatial_dist (context.h:35; cfast_slic.pyx:186,246): on (1, the default)
 *    the spatial term is coef * (|di| + |dj|), off (0) it is coef * hypot(di, dj) (context.cpp:23-40), and the "noq"
 *    float variant sums squares instead of absolute values (context.cpp:462-496).  The window stays (2S+1)^2 and the
 *    "l2" variant ignores it, as in the reference.  Every iterate entry point reads the setting when it enqueues work. */
int fslic_b200_set_manhattan_spatial_dist(fslic_ctx* ctx, int on);

/* == the float-distance contexts ContextRealDist / ContextRealDistL2 / ContextRealDistNoQ (context.h:100-125,
 *    context.cpp:394-499; selected in cfast_slic.pyx:198-252 by SlicModel.real_dist_type): `variant` 0 = "standard"
 *    (the default kernel with float distances and an untruncated float spatial term), 1 = "l2" (squared colour and
 *    spatial distances), 2 = "noq" (float centroids, no quantisation in the update; absolute or, with
 *    fslic_b200_set_manhattan_spatial_dist(ctx, 0), squared differences).  Same buffers and semantics as fslic_b200_iterate; results bit-identical to the reference
 *    (every float operation in its order and rounding). */
int fslic_b200_iterate_real(fslic_ctx* ctx, int variant, const uint8_t* d_images, fslic_cluster* d_clusters,
                            uint16_t* d_labels, int batch, const fslic_params* params, void* stream);

/* == BaseContext::iterate with `preemptive = true` (context.h:32-33, preemptive.h; cfast_slic.pyx:183-184): clusters that
 *    stop moving (L1 movement below max(round(2 S preemptive_thres), 1) pixels in two updates in a row) and have no
 *    moving cluster within 2S stop being assigned and updated; `is_updatable` of the returned records holds the
 *    countdown where it got to.  Same buffers as fslic_b200_iterate; bit-identical to the reference.  S >= 1. */
int fslic_b200_iterate_preemptive(fslic_ctx* ctx, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                                  int batch, const fslic_params* params, float preemptive_thres, void* stream);

/* == the reference's ContextLSC (src/lsc.cpp, lsc.h: linear spectral clustering; cfast_slic.pyx:207-214, arch
 *    "standard") run with num_threads = 1 -- the only thread count at which the reference's result is defined: its
 *    after_update merges per-thread partial sums in arrival order.  Ten per-pixel features (L, a, b and x, y mapped
 *    onto quarter circles), weighted by their means; assign by the squared 10-D distance over the (2S+1)^2 window;
 *    integer Cluster update as fslic_b200_iterate, plus weighted 10-D centroid features.  Same buffers and
 *    semantics as fslic_b200_iterate; labels, pre-CCA labels and Cluster records bit-identical to the reference.
 *    manhattan_spatial_dist has no effect.  The first call allocates about 44 bytes per pixel of max_batch images. */
int fslic_b200_iterate_lsc(fslic_ctx* ctx, const uint8_t* d_images, fslic_cluster* d_clusters, uint16_t* d_labels,
                           int batch, const fslic_params* params, void* stream);

/* Stage probes of the last fslic_b200_iterate_lsc (before_iteration, lsc.cpp:22-195), into caller device buffers (any
 * may be NULL): the feature means float[B][10], the pixel weights float[B][H][W] and the initial centroid features
 * float[B][K][10]. */
int fslic_b200_debug_lsc_stages(fslic_ctx* ctx, float* d_means_out, float* d_weights_out, float* d_cinit_out, int batch,
                                void* stream);

/* The same call as the reference-facing plugin makes it: HOST buffers in, HOST buffers out
 * (what SlicModel.iterate does with a numpy image, cfast_slic.pyx:150-260).  H2D copy, kernels and
 * D2H copy are pipelined over chunks of 32 images on three streams (pass pinned buffers for true overlap);
 * returns when the results are in the host buffers. */
int fslic_b200_iterate_host(fslic_ctx* ctx, const uint8_t* h_images, fslic_cluster* h_clusters, uint16_t* h_labels,
                            int batch, const fslic_params* params);
int fslic_b200_initialize_clusters_host(fslic_ctx* ctx, const uint8_t* h_images, fslic_cluster* h_clusters,
                                        int batch);

/* Streaming form of fslic_b200_iterate_host (no counterpart in the reference, whose iterate() blocks): enqueue
 * the same H2D -> kernels -> D2H work and return at once; fslic_b200_wait() blocks until the labels and clusters
 * are in the host buffers.  The host buffers must be pinned and stay untouched until then.  One batch per
 * context may be in flight (a second _async call waits for the first); a caller that alternates between two
 * contexts overlaps one batch's PCIe copies with the other's kernels. */
int fslic_b200_iterate_host_async(fslic_ctx* ctx, const uint8_t* h_images, fslic_cluster* h_clusters,
                                  uint16_t* h_labels, int batch, const fslic_params* params);
int fslic_b200_wait(fslic_ctx* ctx);

/* == debug_mode (context.h:36; the Recorder of recorder.h, pushed at context.cpp:157,173).  With tracing on, every
 *    image of a fslic_b200_iterate, fslic_b200_iterate_real, fslic_b200_iterate_preemptive or fslic_b200_iterate_lsc
 *    call records T = max_iter + 1 snapshots: s = 0 after seeding (the reference's iteration -1), s = i + 1 after
 *    update i.  Each holds the pre-CCA assignment u16[H*W], the per-pixel minimum distance min_dists[H*W] (u16 for the
 *    default contexts and `preemptive`, float for the float-distance ones and LSC) and the K cluster records.  Labels
 *    and clusters are those of the untraced call; a traced call takes plain launches (no graph replay, no fused
 *    prepare) and a trace kernel per pass that also checks the pass's labels.  Snapshots go to device buffers grown on
 *    demand (T * B * (H*W*(2 + 2 or 4) + K*32) bytes; FSLIC_ENOMEM when they cannot be had).  While tracing is on the
 *    host entry points return FSLIC_EINVAL. */
int fslic_b200_set_trace(fslic_ctx* ctx, int on);
/* CUDA graphs fslic_b200_iterate captured and replays it launched on this context so far (diagnostics). */
int fslic_b200_debug_graph_counts(const fslic_ctx* ctx, int* captures, int* replays);
/* What the last traced call recorded: snapshots T (0: none), batch B, bytes per min_dists entry (2 or 4). */
int fslic_b200_trace_info(const fslic_ctx* ctx, int* snapshots, int* batch, int* dist_bytes);
/* Synchronises the device and copies image `image`'s snapshots to host arrays (any may be NULL): h_assignment
 * u16[T][H*W], h_min_dists [T][H*W] of the recorded type, h_clusters [T][K].  *h_mismatches gets the number of pixels
 * whose label an assign kernel set differently from the trace kernel's argmin over the whole traced call; a nonzero
 * count also returns FSLIC_ECHECK. */
int fslic_b200_trace_snapshots(fslic_ctx* ctx, int image, uint16_t* h_assignment, void* h_min_dists,
                               fslic_cluster* h_clusters, uint32_t* h_mismatches);
/* Host only (no CUDA call): the text of Recorder::get_report (recorder.h:18-47, 90-98) for `snapshots` snapshots laid
 * out like fslic_b200_trace_snapshots' arrays (iterations -1, 0, 1, ...; min_dists float when dist_is_float, else u16).
 * *out gets a malloc'd NUL-terminated buffer of *len bytes, to be released with fslic_b200_free_report. */
int fslic_b200_format_report(int H, int W, int K, int snapshots, int dist_is_float, const uint16_t* assignment,
                             const void* min_dists, const fslic_cluster* clusters, char** out, size_t* len);
void fslic_b200_free_report(char* report);

/* == cca::ConnectivityEnforcer(labels,H,W,K,min_threshold).execute(labels) (cca.cpp:178-265),
 *    in place on d_labels [B,H,W] u16.  H, W come from the context; K (= max label + 1 in
 *    cfast_slic.pyx:377-382) is given by the caller. */
int fslic_b200_enforce_connectivity(fslic_ctx* ctx, uint16_t* d_labels, int batch, int K, int min_threshold,
                                    void* stream);

/* == fast_slic_get_connectivity (src/fast-slic.cpp:16-78; cfast_slic.pyx:262-270): the superpixel adjacency graph of
 *    one label map d_labels u16[H*W] -> d_counts int32[K], d_neighbors u32[K*12] (row k: the first d_counts[k] entries,
 *    in the order the reference's raster scan links them; at most 12 per label, like the reference).  Stateless:
 *    d_scratch must hold fslic_b200_connectivity_scratch_bytes(K) bytes (= fslic_b200_connectivity_batch_scratch_bytes(K,
 *    1)).  Asynchronous on `stream`. */
size_t fslic_b200_connectivity_scratch_bytes(int K);
int fslic_b200_get_connectivity(int device, int H, int W, int K, const uint16_t* d_labels, int32_t* d_counts,
                                uint32_t* d_neighbors, void* d_scratch, size_t scratch_bytes, void* stream);

/* == fast_slic_get_mask_density / fast_slic_cluster_density_to_mask (src/fast-slic.cpp:141-168; cfast_slic.pyx:283-320).
 *    d_mask u8[H*W], d_densities u8[K]; d_scratch int32[K].  Asynchronous on `stream`. */
int fslic_b200_get_mask_density(int device, int H, int W, int K, const fslic_cluster* d_clusters, const uint16_t* d_labels,
                                const uint8_t* d_mask, uint8_t* d_densities, int32_t* d_scratch, void* stream);
int fslic_b200_cluster_density_to_mask(int device, int H, int W, int K, const uint16_t* d_labels, const uint8_t* d_densities,
                                       uint8_t* d_result, void* stream);

/* The three consumers above over `batch` label maps d_labels u16[B,H,W], each image on its own: every image's result is
 * what the single-image call gives for it.  Asynchronous on `stream` and never synchronise, so a CUDA graph can capture
 * them; batch == 0 does nothing.
 * Connectivity: d_counts int32[B,K], d_neighbors u32[B,K,12] (zero past the count); d_replayed int32[B] (or NULL)
 * receives 1 for an image whose pair table overflowed and took the exact single-thread replay of the reference's loop,
 * else 0.  d_scratch holds fslic_b200_connectivity_batch_scratch_bytes(K, batch) bytes: 24 * B * T for the pair tables
 * (T = the table size of fslic_b200_connectivity_scratch_bytes, a power of two >= max(4096, 32 * K)), plus the radix
 * sort's temporary storage for B * T pairs, plus 4 * B; 256 for K <= 0 or B <= 0; (size_t)-1 for K > 65535 or when
 * B * T exceeds 2^31 - 1 (split the batch). */
size_t fslic_b200_connectivity_batch_scratch_bytes(int K, int batch);
int fslic_b200_get_connectivity_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                      int32_t* d_counts, uint32_t* d_neighbors, int32_t* d_replayed, void* d_scratch,
                                      size_t scratch_bytes, void* stream);
/* d_clusters [B,K], d_masks u8[B,H,W], d_densities u8[B,K]; d_scratch int32[B,K]. */
int fslic_b200_get_mask_density_batch(int device, int batch, int H, int W, int K, const fslic_cluster* d_clusters,
                                      const uint16_t* d_labels, const uint8_t* d_masks, uint8_t* d_densities,
                                      int32_t* d_scratch, void* stream);
/* d_densities u8[B,K] -> d_result u8[B,H,W] (0 where the label is >= K). */
int fslic_b200_cluster_density_to_mask_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                             const uint8_t* d_densities, uint8_t* d_result, void* stream);

/* Superpixel pooling (pool.cuh; no counterpart in the reference) over `batch` label maps d_labels u16[B,H,W]: a label
 * outside [0, K) belongs to no superpixel; 1 <= K <= 65534, C >= 1.  Asynchronous on `stream`, never synchronise, no
 * float atomics: each image's result depends only on its own labels and features (DESIGN.md section 4.12 gives the
 * summation order).  batch, H or W == 0 does nothing.
 * Scratch bytes fslic_b200_pool_batch takes for one call: 16 per pixel, 8 per superpixel and the radix sort's temporary
 * storage; 256 for no pixel; (size_t)-1 for a bad K or when batch * H * W > 2^31 - 1 or batch > 65536 (split the batch). */
size_t fslic_b200_pool_batch_scratch_bytes(int batch, int H, int W, int K);
/* d_features f32[B,C,H,W] -> d_out f32[B,C,K]: the sum over each superpixel's pixels, or with `mean` != 0 the sum divided
 * by the pixel count (0 for an empty superpixel); d_counts int32[B,K]: the pixel counts of the label map. */
int fslic_b200_pool_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                          const float* d_features, int mean, float* d_out, int32_t* d_counts, void* d_scratch,
                          size_t scratch_bytes, void* stream);
/* d_values f32[B,C,K] -> d_out f32[B,C,H,W]: each pixel's superpixel value, divided by (float)d_divisor[b,label] when
 * d_divisor (int32[B,K]) is not NULL; 0 where the label is outside [0, K). */
int fslic_b200_pool_unpool_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                 const float* d_values, const int32_t* d_divisor, float* d_out, void* stream);
/* d_q f32[B,C,K] -> d_out int16[B,H,W]: the first index of the maximum of q over C at each pixel's superpixel (a NaN
 * counts as the maximum), -1 where the label is outside [0, K); C <= 32767.  d_node_class: int32[B,K] scratch. */
int fslic_b200_pool_paint_argmax_batch(int device, int batch, int H, int W, int C, int K, const uint16_t* d_labels,
                                       const float* d_q, int32_t* d_node_class, int16_t* d_out, void* stream);
/* d_table int32[B,K] -> d_out int16[B,H,W]: (int16)d_table[b,label] at each pixel, -1 where the label is outside [0, K). */
int fslic_b200_pool_paint_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels,
                                const int32_t* d_table, int16_t* d_out, void* stream);

/* Region adjacency graphs (rag.cuh; no counterpart in the reference) of `batch` label maps d_labels u16[B,H,W]: node
 * b*K + k is label k of image b; an edge joins two labels of one image for every unordered pair of adjacent pixels
 * (connectivity 4: horizontal and vertical neighbours; 8: also both diagonals) that carry them, and its weight is the
 * number of such pixel pairs.  A label outside [0, K) belongs to no node.  1 <= K <= 65534, H * W <= 2^29.  Two calls
 * per batch, asynchronous on `stream`, never synchronise: the count writes the CSR row offsets and the edge total, the
 * caller reads the total back and allocates the edges, the fill writes them (DESIGN.md section 4.13).
 * Scratch bytes of the count (the fill reads it too): 8 per pair-table slot, 16 per node and the scan's temporary
 * storage.  Each image's table has T slots, a power of two: with `exact`, T >= 2 * min(K (K - 1) / 2, pixel pairs of
 * the image), which cannot overflow; else the smaller of that and max(4096, 32 K), which can.  256 for no pixel;
 * (size_t)-1 for bad arguments, H * W > 2^29, B * K >= 2^31 - 1 or an exact table over 2^31 slots. */
size_t fslic_b200_rag_batch_scratch_bytes(int batch, int H, int W, int K, int connectivity, int exact);
/* d_indptr int64[B*K + 1]: edge_base + the exclusive sum of the node degrees; d_info int64[B + 1]: d_info[b] = 1 where
 * image b's table overflowed (its edges are incomplete: count it again with `exact`), d_info[B] = the directed edge
 * total E of the call. */
int fslic_b200_rag_batch_count(int device, int batch, int H, int W, int K, int connectivity, int exact,
                               const uint16_t* d_labels, long long edge_base, long long* d_indptr, long long* d_info,
                               void* d_scratch, size_t scratch_bytes, void* stream);
/* Scratch bytes of the fill for E edges: 20 per edge and the radix sort's temporary storage; 256 for E = 0;
 * (size_t)-1 for E > 2^31 - 1 (split the batch). */
size_t fslic_b200_rag_fill_scratch_bytes(int batch, int K, long long edges);
/* After a count with the same batch, H, W, K, connectivity, exact and d_scratch, and `edges` = its d_info[B]:
 * d_src / d_dst int64[E] (node ids + node_base) and d_boundary int32[E], both directions of every edge, rows in
 * source order, each row sorted by target. */
int fslic_b200_rag_batch_fill(int device, int batch, int H, int W, int K, int connectivity, int exact,
                              long long node_base, long long edges, const void* d_scratch, size_t scratch_bytes,
                              void* d_fill_scratch, size_t fill_bytes, long long* d_src, long long* d_dst,
                              int32_t* d_boundary, void* stream);
/* Region adjacency graphs of `batch` label volumes d_labels u16[B,D,H,W] (DESIGN.md section 4.23): the same graph,
 * tables, calls and outputs as above, with voxel pairs for pixel pairs.  Voxel pairs are the forward half of the
 * 3x3x3 neighbourhood (offsets (dz, dy, dx) whose first non-zero component is positive) with at most 1 (connectivity
 * 6), 2 (18) or 3 (26) non-zero components: 3, 9 or 13 per voxel.  D * H * W <= 2^29, and the volume's pair count
 * P = sum over those offsets of (D - |dz|)(H - |dy|)(W - |dx|) must be at most 2^31 - 1, so that every boundary count
 * fits int32.  Scratch bytes as fslic_b200_rag_batch_scratch_bytes with P for the pixel pairs; (size_t)-1 for bad
 * arguments, D * H * W > 2^29, P > 2^31 - 1, B * K >= 2^31 - 1 or an exact table over 2^31 slots.  The fill takes its
 * scratch from fslic_b200_rag_fill_scratch_bytes. */
size_t fslic_b200_rag3d_batch_scratch_bytes(int batch, int D, int H, int W, int K, int connectivity, int exact);
int fslic_b200_rag3d_batch_count(int device, int batch, int D, int H, int W, int K, int connectivity, int exact,
                                 const uint16_t* d_labels, long long edge_base, long long* d_indptr, long long* d_info,
                                 void* d_scratch, size_t scratch_bytes, void* stream);
int fslic_b200_rag3d_batch_fill(int device, int batch, int D, int H, int W, int K, int connectivity, int exact,
                                long long node_base, long long edges, const void* d_scratch, size_t scratch_bytes,
                                void* d_fill_scratch, size_t fill_bytes, long long* d_src, long long* d_dst,
                                int32_t* d_boundary, void* stream);

/* Superpixels scored against ground truth (groundtruth.cuh; no counterpart in the reference) over `batch` label maps
 * d_labels u16[B,H,W] and maps of the same shape whose element type is `dtype`, one of the FSLIC_GT_* codes (the element
 * size in bytes).  A label outside [0, K) belongs to no superpixel; 1 <= K <= 65534, H * W <= 2^29.  Integer only,
 * asynchronous on `stream`, never synchronise (a CUDA graph can capture them); batch, H or W == 0 launches nothing.
 * DESIGN.md section 4.14 gives the definitions. */
#define FSLIC_GT_UINT8 1
#define FSLIC_GT_INT16 2
#define FSLIC_GT_INT32 4
#define FSLIC_GT_INT64 8
/* d_out int32[B,K,C] (C = num_classes, 1..65536): the number of pixels of image b with label k and class c; pixels with
 * a label outside [0, K) or a class outside [0, C) are not counted. */
int fslic_b200_gt_histogram_batch(int device, int batch, int H, int W, int K, int num_classes, int dtype,
                                  const void* d_classes, const uint16_t* d_labels, int32_t* d_out, void* stream);
/* Scratch bytes of one fslic_b200_gt_scores_batch call: 20 per pixel for the overlap keys and runs, 3/8 per pixel for
 * the boundary bitmaps, 16 per (image, label) and the larger temporary storage of the radix sort and the run-length
 * encoding; 256 for no pixel; (size_t)-1 for bad arguments or when batch * H * W > 2^31 - 1 or batch > 2^17 (split the
 * batch). */
size_t fslic_b200_gt_scores_scratch_bytes(int batch, int H, int W, int K);
/* d_out int64[B,7] per image: counted pixels, the ASA numerator sum_k max_g n_kg, the UE numerator
 * sum_{k,g: n_kg > 0} min(n_kg, n_k - n_kg), gt boundary pixels, those with a superpixel boundary pixel within the
 * Chebyshev `tolerance` (0..32), superpixel boundary pixels valid in gt, those with a gt boundary pixel within it.  A gt
 * value is valid in [0, 2^31 - 1] and, with has_ignore, != ignore. */
int fslic_b200_gt_scores_batch(int device, int batch, int H, int W, int K, int tolerance, int dtype, const void* d_gt,
                               const uint16_t* d_labels, int has_ignore, long long ignore, long long* d_out,
                               void* d_scratch, size_t scratch_bytes, void* stream);
/* d_out u8[B,H,W]: 1 where the right or lower neighbour exists and carries another label, else 0. */
int fslic_b200_gt_boundaries_batch(int device, int batch, int H, int W, const uint16_t* d_labels, uint8_t* d_out,
                                   void* stream);
/* The same over `batch` label volumes d_labels u16[B,D,H,W] and gt of that shape (DESIGN.md section 4.24);
 * D * H * W <= 2^29.  The overlap fields are those of the [B, D*H, W] view.  A boundary voxel has a +x, +y or +z
 * neighbour with another value (valid, for gt), and the window is the box |dz| <= rz, |dy| <= ry, |dx| <= rx (each
 * 0..32) clipped to the volume.  Scratch bytes: as fslic_b200_gt_scores_scratch_bytes with H = D * H and two more
 * bitmaps (5/8 byte per voxel in all); (size_t)-1 for bad arguments or when batch * D * H * W > 2^31 - 1 or
 * batch > 2^17. */
size_t fslic_b200_gt_scores3d_scratch_bytes(int batch, int D, int H, int W, int K);
int fslic_b200_gt_scores3d_batch(int device, int batch, int D, int H, int W, int K, int rz, int ry, int rx, int dtype,
                                 const void* d_gt, const uint16_t* d_labels, int has_ignore, long long ignore,
                                 long long* d_out, void* d_scratch, size_t scratch_bytes, void* stream);
/* d_out u8[B,D,H,W]: 1 where the +x, +y or +z neighbour exists and carries another label, else 0. */
int fslic_b200_gt_boundaries3d_batch(int device, int batch, int D, int H, int W, const uint16_t* d_labels,
                                     uint8_t* d_out, void* stream);

/* Superpixel shapes (props.cuh; no counterpart in the reference) of `batch` label maps d_labels u16[B,H,W]; node
 * n = b*K + k is label k of image b, pixel (row y, column x) has coordinates (y, x).  A label outside [0, K) belongs to
 * no superpixel.  1 <= K <= 65534, H, W <= 65535, H * W <= 2^29.  Outputs, all device memory:
 *   d_area int32[B*K]         pixels labelled k;
 *   d_bbox int32[B*K][4]      (y0, x0, y1, x1): min inclusive, max exclusive; all 0 for an empty node;
 *   d_moments int64[B*K][5]   (sum y, sum x, sum y^2, sum xy, sum x^2) over k's pixels, exact;
 *   d_perimeter int32[B*K]    sides of k's pixels whose 4-neighbour across that side is outside the image or has another
 *                             raw label;
 *   d_border int32[B*K]       those of the sides that lie on the image edge;
 *   d_centroid f64[B*K][2]    (sum y / n, sum x / n);
 *   d_covariance f64[B*K][3]  (sum y^2 / n - cy cy, sum xy / n - cy cx, sum x^2 / n - cx cx);
 * each float64 step one correctly rounded operation, 0.0 for an empty node.  Integer arithmetic up to that, so the result
 * of image b depends on d_labels[b] only.  No scratch; asynchronous on `stream`, never synchronises (a CUDA graph can
 * capture it); batch == 0 does nothing, H or W == 0 zeroes the outputs. */
int fslic_b200_props_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels, int32_t* d_area,
                           int32_t* d_bbox, long long* d_moments, int32_t* d_perimeter, int32_t* d_border,
                           double* d_centroid, double* d_covariance, void* stream);
/* Supervoxel shapes (props3d.cuh; DESIGN.md section 4.23) of `batch` label volumes d_labels u16[B,D,H,W]; node
 * n = b*K + k, voxel (slice z, row y, column x) has coordinates (z, y, x).  A label outside [0, K) belongs to no
 * supervoxel.  1 <= K <= 65534, D, H, W <= 32767, D * H * W <= 2^29.  Outputs, all device memory:
 *   d_area int32[B*K]         voxels labelled k;
 *   d_bbox int32[B*K][6]      (z0, y0, x0, z1, y1, x1): min inclusive, max exclusive; all 0 for an empty node;
 *   d_moments int64[B*K][9]   (sum z, y, x, z^2, zy, zx, y^2, yx, x^2) over k's voxels, exact;
 *   d_surface int64[B*K]      faces of k's voxels whose 6-neighbour across that face is outside the volume or has
 *                             another raw label;
 *   d_border int32[B*K]       those of the faces that lie on the volume's edge;
 *   d_centroid f64[B*K][3]    (sum z / n, sum y / n, sum x / n);
 *   d_covariance f64[B*K][6]  (zz, zy, zx, yy, yx, xx), each sum ab / n - c_a c_b;
 * each float64 step one correctly rounded operation, 0.0 for an empty node.  No scratch; asynchronous on `stream`, never
 * synchronises (a CUDA graph can capture it); batch == 0 does nothing, D, H or W == 0 zeroes the outputs. */
int fslic_b200_props3d_batch(int device, int batch, int D, int H, int W, int K, const uint16_t* d_labels,
                             int32_t* d_area, int32_t* d_bbox, long long* d_moments, long long* d_surface,
                             int32_t* d_border, double* d_centroid, double* d_covariance, void* stream);

/* Superpixels merged into regions (merge.cuh; no counterpart in the reference): single-linkage cuts of a region
 * adjacency graph over `batch` label maps d_labels u16[B,H,W].  Node n = b*K + k is label k of image b, present when a
 * pixel of image b carries k.  1 <= K <= 65534, B * K <= 2^30.
 * Edges: d_src / d_dst int64[E] and d_weight f32[E].  Only entries with src < dst are read, and the weight of the
 * undirected edge {src, dst} is the weight of that entry.  An entry is ignored when an endpoint is outside [0, B*K),
 * the endpoints lie in different images, an endpoint is not present or the weight is NaN.
 * Order: edges by (weight, lower local id, higher local id), -0.0 equal to +0.0; single linkage is Kruskal over it.
 *   FSLIC_MERGE_THRESHOLD: two nodes share a region exactly when a path of edges with (double)weight < threshold joins
 *     them (threshold not NaN).
 *   FSLIC_MERGE_NUM_REGIONS: Kruskal stops after P_b - num_regions merges or when it runs out of edges (P_b: the present
 *     nodes of image b; num_regions >= 1), leaving max(num_regions, c_b) regions where c_b is the number of connected
 *     components among present nodes over non-NaN edges.
 * Outputs: d_region int32[B,K], the region of node b*K + k, regions of an image numbered 0, 1, ... in ascending order of
 * their smallest member, -1 for a node that is not present; d_num_regions int32[B]; d_out int16[B,H,W], the region of
 * each pixel's label (fslic_b200_pool_paint_batch of d_region), -1 where the label is outside [0, K).
 * Integer arithmetic once each weight is a key, so the result of image b depends on its labels and edges only.
 * Asynchronous on `stream`, never synchronises and reads nothing back (a CUDA graph can capture it); batch == 0 does
 * nothing.  DESIGN.md section 4.16 describes the kernels.
 * Scratch bytes: 40 per node, 16 per image, the Boruvka round flags and the larger temporary storage of the segmented
 * radix sort and the scan, each piece aligned to 256; (size_t)-1 for a bad K or B * K > 2^30. */
#define FSLIC_MERGE_THRESHOLD 0
#define FSLIC_MERGE_NUM_REGIONS 1
size_t fslic_b200_merge_scratch_bytes(int batch, int K);
int fslic_b200_merge_batch(int device, int batch, int H, int W, int K, const uint16_t* d_labels, long long edges,
                           const long long* d_src, const long long* d_dst, const float* d_weight, int mode,
                           double threshold, int num_regions, int32_t* d_region, int32_t* d_num_regions,
                           int16_t* d_out, void* d_scratch, size_t scratch_bytes, void* stream);

/* Boundary statistics of region adjacency edges (boundary.cuh; no counterpart in the reference) over `batch` label
 * maps d_labels u16[B,H,W] and value maps d_values f32[B,C,H,W].  The pixel pairs are region adjacency's: the right and
 * down neighbour, with connectivity 8 also the down-right and down-left one; a pair is a boundary pair when both labels
 * are in [0, K) and differ.  1 <= K <= 65534, H * W <= 2^29.  Two calls per chunk of images, asynchronous on `stream`,
 * never synchronise: the select writes the number of boundary pairs, the caller reads it back and sizes the stats'
 * scratch from it, the stats write every graph entry of the chunk's images (DESIGN.md section 4.17).
 * Scratch bytes of the select (the stats read it too): 4 per pixel pair (2 or 4 per pixel) and the selection's
 * temporary storage; 256 for no pixel; (size_t)-1 for bad arguments, H * W > 2^29 or more than 2^31 - 1 pixel pairs
 * (split the batch). */
size_t fslic_b200_boundary_select_scratch_bytes(int batch, int H, int W, int K, int connectivity);
/* d_pairs int32[1]: the number of boundary pairs of the call. */
int fslic_b200_boundary_select_batch(int device, int batch, int H, int W, int K, int connectivity,
                                     const uint16_t* d_labels, int32_t* d_pairs, void* d_scratch, size_t scratch_bytes,
                                     void* stream);
/* Scratch bytes of the stats for `pairs` boundary pairs and `edges` graph entries: 25 per pair, 24 per entry and the
 * largest temporary storage of the radix sorts and the selection; (size_t)-1 for a negative count or one above
 * 2^31 - 1. */
size_t fslic_b200_boundary_stats_scratch_bytes(long long pairs, long long edges);
/* After a select with the same batch, H, W, K, connectivity, d_labels and d_select_scratch, and `pairs` = its
 * d_pairs.  The call's images are images [image_base, image_base + batch) of a graph of `nodes` = B_total * K nodes
 * whose entries are d_src / d_dst int64[E].  Entry e = (u, v) belongs to image b when u // K == v // K == b, both are
 * in [0, nodes) and u != v; its pairs are image b's boundary pairs whose labels are {u % K, v % K}.  For each entry of
 * the call's images: d_count int32[E] = the number n of its pairs, and per channel c d_mean / d_min / d_max f32[E,C]
 * = the mean, min and max of the 2n values of its pairs in ordinal order (anchor, then the other pixel), the sum in
 * pool's order divided by (float)(2n), min / max under -0.0 < +0.0 and NaN when any value is NaN; NaN and 0 for an
 * entry with no pairs.  With `first` != 0 every row is first set to NaN and 0, so that entries of no image are
 * defined: give it to the first call of a batch. */
int fslic_b200_boundary_stats_batch(int device, int batch, int H, int W, int K, int C, int connectivity,
                                    const uint16_t* d_labels, const float* d_values, long long pairs,
                                    const void* d_select_scratch, size_t select_bytes, long long image_base,
                                    long long nodes, long long edges, const long long* d_src, const long long* d_dst,
                                    int first, float* d_mean, float* d_min, float* d_max, int32_t* d_count,
                                    void* d_scratch, size_t scratch_bytes, void* stream);
/* The same over `batch` label volumes d_labels u16[B,D,H,W] and values d_values f32[B,C,D,H,W] (DESIGN.md section
 * 4.24), with region_adjacency_3d's voxel pairs: each voxel (the anchor) with its forward neighbours (dz, dy, dx) of
 * RAG3D_OFFSETS, the first 3 (connectivity 6), 9 (18) or 13 (26); the pair's ordinal is anchor * Ndir + d.  A volume
 * has D * H * W <= 2^29 and at most 2^31 - 1 voxel pairs, a call at most 2^31 - 1 voxels.
 * Scratch bytes of the select (the stats read it too): 6 per voxel and the larger temporary storage of the selection
 * and the pair sum; 256 for no voxel; (size_t)-1 for bad arguments or volumes or calls over those limits. */
size_t fslic_b200_boundary3d_select_scratch_bytes(int batch, int D, int H, int W, int K, int connectivity);
/* d_counts int64[2]: the number of voxels with a boundary pair and the number of boundary pairs of the call. */
int fslic_b200_boundary3d_select_batch(int device, int batch, int D, int H, int W, int K, int connectivity,
                                       const uint16_t* d_labels, long long* d_counts, void* d_scratch,
                                       size_t scratch_bytes, void* stream);
/* Scratch bytes of the stats for `voxels` boundary voxels, `pairs` boundary pairs and `edges` graph entries: 4 per
 * voxel, 34 per pair, 24 per entry and the largest temporary storage of the scan, the radix sorts and the selection;
 * (size_t)-1 for a negative count, one above 2^31 - 1, or voxels > pairs > 13 * voxels. */
size_t fslic_b200_boundary3d_stats_scratch_bytes(long long voxels, long long pairs, long long edges);
/* After a select with the same batch, D, H, W, K, connectivity, d_labels and d_select_scratch, and `voxels` / `pairs`
 * = its d_counts: the outputs of fslic_b200_boundary_stats_batch, with voxel pairs for pixel pairs. */
int fslic_b200_boundary3d_stats_batch(int device, int batch, int D, int H, int W, int K, int C, int connectivity,
                                      const uint16_t* d_labels, const float* d_values, long long voxels,
                                      long long pairs, const void* d_select_scratch, size_t select_bytes,
                                      long long image_base, long long nodes, long long edges, const long long* d_src,
                                      const long long* d_dst, int first, float* d_mean, float* d_min, float* d_max,
                                      int32_t* d_count, void* d_scratch, size_t scratch_bytes, void* stream);

/* k-nearest-neighbour graphs over feature points (knn.cuh; the reference's get_knn_connectivity has no defined result)
 * of `batch` images of K points each, d_points f32[B,K,D], node n = b * K + i.  A node is a candidate when
 * d_present u8[B,K] (NULL: every node) is nonzero and its D coordinates are finite.  s(i, j) = ((+0 + t_0 * t_0) +
 * t_1 * t_1) + ..., t_c = p_i[c] - p_j[c], every float32 operation rounded on its own.  Node i's neighbours are the first
 * min(k, P_b - 1) other candidates of its image under the order of (s, j), P_b the image's candidates; with `symmetric`
 * the edges are those and their reverses, each (source, target) once.  1 <= K <= 65534, 1 <= D <= 64,
 * 1 <= k <= 32, B * K <= 2^30 and 2 * B * K * k <= 2^31 - 1 per call.  Two calls per chunk of images, asynchronous on
 * `stream`, never synchronise: the count writes the chunk's row offsets and its edge total, the caller reads the total
 * back and sizes the outputs, the fill writes the edges (DESIGN.md section 4.18).  Both take the same scratch.
 * Scratch bytes: per node 17 + 4 * DP + 8 * k (DP: D padded to a power of two >= 4), with `symmetric` 72 * k more, and
 * the temporary storage of the selection, scan, radix sort and deduplication; (size_t)-1 for arguments out of range. */
size_t fslic_b200_knn_scratch_bytes(int batch, int K, int D, int k, int symmetric);
/* d_indptr int64[B*K + 1] = edge_base + the offset of each of the call's rows, the last = edge_base + the total;
 * d_total int64[1] = the call's edge total. */
int fslic_b200_knn_count(int device, int batch, int K, int D, int k, int symmetric, const float* d_points,
                         const uint8_t* d_present, long long edge_base, long long* d_indptr, long long* d_total,
                         void* d_scratch, size_t scratch_bytes, void* stream);
/* After a count with the same batch, K, D, k, symmetric and scratch, and `edges` = its total: d_src / d_dst
 * int64[edges] (node ids + node_base) sorted by source then target, and d_distance f32[edges] = s. */
int fslic_b200_knn_fill(int device, int batch, int K, int D, int k, int symmetric, long long node_base, long long edges,
                        const void* d_scratch, size_t scratch_bytes, long long* d_src, long long* d_dst,
                        float* d_distance, void* stream);

/* SLIC over float feature maps (feature_slic.cuh; no counterpart in the reference) of `batch` images d_features
 * f32[B,C,H,W].  S = (int)(int16_t)sqrt((double)(H * W / K)); seeds on initialize_clusters' grid with the features of
 * their pixel, or d_init_position f32[B,K,2] (y, x) clamped into the image and d_init_features f32[B,K,C] as given (both
 * or neither).  Pass t < max_iter assigns the rows i with i % stride == t % stride, then updates; one full assign
 * follows.  Candidates of pixel (i, j): |i - (int)cy| <= S and |j - (int)cx| <= S; distance d = fc + w2 * (ty*ty +
 * tx*tx), fc = (((+0 + t_0*t_0) + t_1*t_1) + ..), t_c = f_c - mu_c, ty = i - cy, tx = j - cx, w2 = (compactness / S)^2,
 * every float32 operation rounded on its own; the winner is the smallest (bits(d) << 32 | k), a NaN distance having
 * the bits 0x7fffffff; a pixel without a candidate keeps its label (initially 0xffff).  Update over the pass rows: n
 * members, cy = (float)((double)sum_i / n), cx likewise, mu = pool's mean (fslic_b200_pool_batch's summation order); a
 * cluster with n = 0 keeps its centre and features.  Outputs: d_labels u16[B,H,W] before connectivity enforcement,
 * d_position f32[B,K,2], d_centroids f32[B,K,C], d_count i32[B,K] (n of the last update, 0 when max_iter = 0), and,
 * unless NULL, d_overflow i32[max_iter + 1]: the tiles of each pass that overflowed to the per-pixel assign kernel.
 * 1 <= C <= 1024, 1 <= K <= min(65534, H * W), H, W <= 32767, H * W <= 2^29, B * K <= 2^30, 1 <= stride <= 255,
 * max_iter >= 0, compactness finite and > 0; B * H * W <= 2^31 - 1 and B <= 65535 per call.  Asynchronous on `stream`,
 * never synchronises (DESIGN.md section 4.19).  Scratch bytes: (size_t)-1 for arguments out of range. */
size_t fslic_b200_feature_slic_scratch_bytes(int batch, int H, int W, int C, int K, int stride, int max_iter);
int fslic_b200_feature_slic(int device, int batch, int H, int W, int C, int K, float compactness, int stride,
                            int max_iter, const float* d_features, const float* d_init_position,
                            const float* d_init_features, uint16_t* d_labels, float* d_position, float* d_centroids,
                            int32_t* d_count, int32_t* d_overflow, void* d_scratch, size_t scratch_bytes, void* stream);

/* Differentiable soft SLIC (soft_slic.cuh; no counterpart in the reference; DESIGN.md section 4.20) over a grid of nh x
 * nw cells, K = nh * nw: pixel (i, j) is in cell (i*nh / H, j*nw / W), and its 9 slots n = (da+1)*3 + (db+1) are the
 * cells (a+da, b+db), invalid outside the grid (value +0.0, in no sum).  Per-pixel maps f32[B,C,H,W], associations and
 * their gradients f32[B,9,H,W], per-cell maps f32[B,C,K], weights Z f32[B,K].  Every float32 operation is rounded on its
 * own in a fixed order: sums over slots in n order, over channels in c order, over a cell's block (the pixels with the
 * cell in a valid slot, a rectangle) in pool's lane order, all from +0.0.  1 <= nh <= H, 1 <= nw <= W, K <= 65534,
 * H * W <= 2^29, B * K <= 2^30, C >= 1.  Asynchronous on `stream`, never synchronise; batch 0 does nothing.
 *   soft_assign: q_n = e_n / sum e, e_n = expf(m - d_n) (glibc's), d_n = sum_c (f_c - mu_{k(n)c})^2, m = fminf of d
 *   soft_assign_backward (d_gd: a f32[B,9,H,W] temporary; either gradient may be NULL): gd_n = q_n * (t - g_n),
 *     t = sum_n q_n g_n; gF_c = 2 * sum_n gd_n (f_c - mu_{k(n)c}); gmu_kc = -2 * block sum of gd (f_c - mu_kc)
 *   soft_pool: A = block sum of q v, Z = block sum of q, M = A / Z where Z != 0, else 0
 *   soft_pool_backward (d_grad_sums f32[B,C,K] and d_grad_weights f32[B,K] temporaries; the last two outputs may be
 *     NULL): gA = gM / Z, gZ = -sum_c gA M (both 0 where Z == 0); gV_c = sum_n q_n gA_{k(n)c};
 *     gQ_n = sum_c gA_{k(n)c} v_c + gZ_{k(n)}
 *   soft_unpool: out_c = sum_n q_n M_{k(n)c}
 *   soft_unpool_backward (either output may be NULL): gM = block sum of q g; gQ_n = sum_c g_c M_{k(n)c}
 *   soft_labels: the cell of each pixel's first largest q over its valid slots, a NaN counting as the maximum */
int fslic_b200_soft_assign(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_features,
                           const float* d_centroids, float* d_assoc, void* stream);
int fslic_b200_soft_assign_backward(int device, int batch, int H, int W, int C, int nh, int nw,
                                    const float* d_features, const float* d_centroids, const float* d_assoc,
                                    const float* d_grad_assoc, float* d_gd, float* d_grad_features,
                                    float* d_grad_centroids, void* stream);
int fslic_b200_soft_pool(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_values,
                         const float* d_assoc, float* d_means, float* d_weights, void* stream);
int fslic_b200_soft_pool_backward(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_values,
                                  const float* d_assoc, const float* d_means, const float* d_weights,
                                  const float* d_grad_means, float* d_grad_sums, float* d_grad_weights,
                                  float* d_grad_values, float* d_grad_assoc, void* stream);
int fslic_b200_soft_unpool(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_values,
                           const float* d_assoc, float* d_out, void* stream);
int fslic_b200_soft_unpool_backward(int device, int batch, int H, int W, int C, int nh, int nw, const float* d_values,
                                    const float* d_assoc, const float* d_grad_out, float* d_grad_values,
                                    float* d_grad_assoc, void* stream);
int fslic_b200_soft_labels(int device, int batch, int H, int W, int nh, int nw, const float* d_assoc,
                           uint16_t* d_labels, void* stream);

/* Message passing over superpixel graphs (message_passing.cuh; no counterpart in the reference; DESIGN.md section
 * 4.21).  A graph is d_indptr int64 [N+1] (CSR offsets) and d_targets int64 [E] (edge_index[1]): the row of entry e is
 * the node n with indptr[n] <= e < indptr[n+1], its target t_e = targets[e].  An entry with t_e outside [0, N) is no
 * edge: it takes part in nothing and receives no gradient.  Every float operation is separately rounded, in a fixed
 * order: row sums over a node's entries in increasing e, column sums over a node's in-entries (the entries targeting
 * it) in increasing e, both from +0.0; no float atomics.  0 <= N, E <= 2^31 - 1, C >= 1, H >= 1 divides C.  Node maps
 * [N,C], entry maps [E,C], weights and scores [E,H]; head h owns channels [h*C/H, (h+1)*C/H).  Asynchronous on
 * `stream`, never synchronise.
 *   mp_gather (end 0: target, 1: source): out[e] = x[t_e] or x[row(e)], +0.0 for no edge
 *   mp_gather_backward: end 1: grad_x[n] = row sum of g[e]; end 0: column sum of g[e] (d_scratch as its
 *     *_scratch_bytes says; unused for end 1)
 *   mp_softmax: per row and head, m = the maximum (NaN wins; -0.0 < +0.0), y_e = expf(s_e - m) (glibc's), Z = row sum
 *     of y, out_e = y_e / Z
 *   mp_softmax_backward: dot = row sum of out_e * g_e; grad_e = out_e * (g_e - dot)
 *   mp_aggregate (reduce 0: sum, 1: mean, 2: max; d_weight [E,H] or NULL): term w[e,h] * x[t_e,c] (x[t_e,c] without a
 *     weight); sum: the row sum; mean: sum / (float)deg, d_deg int32 [N] receives deg; max: the first maximal term
 *     (NaN wins; -0.0 < +0.0), d_amax int32 [N,C] receives its entry (-1 for none); an empty row gives +0.0
 *   mp_aggregate_backward (d_deg for mean, d_amax for max, as the forward wrote them; either output may be NULL):
 *     G = g, or g / (float)deg for mean; grad_x[t,c] = column sum of w[e,h] * G[row(e),c]; grad_w[e,h] = the sum of
 *     G[row(e),c] * x[t_e,c] over head h's channels in pool's lane order; for max only the terms an entry won */
int fslic_b200_mp_gather(int device, long long N, long long E, int C, int end, const long long* d_indptr,
                         const long long* d_targets, const float* d_x, float* d_out, void* stream);
size_t fslic_b200_mp_gather_backward_scratch_bytes(long long N, long long E);
int fslic_b200_mp_gather_backward(int device, long long N, long long E, int C, int end, const long long* d_indptr,
                                  const long long* d_targets, const float* d_grad_out, float* d_grad_x, void* d_scratch,
                                  size_t scratch_bytes, void* stream);
int fslic_b200_mp_softmax(int device, long long N, long long E, int H, const long long* d_indptr,
                          const long long* d_targets, const float* d_scores, float* d_out, void* stream);
int fslic_b200_mp_softmax_backward(int device, long long N, long long E, int H, const long long* d_indptr,
                                   const long long* d_targets, const float* d_out, const float* d_grad_out,
                                   float* d_grad_scores, void* stream);
int fslic_b200_mp_aggregate(int device, long long N, long long E, int C, int H, int reduce, const long long* d_indptr,
                            const long long* d_targets, const float* d_x, const float* d_weight, float* d_out,
                            int32_t* d_deg, int32_t* d_amax, void* stream);
size_t fslic_b200_mp_aggregate_backward_scratch_bytes(long long N, long long E, int C, int reduce);
int fslic_b200_mp_aggregate_backward(int device, long long N, long long E, int C, int H, int reduce,
                                     const long long* d_indptr, const long long* d_targets, const float* d_x,
                                     const float* d_weight, const int32_t* d_deg, const int32_t* d_amax,
                                     const float* d_grad_out, float* d_grad_x, float* d_grad_weight, void* d_scratch,
                                     size_t scratch_bytes, void* stream);

/* Stage probes for the parity tests (the reference's protected quad_image / assignment,
 * context.h:48-50): copies of the last iterate()'s Lab quad image [B,H,W,4] u8 and pre-CCA
 * labels [B,H,W] u16 into caller device buffers (either may be NULL). */
int fslic_b200_debug_stages(fslic_ctx* ctx, uint8_t* d_quad_out, uint16_t* d_precca_out, int batch, void* stream);

/* RGB -> quad stage alone (cielab.h:337-353): d_quad_out [B,H,W,4] u8. */
int fslic_b200_rgb_to_quad(fslic_ctx* ctx, const uint8_t* d_images, uint8_t* d_quad_out, int batch,
                           int convert_to_lab, void* stream);

/* libstdc++ std::partial_sort set selection on the device (cca.cpp:225-228), exposed for
 * differential tests: d_area int32[n]; writes d_kept u8[n] (1 = in the selected top-`middle`). */
int fslic_b200_debug_heap_select(fslic_ctx* ctx, const int32_t* d_area, int n, int middle, uint8_t* d_kept,
                                 void* stream);

/* With collect_timing >= 2: summed device time (CUDA events on the launch stream) and launch count of the
 * dominant kernel -- the fused assign+update kernel on the subsampled passes -- in the last iterate(). */
int fslic_b200_assign_kernel_time(fslic_ctx* ctx, float* total_ms, int* launches);

/* Diagnostics: the 8 int32 CCA counters of image `image` of the last (sub-)batch:
 * ncomp, ncand, nkept, sel_mode, keep_thres, need_sim, heap_ops, kth_area. */
int fslic_b200_debug_cca_counters(fslic_ctx* ctx, int32_t* out8, int image);

/* Milliseconds spent per stage in the last iterate() with collect_timing != 0. */
int fslic_b200_stage_ms(fslic_ctx* ctx, float* out_ms, int count);

/* Milliseconds of the connectivity stage's sub-sections in the last iterate() with collect_timing != 0 and fewer than
 * 4 images, in the reference's order and names (cca.cpp:194-263): build_disjoint_set, flatten, threshold_by_area,
 * sort, substitute, output.  Zeros when the stage was not timed (larger batches overlap the tail on a side stream). */
int fslic_b200_cca_stage_ms(fslic_ctx* ctx, float* out_ms, int count);

/* Geometry queries (S = (int16)sqrt(H*W/K), context.h:60; number of kernel launches per iterate). */
int fslic_b200_get_S(const fslic_ctx* ctx);
int fslic_b200_launches_last_iterate(const fslic_ctx* ctx);

/* Diagnostics: which assign kernel the last pass of the last iterate() used -- 5: the TMA-staged kernel
 * (k_assign5; needs W % 8 == 0 and subsample_stride 3), 4: the LDG kernel (k_assign_warp; any shape, taken where
 * the TMA-staged kernel does not apply), 0: the brute-force kernel / none yet. */
int fslic_b200_debug_assign_impl(const fslic_ctx* ctx);

/* Diagnostics: the launch decisions of the last iterate (any iterate entry point, host or device), as the host made
 * them when it enqueued the work -- no device synchronisation.  Writes min(count, FSLIC_DISPATCH_COUNT) int32 values:
 *   [0..5]   the last update pass launched: kernel, tps, grid, workers, items, trips
 *   [6..11]  the full-assign pass: the same six values
 *   [12]     kernel of the last prepare launch: 3 = k_prepare3, 2 = k_prepare2, 1 = k_prepare, 0 = none
 *   [13]     update passes whose TMA tail ran the next pass's prepare
 *   [14]     rounds of the LSC feature kernel (0 outside LSC)
 * kernel: 5 = TMA-staged, 4 = LDG warp tiles, 0 = generic, 10 / 11 / 12 = float-distance variant 0 / 1 / 2,
 * 13 = preemptive, 14 = LSC, -1 = no such pass.  tps: warp tiles per super tile (1 for the per-pixel kernels).
 * grid: CTAs launched.  workers: warps per CTA (tile kernels) or threads per CTA (per-pixel kernels).  items: super
 * tiles or pixels of the pass over the batch slice it ran on.  trips: ceil(items / (grid * workers)), the rounds of the
 * grid-stride walk.  The blocking host entry point may run a batch as two halves: the values are the second half's. */
#define FSLIC_DISPATCH_COUNT 15
int fslic_b200_debug_dispatch(const fslic_ctx* ctx, int32_t* out, int count);

/* Diagnostics: the launch decisions of the connectivity stage of the last iterate (any entry point) or
 * fslic_b200_enforce_connectivity call, as the host made them when it enqueued the work -- no device synchronisation.
 * Writes min(count, FSLIC_CCA_DISPATCH_COUNT) int32 values:
 *   [0]  heap_smem: the std::partial_sort replay's heap in shared memory (1) or in global memory (0); -1 = no
 *        connectivity stage ran.  Decided per call from K, whether or not an image then needs the replay
 *   [1]  heap_smem_max_k: the largest K whose heap fits shared memory on this device
 *   [2]  sub_batches: sub-batches the batch ran in (the context's scratch holds a bounded number of images)
 *   [3]  split: the first sub-batch ran its settled images' tail on a side stream (4 or more images)
 *   [4]  number_nb: 1024-pixel blocks per warp of the component-numbering kernel, first sub-batch */
#define FSLIC_CCA_DISPATCH_COUNT 5
int fslic_b200_debug_cca_dispatch(const fslic_ctx* ctx, int32_t* out, int count);

/* ---- SimpleCRF (src/simple-crf.{h,hpp,cpp}, csimple_crf.pyx): a mean-field CRF over superpixel nodes with per-frame
 * adjacency lists and node-to-node links between consecutive frames, for temporal smoothing of per-superpixel class
 * probabilities.  Bit-identical to the reference's object code (g++ -O3 -mavx2 -mfma) with glibc's expf, logf and
 * sqrtf.  Frames get times 0, 1, 2, ... from push_frame; the live ones always cover first_time..last_time.  Arrays of
 * a frame are [C][N] float, clusters fslic_cluster[N] (y, x, r, g, b and num_members are read), adjacency lists CSR.
 * All h_* buffers are host memory.  Every copy and kernel of a CRF runs on its stream: the last one passed to
 * inference (NULL at first), which may be any stream, blocking or not.  inference, initialize and reset_inferred
 * return at once; every other call synchronises that stream before it returns.  C * N must be < 2^31. */
typedef struct fslic_crf fslic_crf;

/* == SimpleCRFParams (simple-crf.h:11-19); defaults 10, 10, 13, 13, 80, 0, 3 */
typedef struct fslic_crf_params {
    float spatial_w, temporal_w, spatial_srgb, temporal_srgb, spatial_sxy, spatial_smooth_w, spatial_smooth_sxy;
} fslic_crf_params;

int fslic_b200_crf_create(int device, int num_classes, int num_nodes, fslic_crf** out);
int fslic_b200_crf_destroy(fslic_crf* crf);
int fslic_b200_crf_get_params(const fslic_crf* crf, fslic_crf_params* out);
int fslic_b200_crf_set_params(fslic_crf* crf, const fslic_crf_params* params);
/* first_time / last_time are -1 without frames; any pointer may be NULL */
int fslic_b200_crf_times(const fslic_crf* crf, int* first_time, int* last_time, int* num_frames);
int fslic_b200_crf_push_frame(fslic_crf* crf, int* time_out);
int fslic_b200_crf_pop_frame(fslic_crf* crf, int* time_out); /* *time_out = -1 when there are no frames */

/* Per frame; FSLIC_ENOFRAME when `time` is not live. */
int fslic_b200_crf_set_clusters(fslic_crf* crf, int time, const fslic_cluster* h_clusters);
int fslic_b200_crf_get_clusters(fslic_crf* crf, int time, fslic_cluster* h_out);
/* Rows 0..num_rows-1 (num_rows <= N) get the lists h_neighbors[h_offsets[i] .. h_offsets[i+1]); the others keep
 * theirs.  Neighbours outside [0, N) are refused and change nothing. */
int fslic_b200_crf_set_connectivity(fslic_crf* crf, int time, int num_rows, const int32_t* h_offsets,
                                    const int32_t* h_neighbors);
/* h_offsets [N + 1]; h_neighbors (may be NULL) receives at most `cap` neighbours */
int fslic_b200_crf_get_connectivity(fslic_crf* crf, int time, int32_t* h_offsets, int32_t* h_neighbors, long long cap);
int fslic_b200_crf_set_unary(fslic_crf* crf, int time, const float* h_unary);
int fslic_b200_crf_get_unary(fslic_crf* crf, int time, float* h_out);
int fslic_b200_crf_set_unbiased(fslic_crf* crf, int time);                      /* logf(C) everywhere */
int fslic_b200_crf_set_mask(fslic_crf* crf, int time, const int32_t* h_classes, float confidence); /* classes in [0,C) */
int fslic_b200_crf_set_proba(fslic_crf* crf, int time, const float* h_proba);   /* -logf(p) */
int fslic_b200_crf_get_inferred(fslic_crf* crf, int time, float* h_out);
int fslic_b200_crf_reset_inferred(fslic_crf* crf, int time);                   /* q = expf(-unary) */
int fslic_b200_crf_initialize(fslic_crf* crf);                                 /* reset_inferred on every frame */
/* max_iter Jacobi mean-field steps over all frames: 1 + 2 max_iter kernel launches, no host synchronisation.
 * FSLIC_ENOFRAME without frames (max_iter > 0). */
int fslic_b200_crf_inference(fslic_crf* crf, unsigned long long max_iter, void* stream);
int fslic_b200_crf_spatial_pairwise_energy(fslic_crf* crf, int time, int node_i, int node_j, float* out);
/* node's energy between frame `time` of crf and frame `other_time` of `other` (may be crf), with crf's params */
int fslic_b200_crf_temporal_pairwise_energy(fslic_crf* crf, int time, int node, fslic_crf* other, int other_time,
                                            float* out);

/* glibc's expf as the CRF evaluates it (fast_slic_b200/csrc/glibc_expf.cuh) over the bit patterns first,
 * first + 1, ... (n values, wrapping at 2^32): the host compile into h_out, the device compile into d_out. */
int fslic_b200_debug_expf_host(uint32_t first, long long n, float* h_out);
int fslic_b200_debug_expf_device(int device, uint32_t first, long long n, float* d_out, void* stream);

/* ---- The CRF fed from device memory (fast_slic_b200/csrc/crf_feed.cuh).  A separate prefix from the reference's
 * fslic_b200_crf_* surface above.  All d_* buffers are device memory on the CRF's device.  Each call adopts `stream`
 * like fslic_b200_crf_inference (waiting for the CRF's previous stream if it differs) and enqueues its work there
 * without waiting for it; labels, clusters, graphs and unaries never pass through the host.  Each frame equals what the
 * host path stores for the same input, bit for bit.  After a device push, the host-side readers of a frame
 * (get_clusters, get_connectivity, set_connectivity, the pairwise energies) first wait for the stream and download the
 * frame's records and adjacency lists once. */
/* Scratch bytes fslic_b200_crfdev_push_label_frames needs for `batch` label maps with K labels; (size_t)-1 if no
 * single call can take that batch. */
size_t fslic_b200_crfdev_push_scratch_bytes(int K, int batch);
/* Pushes `batch` frames.  Frame b holds d_clusters[b] ([K] records, converted as push_slic_frame converts them: y, x,
 * r, g, b and num_members truncated to int32 the way x86 numpy does, with INT_MIN for NaN, inf and out-of-range values),
 * the adjacency graph of d_labels[b] (int16 [H][W]; labels outside [0, K) ignored), and unbiased unaries.  K must
 * equal num_nodes.  Bad arguments are refused before anything is pushed.  times_out [batch] (host, may be NULL)
 * receives the new frames' times.  The one host wait is the frame-table upload every push makes; it covers work
 * enqueued before the call, not this push's kernels. */
int fslic_b200_crfdev_push_label_frames(fslic_crf* crf, int batch, int H, int W, int K, const uint16_t* d_labels,
                                        const fslic_cluster* d_clusters, void* d_scratch, size_t scratch_bytes,
                                        void* stream, int* times_out);
int fslic_b200_crfdev_set_unary(fslic_crf* crf, int time, const float* d_unary, void* stream);
int fslic_b200_crfdev_set_proba(fslic_crf* crf, int time, const float* d_proba, void* stream); /* -logf(p) */
/* classes int32 [N] are checked on the device; the call waits for that 4-byte flag and changes nothing (FSLIC_EINVAL)
 * if any class is outside [0, C) */
int fslic_b200_crfdev_set_mask(fslic_crf* crf, int time, const int32_t* d_classes, float confidence, void* stream);
int fslic_b200_crfdev_get_inferred(fslic_crf* crf, int time, float* d_out, void* stream);

/* ---- Groups: the CRFs of many video streams driven together.  crfs[0 .. n) are n distinct CRFs on one device with
 * the same num_classes C and num_nodes N; each keeps its own frames, params and time chain, and every result equals
 * what the member's own calls give, bit for bit.  The members of one call share each launch (up to 64 per launch set;
 * larger groups take several on the same stream).  Every call checks all its arguments before it enqueues anything
 * (a NULL or repeated member, mismatched device, C or N: FSLIC_EINVAL; for inference and the newest-frame calls, a
 * member without frames: FSLIC_ENOFRAME), so a refused call changes no member.  Each call adopts `stream` for every
 * member like fslic_b200_crf_inference, waiting once for each different stream they were on.  Afterwards every member
 * is in the state its own calls would have left it in, and its own entry points carry on from there.  d_* buffers are
 * device memory on the members' device; [n][C][N] buffers are float and hold member k's values at k. */
/* max_iter Jacobi steps of every member: 1 + 2 max_iter launches per 64 members, no host wait.  No-op for max_iter 0. */
int fslic_b200_crfgroup_inference(fslic_crf* const* crfs, int n, unsigned long long max_iter, void* stream);
/* Frame k, built from d_labels[k] and d_clusters[k] as fslic_b200_crfdev_push_label_frames builds it, is appended to
 * crfs[k]; one adjacency-graph pass over the n maps.  d_scratch as fslic_b200_crfdev_push_scratch_bytes(K, n) says.
 * times_out [n] (host, may be NULL) receives the new times.  One host wait, for the members' frame-table uploads. */
int fslic_b200_crfdev_group_push_label_frames(fslic_crf* const* crfs, int n, int H, int W, int K,
                                              const uint16_t* d_labels, const fslic_cluster* d_clusters,
                                              void* d_scratch, size_t scratch_bytes, void* stream, int* times_out);
/* set_proba (-logf(p)) of the newest frame of each member from d_proba [n][C][N] */
int fslic_b200_crfdev_group_set_proba(fslic_crf* const* crfs, int n, const float* d_proba, void* stream);
/* reset_inferred (q = expf(-unary)) of the newest frame of each member */
int fslic_b200_crfdev_group_reset_inferred(fslic_crf* const* crfs, int n, void* stream);
/* q of the newest frame of each member into d_out [n][C][N] */
int fslic_b200_crfdev_group_get_inferred(fslic_crf* const* crfs, int n, float* d_out, void* stream);
/* pop_frame of every member: times_out[k] (host, may be NULL) = the popped time, -1 for a member without frames.  One
 * host wait per stream the members are on. */
int fslic_b200_crfgroup_pop_frame(fslic_crf* const* crfs, int n, int* times_out);

/* Supervoxels (supervoxel.cuh, sv_cca.cuh; no counterpart in the reference; DESIGN.md section 4.22).
 * Connectivity enforcement of `batch` label volumes d_labels u16[B,D,H,W] into d_out i16[B,D,H,W] (d_out may be
 * d_labels): components are the 6-connected sets of equal labels, numbered by leader (smallest raster index) order;
 * those of area >= min_size are candidates, of more than K the K first by (area descending, leader ascending) are
 * kept and take 0, 1, .. in leader order; component 0 takes 0 if not kept; every other component takes the label of
 * the component of its leader's predecessor voxel (leader - 1 if x > 0, else - W if y > 0, else - H*W).  1 <= K <=
 * 65534, min_size >= 0, D, H, W <= 32767, D*H*W <= 2^29; B*D*H*W < 2^31 - 1 and B <= 65535 per call.  Scratch bytes:
 * (size_t)-1 for arguments out of range. */
size_t fslic_b200_sv_enforce_scratch_bytes(int batch, int D, int H, int W);
int fslic_b200_sv_enforce(int device, int batch, int D, int H, int W, int K, int min_size, const uint16_t* d_labels,
                          int16_t* d_out, void* d_scratch, size_t scratch_bytes, void* stream);
/* SLIC over `batch` volumes d_volumes f32[B,C,D,H,W] on an nd x nh x nw seed grid (K = nd*nh*nw <= 65534, 1 <= n_a <=
 * L_a): seed k = (iz*nh + iy)*nw + ix at the integer centre (lo + hi - 1) / 2 of its cell [i*L/n, (i+1)*L/n) on every
 * axis with that voxel's features.  Pass t < max_iter assigns the voxels of the rows y % stride == t % stride of every
 * slice, then updates; one full assign follows, then the enforcement above with min_size.  Candidates of voxel v:
 * |v_a - (int)c_a| <= R_a = ceil(L_a / n_a) on every axis; distance d = fc + ((w2z*(tz*tz) + w2y*(ty*ty)) +
 * w2x*(tx*tx)), fc = (((+0 + t_0*t_0) + t_1*t_1) + ..), t_c = f_c - mu_c, t_a = v_a - c_a, every float32 operation
 * rounded on its own; the winner is the smallest (bits(d) << 32 | k), a NaN distance having the bits 0x7fffffff; a
 * voxel without a candidate keeps its label (initially 0xffff).  Update: c_a = (float)((double)sum v_a / n), mu =
 * pool's mean over the pass voxels; a cluster with n = 0 keeps both.  Outputs: d_labels i16[B,D,H,W] after
 * enforcement, d_position f32[B,K,3] (z, y, x), d_centroids f32[B,K,C], d_count i32[B,K] (n of the last update, 0 when
 * max_iter = 0), and unless NULL d_overflow i32[max_iter + 1]: the tiles of each pass that went to the per-voxel
 * assign kernel.  1 <= C <= 1024, B*K <= 2^30, 1 <= stride <= 255, max_iter >= 0, w2 finite and >= 0; per call as
 * fslic_b200_sv_enforce.  Asynchronous on `stream`, never synchronises. */
size_t fslic_b200_sv_slic_scratch_bytes(int batch, int D, int H, int W, int C, int nd, int nh, int nw, int stride,
                                        int max_iter);
int fslic_b200_sv_slic(int device, int batch, int D, int H, int W, int C, int nd, int nh, int nw, float w2z, float w2y,
                       float w2x, int stride, int max_iter, int min_size, const float* d_volumes, int16_t* d_labels,
                       float* d_position, float* d_centroids, int32_t* d_count, int32_t* d_overflow, void* d_scratch,
                       size_t scratch_bytes, void* stream);

/* glibc's logf as the device feed evaluates it (fast_slic_b200/csrc/glibc_logf.cuh), like the expf pair above. */
int fslic_b200_debug_logf_host(uint32_t first, long long n, float* h_out);
int fslic_b200_debug_logf_device(int device, uint32_t first, long long n, float* d_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FSLIC_B200_H */
