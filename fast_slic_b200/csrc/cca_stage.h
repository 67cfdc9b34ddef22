// fast_slic_b200/csrc/cca_stage.h -- the host side of connectivity enforcement (cca_stage.cu, kernels in cca.cuh):
// its scratch, side streams, timing and launch sequence, owned by one CcaStage per context.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <cuda_runtime.h>

struct CcaCounters;  // per-image scalars of the kernels (cca.cuh)

// Slots of the selection heap per image: enough for every K a u16 label map can have (K + 2 <= CCA_HEAP_K)
constexpr int CCA_HEAP_K = 65536 + 8;

// What cca_run enqueued (fslic_b200_debug_cca_dispatch)
struct CcaDispatch {
    int heap_smem = -1;       // k_cca_select's heap: 1 = shared memory, 0 = global memory, -1 = no connectivity stage ran
    int heap_smem_max_k = 0;  // largest K whose heap fits shared memory on this device
    int sub_batches = 0;      // sub-batches of at most CcaStage::batch images
    int split = 0;            // first sub-batch: settled images' tail on the side stream (nb >= 4)
    int number_nb = 0;        // first sub-batch: 1024-pixel blocks per k_ccl_number warp
};

// Host-output hook of cca_run (iterate_host only): label maps are copied to the host as soon as they are final --
// for the images k_cca_threshold settled that is while the std::partial_sort replay of the others still runs.
struct HostOut {
    uint16_t* h_labels;      // destination of image 0 of this call
    cudaStream_t out_stream;
    bool done;               // set when cca_run issued the label copies itself
};

// A side stream and its events: the finishing kernels of the settled images run there, beside the replay
struct CcaLane {
    cudaStream_t side = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr, tail = nullptr;
};

struct CcaStage {
    int H = 0, W = 0, N = 0, num_sms = 0, max_smem_optin = 0;
    int batch = 1;             // images per sub-batch: the scratch holds this many
    void* scratch = nullptr;   // one allocation, laid out by cca_layout (cca_stage.cu)
    CcaCounters* h_counters = nullptr;  // pinned, 64 entries: lets the host path learn which images need the replay
    // the blocking host path runs the two halves of a batch as two calls that overlap on the device: one lane each
    CcaLane lanes[2];
    // the reference's sub-sections of "cca" (cca.cpp:194-263): build_disjoint_set, flatten, threshold_by_area, sort,
    // substitute, output -- event-timed when timing is on and the batch is not split across streams
    cudaEvent_t ev[7] = {};
    float ms[6] = {};
    bool timing = false, timed = false;
};

// Sizes the scratch for up to max_batch images (device_bytes: the device's memory, 0 if unknown) and creates the
// stage's allocations, streams and events.  On an error, cca_stage_destroy frees what was made.
cudaError_t cca_stage_create(CcaStage& s, int H, int W, int max_batch, size_t device_bytes, int num_sms, int max_smem_optin);
void cca_stage_destroy(CcaStage& s);

// Connectivity enforcement of `batch` images from d_in into d_out (may alias) on st, in sub-batches of s.batch images.
// `slot` / `lane`: the window of the scratch (images slot .. slot + batch) and the side stream the call uses.
int cca_run(CcaStage& s, CcaDispatch& d, const uint16_t* d_in, uint16_t* d_out, int batch, int K, int thres,
            cudaStream_t st, int* launches, HostOut* ho = nullptr, int slot = 0, int lane = 0);

// Event timing of the sub-sections: armed before a call, read back (into s.ms) after its end was synchronised
void cca_set_timing(CcaStage& s, bool on);
void cca_read_timing(CcaStage& s);
// Waits for both side streams (error path of the host entry points); errors are left to the caller
void cca_sync_lanes(const CcaStage& s);

// The diagnostics entry points
int cca_heap_select(const CcaStage& s, const int32_t* d_area, int n, int middle, uint8_t* d_kept, cudaStream_t st);
int cca_read_counters(const CcaStage& s, int32_t* out8, int image);
void cca_read_dispatch(const CcaDispatch& d, int32_t* out, int count);
void cca_read_ms(const CcaStage& s, float* out_ms, int count);
