// fast_slic_b200/csrc/capi_common.h -- what the translation units of the extern "C" boundary share: the error message
// fslic_b200_last_error returns, the device guard, the CUDA error check, the launch-size helpers, the limits of the
// label-map entry points and the scratch carve.
#pragma once
#include <string>
#include <cuda_runtime.h>
#include "../../include/fslic_b200.h"
#include "common.cuh"

// Stores msg as this thread's fslic_b200_last_error() and returns code.  Defined once, in capi.cu, next to the one
// thread-local message that the entry points of every translation unit (capi*.cu) write.
int set_err(int code, const std::string& msg);

// Every entry point runs on the context's device and puts the caller's current device back on return
// (a single-process multi-GPU PyTorch program must not find its current device changed behind its back).
struct DeviceGuard {
    int prev = -1;
    bool changed = false;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int dev) {
        err = cudaGetDevice(&prev);
        if (err == cudaSuccess && prev != dev) {
            err = cudaSetDevice(dev);
            changed = err == cudaSuccess;
        }
    }
    ~DeviceGuard() {
        if (changed) cudaSetDevice(prev);
    }
};
#define USE_DEVICE(dev)                                                                               \
    DeviceGuard dev_guard__(dev);                                                                     \
    if (dev_guard__.err != cudaSuccess)                                                               \
        return set_err(FSLIC_ECUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(dev_guard__.err))

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess)                                                                       \
            return set_err(FSLIC_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e__));         \
    } while (0)

// CTAs of 256 threads for a grid-stride kernel over `items` on `device`: one per 256 items, at least 1, at most 16 per
// SM of the device
static inline long grid_for(long items, int device) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 1;
    const long blocks = (items + 255) / 256, cap = 16L * sms;
    return blocks < 1 ? 1 : (blocks > cap ? cap : blocks);
}

// A grid of (x, y) blocks of 256 over `per_image` items of each of `batch` images: y = images (at most 65535, the
// kernels loop over the rest), x = enough blocks for one image, at most about 16 per SM over the whole grid
static inline dim3 image_grid(int batch, long per_image, int device) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0) sms = 1;
    const unsigned y = batch < 65535 ? (unsigned)batch : 65535u;
    long x = (per_image + 255) / 256;
    const long cap = 16L * sms / y;
    if (x > cap) x = cap;
    if (x < 1) x = 1;
    return dim3((unsigned)x, y);
}

static inline int bit_length(unsigned long long v) {
    int n = 0;
    for (; v; v >>= 1) n++;
    return n;
}

// Labels of the label-map entry points are read as uint16 and 65535 is no superpixel.  Where a count over one image
// must fit int32, an image has at most MAX_IMAGE_PIXELS pixels.
#define MAX_K 65534
#define MAX_IMAGE_PIXELS (1LL << 29)

static inline bool labels_shape_ok(int batch, int H, int W, int K) {
    return batch >= 0 && H >= 0 && W >= 0 && K >= 1 && K <= MAX_K;
}

// Hands out the pieces of one scratch buffer in order, each 256-byte aligned.  With a null base it hands out null
// pointers and only counts: one layout function gives both a *_scratch_bytes result (total) and the entry point's
// pointers, so the two cannot drift apart.
struct Carve {
    unsigned char* base;
    size_t total = 0;
    explicit Carve(void* p) : base(static_cast<unsigned char*>(p)) {}
    template <typename T>
    T* take(size_t bytes) {
        T* q = base ? reinterpret_cast<T*>(base + total) : nullptr;
        total += align_up(bytes, 256);
        return q;
    }
};
