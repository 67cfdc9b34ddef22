// fast_slic_b200/csrc/capi_common.h -- what the translation units of the extern "C" boundary share: the error message
// fslic_b200_last_error returns, the device guard, the CUDA error check and the launch-size helpers.
#pragma once
#include <string>
#include <cuda_runtime.h>
#include "../../include/fslic_b200.h"

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

static inline int bit_length(unsigned long long v) {
    int n = 0;
    for (; v; v >>= 1) n++;
    return n;
}
