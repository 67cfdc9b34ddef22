// fast_slic_b200/csrc/common.cuh -- shared declarations for the sm_90a SLIC kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/fslic_b200.h"

#define FSLIC_FULL 0xffffffffu
#define CONN_MAX 12  // neighbours per label in the adjacency graph (max_conn, fast-slic.cpp:17)

// Out-of-window entries of the spatial patch.  Every in-window distance must stay below it and
// BIGSP + 765 (max colour SAD) must stay below 65536 so `d * 65536 + rank` never wraps.
#define FSLIC_BIGSP 64770u

// Per-cluster record the assign kernels read (16 B, one LDG.128).  Rebuilt by k_prepare every pass.
struct __align__(16) CInfo {
    int32_t cyx;       // (int16)cy | (int16)cx << 16   -- truncated + clamped centre (context.cpp:209-212,266)
    uint32_t color;    // cr | cg << 8 | cb << 16       -- (int16) casts of Cluster.r/g/b, always 0..255 here
    uint32_t sortkey;  // phase << 16 | k               -- the reference's visiting order (context.cpp:214-242)
    uint32_t pad;
};

__device__ __forceinline__ uint32_t sad4_acc(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;  // |a0-b0|+|a1-b1|+|a2-b2|+|a3-b3| + c   (SASS: VABSDIFF4.U8.ACC)
}

__device__ __forceinline__ uint32_t ld_nc_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// Slot hash of a label-pair key (a << 16 | b) in the open-addressing pair tables (graph.cuh, rag.cuh)
__device__ __forceinline__ uint32_t conn_hash(uint32_t key) {
    key ^= key >> 15;
    key *= 0x2c1b3c6du;
    key ^= key >> 12;
    key *= 0x297a2d39u;
    key ^= key >> 15;
    return key;
}

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
