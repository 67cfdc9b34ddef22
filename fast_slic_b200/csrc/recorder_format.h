// fast_slic_b200/csrc/recorder_format.h -- host-only text of the reference's debug_mode report (fslic_b200_format_report).
//
// The bytes Recorder::get_report (recorder.h:18-47, 90-98) streams out: `", "` between keys, `","` inside arrays,
// integers as integers and floats through `ostream <<` with default flags, i.e. printf's %.6g of the value as a double
// ("12", "12.3457", "3.40282e+38", "-0", "inf").  No CUDA call: the CPU suite tests it without a device.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace recorder_fmt {

// writes v at p, returns the end
static inline char* put_uint(char* p, uint32_t v) {
    char tmp[10];
    int n = 0;
    do {
        tmp[n++] = (char)('0' + v % 10);
        v /= 10;
    } while (v);
    while (n) *p++ = tmp[--n];
    return p;
}

static inline char* put_int(char* p, int v) {
    if (v < 0) {
        *p++ = '-';
        return put_uint(p, 0u - (uint32_t)v);
    }
    return put_uint(p, (uint32_t)v);
}

// %.6g of (double)v.  Integral values below 1e6 print as plain integers under %.6g: that common case (centres, colours,
// quantised distances) skips printf.
static inline char* put_float(char* p, float v) {
    if (v > -1e6f && v < 1e6f && v == (float)(int)v && !(v == 0.f && signbit(v))) return put_int(p, (int)v);
    char tmp[32];  // format_report sizes its buffer for kMaxNumber bytes per value: snprintf may not be told more
    const int n = snprintf(tmp, sizeof(tmp), "%.6g", (double)v);
    memcpy(p, tmp, (size_t)n);
    return p + n;
}

static inline char* put_str(char* p, const char* s) {
    const size_t n = strlen(s);
    memcpy(p, s, n);
    return p + n;
}

// Longest text of one value: %.6g of a float ("-1.17549e-38", "-nan") or a 32-bit integer, plus a separator; of one
// assignment entry: "65535,".
static const size_t kMaxNumber = 16;
static const size_t kMaxLabel = 6;
static const size_t kMaxCluster = 12 * kMaxNumber + 120;

// The report of `snapshots` snapshots (iterations -1, 0, 1, ...): assignment u16 [snapshots][H*W], min_dists u16 or
// float [snapshots][H*W], clusters [snapshots][K].  Returns a malloc'd, NUL-terminated buffer (NULL when out of memory).
static char* format_report(int H, int W, int K, int snapshots, bool dist_is_float, const uint16_t* assignment,
                           const void* min_dists, const fslic_cluster* clusters, size_t* len) {
    const size_t N = (size_t)H * W;
    // fixed text of a snapshot: '{"iteration": ', the number, the three array openings, ']}' and ',' -- 78 bytes at most
    // and per pixel one assignment entry and one min_dists value
    const size_t cap = 128 + (size_t)snapshots * (128 + (size_t)K * kMaxCluster + N * (kMaxLabel + kMaxNumber));
    char* buf = static_cast<char*>(malloc(cap));
    if (!buf) return nullptr;
    char* p = buf;
    p = put_str(p, "{\"height\": ");
    p = put_int(p, H);
    p = put_str(p, ", \"width\": ");
    p = put_int(p, W);
    p = put_str(p, ", \"snapshots\": [");
    for (int s = 0; s < snapshots; s++) {
        if (s > 0) *p++ = ',';
        p = put_str(p, "{\"iteration\": ");
        p = put_int(p, s - 1);
        p = put_str(p, ", \"clusters\": [");
        const fslic_cluster* cl = clusters + (size_t)s * K;
        for (int k = 0; k < K; k++) {
            const fslic_cluster& c = cl[k];
            if (k > 0) *p++ = ',';
            p = put_str(p, "{\"yx\": [");
            p = put_float(p, c.y);
            *p++ = ',';
            p = put_float(p, c.x);
            p = put_str(p, "], \"color\": [");
            p = put_float(p, c.r);
            *p++ = ',';
            p = put_float(p, c.g);
            *p++ = ',';
            p = put_float(p, c.b);
            p = put_str(p, "], \"is_updatable\": ");
            p = put_int(p, c.is_updatable);
            p = put_str(p, ", \"is_active\": ");
            p = put_int(p, c.is_active);
            p = put_str(p, ", \"number\": ");
            p = put_uint(p, c.number);
            p = put_str(p, ", \"num_members\": ");
            p = put_uint(p, c.num_members);
            *p++ = '}';
        }
        p = put_str(p, "], \"assignment\": [");
        const uint16_t* a = assignment + (size_t)s * N;
        for (size_t i = 0; i < N; i++) {
            if (i > 0) *p++ = ',';
            p = put_uint(p, a[i]);
        }
        p = put_str(p, "], \"min_dists\": [");
        if (dist_is_float) {
            const float* d = static_cast<const float*>(min_dists) + (size_t)s * N;
            for (size_t i = 0; i < N; i++) {
                if (i > 0) *p++ = ',';
                p = put_float(p, d[i]);
            }
        } else {
            const uint16_t* d = static_cast<const uint16_t*>(min_dists) + (size_t)s * N;
            for (size_t i = 0; i < N; i++) {
                if (i > 0) *p++ = ',';
                p = put_uint(p, d[i]);
            }
        }
        p = put_str(p, "]}");
    }
    p = put_str(p, "]}");
    *p = '\0';
    *len = (size_t)(p - buf);
    char* shrunk = static_cast<char*>(realloc(buf, *len + 1));
    return shrunk ? shrunk : buf;
}

}  // namespace recorder_fmt
