// glibc_logf.cuh -- a bit-exact clone of glibc's single-precision logf (the __logf_fma variant that libm's IFUNC picks
// on every FMA-capable x86 host), for the host and the device.
//
// The CRF's unary setters (set_proba, set_mask, set_unbiased) compute -logf with glibc, as the reference does.  glibc's
// logf is not correctly rounded, so CUDA's logf/__logf will not do; the device feed (crf_feed.cuh) uses this clone.
// The scheme is the published one (Arm optimized-routines, glibc sysdeps/ieee754/flt-32/e_logf.c): x = 2^k z with z
// in [0x3f330000, 2 * 0x3f330000), a 16-entry (1/c, log c) table picked by the top mantissa bits of z, and log1p(z/c - 1)
// as a degree-3 polynomial in double.  Which operations the FMA build contracts was read from libm's object code:
//   r  = fma(z, invc, -1.0)
//   y0 = fma((double)k, Ln2, logc)
//   y  = fma(r2, A0, fma(A1, r, A2))            r2 = r * r
//   y  = fma(r2, y, r + y0)
// The special cases are its slow path's, in its order: x == 1 gives +0; then, for x outside the normal positives,
// ±0 gives -inf (__math_divzerof), +inf gives +inf, a negative x or NaN goes to __math_invalidf ((x - x) / (x - x)),
// and a subnormal is scaled by 2^23 and its exponent taken back.  On x86, __math_invalidf gives the NaN input quieted
// with its sign and payload, and the default NaN 0xffc00000 for a negative non-NaN; both are written as bit patterns
// here, so the host and the device compiles equal glibc on all 2^32 inputs.
#pragma once
#include <stdint.h>
#include <math.h>
#include "glibc_expf.cuh"  // gexpf::f2u / u2f / u2d

namespace glogf {

// (bits of 1/c, bits of log c) for the 16 subintervals
#define GLOGF_TABLE                                                                                       \
    0x3ff661ec79f8f3beull, 0xbfd57bf7808caadeull, 0x3ff571ed4aaf883dull, 0xbfd2bef0a7c06ddbull,           \
    0x3ff49539f0f010b0ull, 0xbfd01eae7f513a67ull, 0x3ff3c995b0b80385ull, 0xbfcb31d8a68224e9ull,           \
    0x3ff30d190c8864a5ull, 0xbfc6574f0ac07758ull, 0x3ff25e227b0b8ea0ull, 0xbfc1aa2bc79c8100ull,           \
    0x3ff1bb4a4a1a343full, 0xbfba4e76ce8c0e5eull, 0x3ff12358f08ae5baull, 0xbfb1973c5a611cccull,           \
    0x3ff0953f419900a7ull, 0xbfa252f438e10c1eull, 0x3ff0000000000000ull, 0x0000000000000000ull,           \
    0x3fee608cfd9a47acull, 0x3faaa5aa5df25984ull, 0x3feca4b31f026aa0ull, 0x3fbc5e53aa362eb4ull,           \
    0x3feb2036576afce6ull, 0x3fc526e57720db08ull, 0x3fe9c2d163a1aa2dull, 0x3fcbc2860d224770ull,           \
    0x3fe886e6037841edull, 0x3fd1058bc8a07ee1ull, 0x3fe767dcf5534862ull, 0x3fd4043057b6ee09ull

__device__ const uint64_t kTabDev[32] = {GLOGF_TABLE};
static const uint64_t kTabHost[32] = {GLOGF_TABLE};

__host__ __device__ inline float logf(float x) {
    const double kLn2 = 0x1.62e42fefa39efp-1;
    const double kA0 = -0x1.00ea348b88334p-2, kA1 = 0x1.5575b0be00b6ap-2, kA2 = -0x1.ffffef20a4123p-2;
    uint32_t ix = gexpf::f2u(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {  // x < 0x1p-126, inf or NaN
        if (ix * 2u == 0u) return gexpf::u2f(0xff800000u);  // __math_divzerof(1): -1 / 0
        if (ix == 0x7f800000u) return x;                     // log(inf) = inf
        if ((ix & 0x80000000u) || ix * 2u >= 0xff000000u)    // __math_invalidf
            return gexpf::u2f(ix * 2u > 0xff000000u ? ix | 0x00400000u : 0xffc00000u);
        ix = gexpf::f2u(x * 0x1p23f) - (23u << 23);          // subnormal: exact scaling
    }
    const uint32_t tmp = ix - 0x3f330000u;
    const int i = (int)((tmp >> 19) % 16u);
    const int k = (int32_t)tmp >> 23;
    const uint32_t iz = ix - (tmp & 0xff800000u);
    const double z = (double)gexpf::u2f(iz);
#ifdef __CUDA_ARCH__
    const double invc = gexpf::u2d(kTabDev[2 * i]), logc = gexpf::u2d(kTabDev[2 * i + 1]);
    const double r = __fma_rn(z, invc, -1.0);
    const double y0 = __fma_rn((double)k, kLn2, logc);
    const double r2 = __dmul_rn(r, r);
    double y = __fma_rn(kA1, r, kA2);
    y = __fma_rn(r2, kA0, y);
    y = __fma_rn(r2, y, __dadd_rn(r, y0));
    return __double2float_rn(y);
#else
    const double invc = gexpf::u2d(kTabHost[2 * i]), logc = gexpf::u2d(kTabHost[2 * i + 1]);
    const double r = fma(z, invc, -1.0);
    const double y0 = fma((double)k, kLn2, logc);
    const double r2 = r * r;
    double y = fma(kA1, r, kA2);
    y = fma(r2, kA0, y);
    y = fma(r2, y, r + y0);
    return (float)y;
#endif
}

// -logf(x) with the sign flipped as a bit, which is what x86's negation does to every value, NaN included
__host__ __device__ inline float neg_logf(float x) { return gexpf::u2f(gexpf::f2u(logf(x)) ^ 0x80000000u); }

#undef GLOGF_TABLE
}  // namespace glogf
