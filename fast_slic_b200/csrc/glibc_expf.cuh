// glibc_expf.cuh -- a bit-exact clone of glibc's single-precision expf (the __expf_fma variant that libm's IFUNC picks
// on every FMA-capable x86 host), for the host and the device.
//
// The CRF (crf.cuh) must reproduce the reference's object code, which calls glibc expf.  glibc's expf is not correctly
// rounded (it differs from (float)exp((double)x) on ~170k of the 2^32 inputs), so neither CUDA's expf/__expf nor a
// correctly rounded expf will do.  The scheme is the published one (Arm optimized-routines, glibc sysdeps/ieee754/flt-32
// e_expf.c): x*32/ln2 is split into an integer k and a remainder r in double precision, 2^(k/32) comes from a 32-entry
// table with the exponent added by integer shift, and 2^(r/32) is a degree-3 polynomial.  Which operations the FMA
// build contracts was read from libm's object code:
//   kd = fma(InvLn2N, xd, SHIFT)     z is never rounded on its own
//   r  = fma(InvLn2N, xd, -(kd - SHIFT))
//   y  = fma(fma(C0, r, C1), r*r, fma(C2, r, 1)) * s
// and the special cases are the ones its slow path tests, in its order (below).  NaN inputs come back quieted with
// their sign and payload, which is what x86's `x + x` does, so the clone equals glibc on all 2^32 bit patterns.
#pragma once
#include <stdint.h>
#include <string.h>
#include <math.h>

namespace gexpf {

// bits of 2^(i/32) rounded to double, minus i << 47 (the exponent is added back from k)
#define GEXPF_TABLE                                                                                         \
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,             \
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,             \
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,             \
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,             \
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,             \
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,             \
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,             \
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull

__device__ const uint64_t kTabDev[32] = {GEXPF_TABLE};
static const uint64_t kTabHost[32] = {GEXPF_TABLE};

__host__ __device__ inline uint32_t f2u(float f) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(f);
#else
    uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
__host__ __device__ inline float u2f(uint32_t u) {
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f; memcpy(&f, &u, 4); return f;
#endif
}
__host__ __device__ inline uint64_t d2u(double d) {
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t u; memcpy(&u, &d, 8); return u;
#endif
}
__host__ __device__ inline double u2d(uint64_t u) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)u);
#else
    double d; memcpy(&d, &u, 8); return d;
#endif
}

__host__ __device__ inline float expf(float x) {
    const double kShift = 0x1.8p52, kInvLn2N = 0x1.71547652b82fep+5;  // 32 / ln 2
    const double kC0 = 0x1.c6af84b912394p-20, kC1 = 0x1.ebfce50fac4f3p-13, kC2 = 0x1.62e42ff0c52d6p-6;
    const uint32_t ux = f2u(x);
    const uint32_t abstop = (ux >> 20) & 0x7ff;
    if (abstop >= 0x42b) {                                   // |x| >= 88, inf or NaN
        if (ux == 0xff800000u) return 0.0f;                  // exp(-inf)
        if (abstop >= 0x7f8) return ux == 0x7f800000u ? x : u2f(ux | 0x00400000u);  // +inf; NaN quieted (x + x)
        if (x > 0x1.62e42ep6f) return u2f(0x7f800000u);      // __math_oflowf: 0x1p97f * 0x1p97f
        if (x < -0x1.9fe368p6f) return 0.0f;                 // __math_uflowf: 0x1p-95f * 0x1p-95f
        if (x < -0x1.9d1d9ep6f) return u2f(1u);              // __math_may_uflowf: 0x1.4p-75f * 0x1.4p-75f = 0x1p-149
    }
#ifdef __CUDA_ARCH__
    const double xd = (double)x;
    double kd = __fma_rn(kInvLn2N, xd, kShift);
    const uint64_t ki = d2u(kd);
    kd = __dadd_rn(kd, -kShift);
    const double r = __fma_rn(kInvLn2N, xd, -kd);
    const double s = u2d(kTabDev[ki & 31] + (ki << 47));
    const double z = __fma_rn(kC0, r, kC1);
    const double r2 = __dmul_rn(r, r);
    double y = __fma_rn(kC2, r, 1.0);
    y = __fma_rn(z, r2, y);
    return __double2float_rn(__dmul_rn(y, s));
#else
    const double xd = (double)x;
    double kd = fma(kInvLn2N, xd, kShift);
    const uint64_t ki = d2u(kd);
    kd = kd - kShift;
    const double r = fma(kInvLn2N, xd, -kd);
    const double s = u2d(kTabHost[ki & 31] + (ki << 47));
    const double z = fma(kC0, r, kC1);
    const double r2 = r * r;
    double y = fma(kC2, r, 1.0);
    y = fma(z, r2, y);
    return (float)(y * s);
#endif
}

#undef GEXPF_TABLE
}  // namespace gexpf
