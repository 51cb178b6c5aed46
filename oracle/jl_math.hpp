// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product path: only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use it.
//
// CPU restatement of the Julia Base math the reference's classic-control envs call
// (the reference is 100 % Julia and cannot run here; see DESIGN.md "Oracle").
//
// What is restated (Julia 1.10 semantics, base/special/trig.jl + rem_pio2.jl, which are
// Julia ports of FreeBSD msun k_sinf/k_cosf/k_sin/k_cos/e_rem_pio2f):
//   * sin/cos(::Float32): evaluated on the widened Float64 argument with the msun
//     float kernels, rounded once; tiny-argument short cuts; Cody–Waite reduction.
//   * sin/cos(::Float64): msun double kernels for |x| < pi/4, 3-stage Cody–Waite beyond.
//   * `@horner` expands to `muladd`, which LLVM fuses on every FMA-capable x86-64
//     (Haswell+, i.e. every x86-64 GPU host) -> restated as an explicit fma().  Everything
//     else is NOT contracted (compile with -ffp-contract=off).
//   * mod(::Float64, ::Float64), clamp.
// Call sites in the reference: CartPoleEnv.jl:122-123 (cos/sin theta),
// PendulumEnv.jl:70-71,108 (sin/cos/mod), MountainCarEnv.jl:122 (cos(3x)).
// PARITY UNPINNED: the reference has no golden trajectory for these envs (SURVEY §8c);
// this file is pinned only by the Appendix-C known answers in tests/.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace jl {

static inline double muladd(double a, double b, double c) { return __builtin_fma(a, b, c); }

// ---- Float32 kernels (argument already widened to double: DoubleFloat32.hi) --------
static inline float sin_kernel_f32(double y) {
    const double S1 = -0.16666666641626524, S2 = 0.008333329385889463;
    double z = y * y;
    double w = z * z;
    double r = muladd(z, 2.718311493989822e-6, -0.00019839334836096632);
    double s = z * y;
    return (float)((y + s * muladd(z, S2, S1)) + (s * w) * r);
}
static inline float cos_kernel_f32(double y) {
    const double C0 = -0.499999997251031, C1 = 0.04166662332373906;
    const double C2 = -0.001388676377460993, C3 = 2.439044879627741e-5;
    double z = y * y;
    double w = z * z;
    double r = muladd(z, C3, C2);
    return (float)(((1.0 + z * C0) + w * C1) + (w * z) * r);
}

static const double PI_D = 3.141592653589793;  // Float64(pi)

// rem_pio2_kernel(x::Float32): returns n and the reduced argument (double).
// Supported range |x| < Float32(pi)/2 * 2^28 (the "medium" Cody–Waite range); the
// Payne–Hanek branch for larger |x| is not restated (no env can reach it).
static inline int rem_pio2_f32(float x, double* y) {
    const double pio2_1 = 1.57079631090164184570e+00;
    const double pio2_1t = 1.58932547735281966916e-08;
    const double inv_pio2 = 6.36619772367581382433e-01;
    double xd = (double)x;
    double ax = std::fabs(xd);
    if (ax <= PI_D * 5 / 4) {
        if (ax <= PI_D * 3 / 4) {
            if (x > 0) { *y = xd - PI_D / 2; return 1; }
            *y = xd + PI_D / 2; return -1;
        }
        if (x > 0) { *y = xd - PI_D; return 2; }
        *y = xd + PI_D; return -2;
    } else if (ax <= PI_D * 9 / 4) {
        if (ax <= PI_D * 7 / 4) {
            if (x > 0) { *y = xd - PI_D * 3 / 2; return 3; }
            *y = xd + PI_D * 3 / 2; return -3;
        }
        if (x > 0) { *y = xd - PI_D * 4 / 2; return 4; }
        *y = xd + PI_D * 4 / 2; return -4;
    }
    double fn = std::nearbyint(xd * inv_pio2);  // round-half-even, like Julia round()
    double r = xd - fn * pio2_1;
    double w = fn * pio2_1t;
    *y = r - w;
    return (int)(long long)fn;
}

static inline float sin32(float x) {
    float ax = std::fabs(x);
    if (ax < 0.78539819f /* Float32(pi)/4 */) {
        if (ax < 0x1.6a09e6p-12f /* sqrt(eps(Float32)) */) return x;
        return sin_kernel_f32((double)x);
    }
    if (std::isnan(x) || std::isinf(x)) return NAN;  // Julia throws DomainError on Inf
    double y;
    int n = rem_pio2_f32(x, &y) & 3;
    if (n == 0) return sin_kernel_f32(y);
    if (n == 1) return cos_kernel_f32(y);
    if (n == 2) return -sin_kernel_f32(y);
    return -cos_kernel_f32(y);
}
static inline float cos32(float x) {
    float ax = std::fabs(x);
    if (ax < 0.78539819f) {
        if (ax < 0x1p-12f /* sqrt(eps(Float32)/2) */) return 1.0f;
        return cos_kernel_f32((double)x);
    }
    if (std::isnan(x) || std::isinf(x)) return NAN;
    double y;
    int n = rem_pio2_f32(x, &y) & 3;
    if (n == 0) return cos_kernel_f32(y);
    if (n == 1) return -sin_kernel_f32(y);
    if (n == 2) return -cos_kernel_f32(y);
    return sin_kernel_f32(y);
}

// ---- Float64 kernels -----------------------------------------------------------------
static const double DS1 = -1.66666666666666324348e-01, DS2 = 8.33333333332248946124e-03,
                    DS3 = -1.98412698298579493134e-04, DS4 = 2.75573137070700676789e-06,
                    DS5 = -2.50507602534068634195e-08, DS6 = 1.58969099521155010221e-10;
static const double DC1 = 4.16666666666666019037e-02, DC2 = -1.38888888888741095749e-03,
                    DC3 = 2.48015872894767294178e-05, DC4 = -2.75573143513906633035e-07,
                    DC5 = 2.08757232129817482790e-09, DC6 = -1.13596475577881948265e-11;

static inline double sin_kernel_f64(double y) {  // sin_kernel(y::Float64)
    double y2 = y * y, y4 = y2 * y2;
    double r = muladd(y2, muladd(y2, DS4, DS3), DS2) + y2 * y4 * muladd(y2, DS6, DS5);
    double y3 = y2 * y;
    return y + y3 * (DS1 + y2 * r);
}
static inline double sin_kernel_f64(double hi, double lo) {  // DoubleFloat64
    double y2 = hi * hi, y4 = y2 * y2;
    double r = muladd(y2, muladd(y2, DS4, DS3), DS2) + y2 * y4 * muladd(y2, DS6, DS5);
    double y3 = y2 * hi;
    return hi - ((y2 * (0.5 * lo - y3 * r) - lo) - y3 * DS1);
}
static inline double cos_kernel_f64(double hi, double lo) {
    double y2 = hi * hi, y4 = y2 * y2;
    double r = y2 * muladd(y2, muladd(y2, DC3, DC2), DC1) +
               y4 * y4 * muladd(y2, muladd(y2, DC6, DC5), DC4);
    double half = 0.5 * y2;
    double w = 1.0 - half;
    return w + (((1.0 - w) - half) + (y2 * r - hi * lo));
}
static inline uint32_t highword(double x) {
    uint64_t b; std::memcpy(&b, &x, 8); return (uint32_t)(b >> 32);
}
// cody_waite_2c_pio2(x, fn, n) (rem_pio2.jl): two-constant reduction for |x| <= 9pi/4 away from multiples of pi/2
static inline int cody_waite_2c(double x, double fn, int n, double* y1o, double* y2o) {
    const double pio2_1 = 1.57079632673412561417e+00, pio2_1t = 6.07710050650619224932e-11;
    double z = muladd(-fn, pio2_1, x);
    double w = fn * pio2_1t;
    double y1 = z - w;
    *y1o = y1;
    *y2o = (z - y1) - w;
    return n;
}
// cody_waite_ext_pio2 (medium range, |x| < 2^20*pi/2): up to three rounds
static inline int cody_waite_ext(double x, uint32_t xhp, double* y1o, double* y2o) {
    const double pio2_1 = 1.57079632673412561417e+00, pio2_1t = 6.07710050650619224932e-11;
    const double pio2_2 = 6.07710050630396597660e-11, pio2_2t = 2.02226624879595063154e-21;
    const double pio2_3 = 2.02226624871116645580e-21, pio2_3t = 8.47842766036889956997e-32;
    double fn = std::nearbyint(x * 6.36619772367581382433e-01);
    double r = muladd(-fn, pio2_1, x);
    double w = fn * pio2_1t;
    int j = (int)(xhp >> 20);
    double y1 = r - w;
    int i = j - (int)((highword(y1) >> 20) & 0x7ff);
    if (i > 16) {
        double t = r;
        w = fn * pio2_2;
        r = t - w;
        w = muladd(fn, pio2_2t, -((t - r) - w));
        y1 = r - w;
        i = j - (int)((highword(y1) >> 20) & 0x7ff);
        if (i > 49) {
            t = r;
            w = fn * pio2_3;
            r = t - w;
            w = muladd(fn, pio2_3t, -((t - r) - w));
            y1 = r - w;
        }
    }
    *y1o = y1;
    *y2o = (r - y1) - w;
    return (int)(long long)fn;
}
// rem_pio2_kernel(x::Float64) (base/special/rem_pio2.jl, a port of msun e_rem_pio2.c): the decision tree on the high word —
// |x| <= 9pi/4 takes the two-constant scheme with fn = +-1..4 unless x is close to a multiple of pi/2; everything else up to
// 2^20 pi/2 the extended scheme.  Payne-Hanek beyond is not restated (no env can reach it).  UNPINNED like the rest of this file
// (recalled from the Julia sources; the constants are msun's, pinned by tests/test_oracle_msun_constants.py).
static inline int rem_pio2_f64(double x, double* y1o, double* y2o) {
    const uint32_t xhp = highword(x) & 0x7fffffffu;
    const bool pos = x > 0.0;
    if (xhp <= 0x400f6a7au) {                      // |x| ~<= 5pi/4
        if ((xhp & 0xfffffu) == 0x921fbu) return cody_waite_ext(x, xhp, y1o, y2o);
        if (xhp <= 0x4002d97cu) return pos ? cody_waite_2c(x, 1.0, 1, y1o, y2o) : cody_waite_2c(x, -1.0, -1, y1o, y2o);
        return pos ? cody_waite_2c(x, 2.0, 2, y1o, y2o) : cody_waite_2c(x, -2.0, -2, y1o, y2o);
    }
    if (xhp <= 0x401c463bu) {                      // |x| ~<= 9pi/4
        if (xhp <= 0x4015fdbcu) {                  // |x| ~<= 7pi/4
            if (xhp == 0x4012d97cu) return cody_waite_ext(x, xhp, y1o, y2o);
            return pos ? cody_waite_2c(x, 3.0, 3, y1o, y2o) : cody_waite_2c(x, -3.0, -3, y1o, y2o);
        }
        if (xhp == 0x401921fbu) return cody_waite_ext(x, xhp, y1o, y2o);
        return pos ? cody_waite_2c(x, 4.0, 4, y1o, y2o) : cody_waite_2c(x, -4.0, -4, y1o, y2o);
    }
    return cody_waite_ext(x, xhp, y1o, y2o);
}
static inline double sin64(double x) {
    double ax = std::fabs(x);
    if (ax < PI_D / 4) {
        if (ax < 0x1p-26 /* sqrt(eps(Float64)) */) return x;
        return sin_kernel_f64(x);
    }
    if (std::isnan(x) || std::isinf(x)) return NAN;
    double hi, lo;
    int n = rem_pio2_f64(x, &hi, &lo) & 3;
    if (n == 0) return sin_kernel_f64(hi, lo);
    if (n == 1) return cos_kernel_f64(hi, lo);
    if (n == 2) return -sin_kernel_f64(hi, lo);
    return -cos_kernel_f64(hi, lo);
}
static inline double cos64(double x) {
    double ax = std::fabs(x);
    if (ax < PI_D / 4) {
        if (ax < 0x1.6a09e667f3bcdp-27 /* sqrt(eps(Float64)/2) */) return 1.0;
        return cos_kernel_f64(x, 0.0);
    }
    if (std::isnan(x) || std::isinf(x)) return NAN;
    double hi, lo;
    int n = rem_pio2_f64(x, &hi, &lo) & 3;
    if (n == 0) return cos_kernel_f64(hi, lo);
    if (n == 1) return -sin_kernel_f64(hi, lo);
    if (n == 2) return -cos_kernel_f64(hi, lo);
    return sin_kernel_f64(hi, lo);
}

static inline float jsin(float x) { return sin32(x); }
static inline float jcos(float x) { return cos32(x); }
static inline double jsin(double x) { return sin64(x); }
static inline double jcos(double x) { return cos64(x); }

// Base.mod(x::Float64, y::Float64) (base/float.jl): rem = fmod, sign fix-up.
static inline double jmod(double x, double y) {
    double r = std::fmod(x, y);
    if (r == 0) return std::copysign(r, y);
    if ((r > 0) != (y > 0)) return r + y;
    return r;
}
template <class T> static inline T jclamp(T x, T lo, T hi) {
    return x > hi ? hi : (x < lo ? lo : x);
}
// x * b for b::Bool ("strong zero": x*false == copysign(0, x), also for NaN/Inf).
template <class T> static inline T mul_bool(T x, bool b) { return b ? x : std::copysign((T)0, x); }

}  // namespace jl
