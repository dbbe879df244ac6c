// resize_host.cpp — pixo's Lanczos3 contribution tables (src/resize.rs:391-456), computed on the host once
// per geometry: O(width + height) work that every frame of a batch shares.
//
// lanczos_kernel calls f32::sin.  In pixo's wasm build that is the Rust libm port of musl's sinf: the
// argument is reduced and evaluated in double precision, then rounded once to f32.  It is not correctly
// rounded, so neither CUDA's sinf nor (float)sin((double)x) reproduces it everywhere, and a weight one ulp
// off moves an output byte whenever a sum lands next to a .5 boundary.  resize_sinf restates it for the
// arguments the kernel passes (|pi x| < 3 pi, plus the medium range reduction for safety); DESIGN.md
// section 7 records how it was checked against the wasm.  Compiled without contraction or fast-math.
#include "resize_host.hpp"

#include <math.h>
#include <string.h>

namespace pixo {

namespace {

// __sindf / __cosdf: sin and cos on |x| <= pi/4 as double polynomials, rounded once to f32
float k_sin(double x)
{
    const double S1 = -0x15555554cbac77.0p-55, S2 = 0x111110896efbb2.0p-59, S3 = -0x1a00f9e2cae774.0p-65,
                 S4 = 0x16cd878c3b46a7.0p-71;
    const double z = x * x, w = z * z, r = S3 + z * S4, s = z * x;
    return (float)((x + s * (S1 + z * S2)) + s * w * r);
}

float k_cos(double x)
{
    const double C0 = -0x1ffffffd0c5e81.0p-54, C1 = 0x155553e1053a42.0p-57, C2 = -0x16c087e80f1e27.0p-62,
                 C3 = 0x199342e0ee5069.0p-68;
    const double z = x * x, w = z * z, r = C2 + z * C3;
    return (float)(((1.0 + z * C0) + w * C1) + (w * z) * r);
}

const float kEps = 1.1920928955078125e-7f;  // f32::EPSILON

float lanczos3(float x)
{
    const float a = 3.0f, pi = 3.14159265358979323846f;
    if (fabsf(x) < kEps) return 1.0f;
    if (fabsf(x) >= a) return 0.0f;
    const float pi_x = pi * x, pi_x_a = pi * x / a;
    return (a * resize_sinf(pi_x) * resize_sinf(pi_x_a)) / (pi_x * pi_x_a);
}

}  // namespace

float resize_sinf(float x)
{
    const double pio2 = 1.57079632679489661923;
    const double p1 = 1 * pio2, p2 = 2 * pio2, p3 = 3 * pio2, p4 = 4 * pio2;
    uint32_t ix;
    memcpy(&ix, &x, 4);
    const bool neg = ix >> 31;
    ix &= 0x7fffffffu;
    const double d = x;
    if (ix <= 0x3f490fdau) return ix < 0x39800000u ? x : k_sin(d);            // |x| <= pi/4 (tiny: x)
    if (ix <= 0x407b53d1u) {                                                    // |x| <= 5pi/4
        if (ix <= 0x4016cbe3u) return neg ? -k_cos(d + p1) : k_cos(d - p1);    // |x| <= 3pi/4
        return k_sin(neg ? -(d + p2) : -(d - p2));
    }
    if (ix <= 0x40e231d5u) {                                                    // |x| <= 9pi/4
        if (ix <= 0x40afeddfu) return neg ? k_cos(d + p3) : -k_cos(d - p3);    // |x| <= 7pi/4
        return k_sin(neg ? d + p4 : d - p4);
    }
    if (ix >= 0x7f800000u) return x - x;
    if (ix >= 0x4dc90fdbu) return NAN;  // large-argument reduction: the resizer never gets there
    // medium __rem_pio2f: n = rint(x * 2/pi) by adding and subtracting 1.5 * 2^52, y = x - n pi/2 in two parts
    const double toint = 6755399441055744.0, invpio2 = 6.36619772367581382433e-01,
                 pio2_1 = 1.57079631090164184570e+00, pio2_1t = 1.58932547735281966916e-08;
    volatile double t = d * invpio2 + toint;
    const double fn = t - toint;
    const double y = d - fn * pio2_1 - fn * pio2_1t;
    switch ((int)fn & 3) {
    case 0: return k_sin(y);
    case 1: return k_cos(y);
    case 2: return k_sin(-y);
    default: return -k_cos(y);
    }
}

void resize_axis(uint32_t src, uint32_t dst, bool weights, ResizeAxis &a)
{
    const float scale = (float)src / (float)dst;
    const float fscale = scale > 1.0f ? scale : 1.0f;
    const float support = 3.0f * fscale;
    a.start.resize(dst);
    a.count.resize(dst);
    a.offset.resize(dst);
    uint64_t total = 0;
    for (uint32_t d = 0; d < dst; ++d) {
        const float center = ((float)d + 0.5f) * scale - 0.5f;
        // `as isize` / `as usize` on wasm32: saturating 32-bit conversions
        const float lo = floorf(center - support), hi = ceilf(center + support);
        int64_t s = lo <= -2147483648.0f ? INT32_MIN : lo >= 2147483648.0f ? INT32_MAX : (int64_t)lo;
        if (s < 0) s = 0;
        uint64_t e = hi <= 0.0f ? 0 : hi >= 4294967296.0f ? UINT32_MAX : (uint64_t)hi;
        e = e + 1 < src ? e + 1 : src;
        a.start[d] = (uint32_t)s;
        a.count[d] = e > (uint64_t)s ? (uint32_t)(e - (uint64_t)s) : 0;
        a.offset[d] = total;
        total += a.count[d];
    }
    if (!weights) return;
    a.w.resize(total);
    for (uint32_t d = 0; d < dst; ++d) {
        const float center = ((float)d + 0.5f) * scale - 0.5f;
        float *w = a.w.data() + a.offset[d], sum = 0.0f;
        for (uint32_t i = 0; i < a.count[d]; ++i) {
            w[i] = lanczos3(((float)(a.start[d] + i) - center) / fscale);
            sum += w[i];
        }
        if (fabsf(sum) > kEps)
            for (uint32_t i = 0; i < a.count[d]; ++i) w[i] /= sum;
    }
}

}  // namespace pixo
