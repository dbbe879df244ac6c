/*
 * resize.c — plain C restatement of pixo's resizers (src/resize.rs @ 437bf63) for the tests: validation
 * (resize_impl :195-296), Nearest (:299-330), Bilinear (:333-389) and separable Lanczos3 (:391-602), all
 * in single-rounding binary32 as pixo's wasm build runs them (no FMA: build with -ffp-contract=off).
 *
 * lanczos_kernel calls f32::sin, which on that build is the Rust libm port of musl's sinf: a polynomial in
 * double precision, rounded once to f32 (not correctly rounded).  rz_sinf restates that function (the
 * |x| <= 9pi/4 quadrant branches, the __sindf / __cosdf kernels and the medium __rem_pio2f reduction); it
 * is checked against the wasm's own sinf by tests/test_resize.py (tests/golden/resize/sinf.npy) and
 * exhaustively over [-3pi, 3pi] by oracle/wasm_ref/resize_ref.c.  Test infrastructure only.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- sinf --------------------------------------------------------------------------------- */
static const double kS1 = -0x15555554cbac77.0p-55, kS2 = 0x111110896efbb2.0p-59,
                    kS3 = -0x1a00f9e2cae774.0p-65, kS4 = 0x16cd878c3b46a7.0p-71;
static const double kC0 = -0x1ffffffd0c5e81.0p-54, kC1 = 0x155553e1053a42.0p-57,
                    kC2 = -0x16c087e80f1e27.0p-62, kC3 = 0x199342e0ee5069.0p-68;
static const double kPio2 = 1.57079632679489661923;  /* M_PI_2 as a double */

/* sin on |x| <= pi/4, degree-9 odd polynomial, one rounding to f32 at the end */
static float sindf(double x)
{
    double z = x * x, w = z * z, r = kS3 + z * kS4, s = z * x;
    return (float)((x + s * (kS1 + z * kS2)) + s * w * r);
}

/* cos on |x| <= pi/4 */
static float cosdf(double x)
{
    double z = x * x, w = z * z, r = kC2 + z * kC3;
    return (float)(((1.0 + z * kC0) + w * kC1) + (w * z) * r);
}

float rz_sinf(float x)
{
    const double s1 = 1 * kPio2, s2 = 2 * kPio2, s3 = 3 * kPio2, s4 = 4 * kPio2;
    uint32_t ix;
    memcpy(&ix, &x, 4);
    const int sign = (int)(ix >> 31);
    ix &= 0x7fffffffu;
    const double xd = (double)x;
    if (ix <= 0x3f490fdau) {                 /* |x| <= ~pi/4 */
        if (ix < 0x39800000u) return x;      /* |x| < 2^-12 */
        return sindf(xd);
    }
    if (ix <= 0x407b53d1u) {                 /* |x| <= ~5pi/4 */
        if (ix <= 0x4016cbe3u)               /* |x| <= ~3pi/4 */
            return sign ? -cosdf(xd + s1) : cosdf(xd - s1);
        return sindf(sign ? -(xd + s2) : -(xd - s2));
    }
    if (ix <= 0x40e231d5u) {                 /* |x| <= ~9pi/4 */
        if (ix <= 0x40afeddfu)               /* |x| <= ~7pi/4 */
            return sign ? cosdf(xd + s3) : -cosdf(xd - s3);
        return sindf(sign ? xd + s4 : xd - s4);
    }
    if (ix >= 0x7f800000u) return x - x;
    if (ix >= 0x4dc90fdbu) return NAN;       /* large arguments: never reached by the resizer */
    /* medium __rem_pio2f: n = rint(x * 2/pi) by the 1.5 * 2^52 trick, y = x - n * pi/2 in two parts */
    const double toint = 1.5 / 2.220446049250313080847e-16, invpio2 = 6.36619772367581382433e-01,
                 pio2_1 = 1.57079631090164184570e+00, pio2_1t = 1.58932547735281966916e-08;
    volatile double t = xd * invpio2 + toint;
    const double fn = t - toint;
    const int n = (int)fn;
    const double y = xd - fn * pio2_1 - fn * pio2_1t;
    switch (n & 3) {
    case 0: return sindf(y);
    case 1: return cosdf(y);
    case 2: return sindf(-y);
    default: return -cosdf(y);
    }
}

void rz_sinf_many(const float *x, float *y, size_t n)
{
    for (size_t i = 0; i < n; i++) y[i] = rz_sinf(x[i]);
}

/* ---- Lanczos3 contributions (precompute_contributions :416-456) --------------------------- */
static float lanczos_kernel(float x)
{
    const float a = 3.0f, pi = 3.14159265358979323846f, eps = 1.1920928955078125e-7f;
    if (fabsf(x) < eps) return 1.0f;
    if (fabsf(x) >= a) return 0.0f;
    const float pi_x = pi * x, pi_x_a = pi * x / a;
    return (a * rz_sinf(pi_x) * rz_sinf(pi_x_a)) / (pi_x * pi_x_a);
}

/* the range of source indices of destination index d: start and count (end - start) */
static void contrib_range(uint32_t src, uint32_t dst, uint32_t d, float scale, float support, uint32_t *start,
                          uint32_t *count)
{
    const float center = ((float)d + 0.5f) * scale - 0.5f;
    const float lo = floorf(center - support), hi = ceilf(center + support);
    /* `as isize` / `as usize` on wasm32 saturate at the 32-bit limits */
    int64_t s = lo <= -2147483648.0f ? INT32_MIN : lo >= 2147483648.0f ? INT32_MAX : (int64_t)lo;
    if (s < 0) s = 0;
    uint64_t e = hi <= 0.0f ? 0 : hi >= 4294967296.0f ? UINT32_MAX : (uint64_t)hi;
    e = e + 1 < src ? e + 1 : src;
    *start = (uint32_t)s;
    *count = e > (uint64_t)s ? (uint32_t)(e - (uint64_t)s) : 0;
}

/* start/count/offset per destination index and the concatenated normalised weights.  Returns the number
 * of weights; with weights NULL only the ranges (and the total) are produced. */
size_t rz_contrib(uint32_t src, uint32_t dst, uint32_t *start, uint32_t *count, uint64_t *offset, float *weights)
{
    const float scale = (float)src / (float)dst;
    const float fscale = scale > 1.0f ? scale : 1.0f;
    const float support = 3.0f * fscale;
    size_t total = 0;
    for (uint32_t d = 0; d < dst; d++) {
        uint32_t s, c;
        contrib_range(src, dst, d, scale, support, &s, &c);
        if (start) start[d] = s;
        if (count) count[d] = c;
        if (offset) offset[d] = total;
        if (weights) {
            const float center = ((float)d + 0.5f) * scale - 0.5f;
            float *w = weights + total, sum = 0.0f;
            for (uint32_t i = 0; i < c; i++) {
                w[i] = lanczos_kernel(((float)(s + i) - center) / fscale);
                sum += w[i];
            }
            if (fabsf(sum) > 1.1920928955078125e-7f)
                for (uint32_t i = 0; i < c; i++) w[i] /= sum;
        }
        total += c;
    }
    return total;
}

/* ---- the resizers -------------------------------------------------------------------------- */
static uint8_t to_u8(float v)
{
    v = roundf(v);                       /* half away from zero, as f32::round */
    return (uint8_t)(v < 0.0f ? 0.0f : v > 255.0f ? 255.0f : v);
}

static void nearest(const uint8_t *in, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, int bpp, uint8_t *out)
{
    const float xr = (float)sw / (float)dw, yr = (float)sh / (float)dh;
    for (uint32_t y = 0; y < dh; y++) {
        float fy = fminf(fmaxf(roundf(((float)y + 0.5f) * yr - 0.5f), 0.0f), (float)(sh - 1));
        const size_t sy = (size_t)fy;
        for (uint32_t x = 0; x < dw; x++) {
            float fx = fminf(fmaxf(roundf(((float)x + 0.5f) * xr - 0.5f), 0.0f), (float)(sw - 1));
            const size_t sx = (size_t)fx;
            memcpy(out + ((size_t)y * dw + x) * bpp, in + (sy * sw + sx) * bpp, (size_t)bpp);
        }
    }
}

/* pixo indexes out of bounds (and panics) when f32 rounding puts floor(d * ratio) at src; that needs a
 * source side above 2^23 and is clamped here, as in the library */
static void bilinear(const uint8_t *in, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, int bpp, uint8_t *out)
{
    const float xr = dw > 1 ? (float)(sw - 1) / (float)(dw - 1) : 0.0f;
    const float yr = dh > 1 ? (float)(sh - 1) / (float)(dh - 1) : 0.0f;
    for (uint32_t y = 0; y < dh; y++) {
        const float syf = (float)y * yr;
        size_t y0 = (size_t)floorf(syf);
        if (y0 > sh - 1) y0 = sh - 1;
        const size_t y1 = y0 + 1 < sh ? y0 + 1 : sh - 1;
        const float yf = syf - (float)y0;
        for (uint32_t x = 0; x < dw; x++) {
            const float sxf = (float)x * xr;
            size_t x0 = (size_t)floorf(sxf);
            if (x0 > sw - 1) x0 = sw - 1;
            const size_t x1 = x0 + 1 < sw ? x0 + 1 : sw - 1;
            const float xf = sxf - (float)x0;
            const uint8_t *p00 = in + (y0 * sw + x0) * bpp, *p01 = in + (y0 * sw + x1) * bpp;
            const uint8_t *p10 = in + (y1 * sw + x0) * bpp, *p11 = in + (y1 * sw + x1) * bpp;
            uint8_t *o = out + ((size_t)y * dw + x) * bpp;
            for (int c = 0; c < bpp; c++) {
                const float top = (float)p00[c] * (1.0f - xf) + (float)p01[c] * xf;
                const float bottom = (float)p10[c] * (1.0f - xf) + (float)p11[c] * xf;
                o[c] = to_u8(top * (1.0f - yf) + bottom * yf);
            }
        }
    }
}

static int lanczos3(const uint8_t *in, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, int bpp, uint8_t *out)
{
    uint32_t *hs = malloc(sizeof(uint32_t) * dw * 2), *vs = malloc(sizeof(uint32_t) * dh * 2);
    uint64_t *ho = malloc(8 * (size_t)dw), *vo = malloc(8 * (size_t)dh);
    if (!hs || !vs || !ho || !vo) return -1;
    const size_t nh = rz_contrib(sw, dw, hs, hs + dw, ho, NULL), nv = rz_contrib(sh, dh, vs, vs + dh, vo, NULL);
    float *hw = malloc(sizeof(float) * (nh ? nh : 1)), *vw = malloc(sizeof(float) * (nv ? nv : 1));
    uint8_t *tmp = malloc((size_t)sh * dw * bpp);
    if (!hw || !vw || !tmp) return -1;
    rz_contrib(sw, dw, NULL, NULL, NULL, hw);
    rz_contrib(sh, dh, NULL, NULL, NULL, vw);
    for (uint32_t y = 0; y < sh; y++) {                   /* horizontal pass: u8 intermediate */
        const uint8_t *row = in + (size_t)y * sw * bpp;
        for (uint32_t x = 0; x < dw; x++) {
            float acc[4] = {0, 0, 0, 0};
            for (uint32_t i = 0; i < hs[dw + x]; i++) {
                const float w = hw[ho[x] + i];
                const uint8_t *p = row + (size_t)(hs[x] + i) * bpp;
                for (int c = 0; c < bpp; c++) acc[c] += (float)p[c] * w;
            }
            for (int c = 0; c < bpp; c++) tmp[((size_t)y * dw + x) * bpp + c] = to_u8(acc[c]);
        }
    }
    const size_t rs = (size_t)dw * bpp;
    for (uint32_t y = 0; y < dh; y++) {                   /* vertical pass */
        for (uint32_t x = 0; x < dw; x++) {
            float acc[4] = {0, 0, 0, 0};
            for (uint32_t i = 0; i < vs[dh + y]; i++) {
                const float w = vw[vo[y] + i];
                const uint8_t *p = tmp + (size_t)(vs[y] + i) * rs + (size_t)x * bpp;
                for (int c = 0; c < bpp; c++) acc[c] += (float)p[c] * w;
            }
            for (int c = 0; c < bpp; c++) out[(size_t)y * rs + (size_t)x * bpp + c] = to_u8(acc[c]);
        }
    }
    free(hs); free(vs); free(ho); free(vo); free(hw); free(vw); free(tmp);
    return 0;
}

/* Status codes as include/pixo_b200.h numbers them: 2 InvalidDimensions, 3 ImageTooLarge, 5
 * InvalidDataLength, 7 unknown colour type or algorithm (the wasm binding's check, made first), 11 no
 * memory.  out: dw*dh*bpp bytes. */
int rz_resize(const uint8_t *in, size_t len, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, uint32_t ct,
              uint32_t alg, uint8_t *out)
{
    if (ct > 3 || alg > 2) return 7;
    if (sw == 0 || sh == 0 || dw == 0 || dh == 0) return 2;
    const uint32_t mx = 1u << 24;
    if (sw > mx || sh > mx || dw > mx || dh > mx) return 3;
    const int bpp = (int)ct + 1;
    if (len != (size_t)sw * sh * bpp) return 5;
    if (alg == 0) nearest(in, sw, sh, dw, dh, bpp, out);
    else if (alg == 1) bilinear(in, sw, sh, dw, dh, bpp, out);
    else if (lanczos3(in, sw, sh, dw, dh, bpp, out)) return 11;
    return 0;
}
