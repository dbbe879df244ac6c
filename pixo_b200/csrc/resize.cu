// resize.cu — pixo's three resizers (src/resize.rs) on the GPU, byte-identical: Nearest (:299-330), Bilinear
// (:333-389) and separable Lanczos3 (:391-602).
//
// Every output channel is computed by one thread with the reference's binary32 operations in the
// reference's order, each rounded on its own (__fmul_rn / __fadd_rn; the build also passes -fmad=false):
// no FMA, no tree reduction.  f32::round is roundf (half away from zero).  Lanczos3 runs as pixo does: a
// horizontal pass into a u8 intermediate of source rows x destination columns, already rounded and
// clamped, then a vertical pass over it.  The intermediate lives in device scratch of at most
// kResizeScratch bytes: frames that fit go through together, a larger frame is done in bands of
// destination rows (and, where one row's taps alone exceed the cap, in column chunks).  The weight tables
// come from the host (resize_host.cpp): pixo's sinf is not CUDA's.
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "resize_host.hpp"

namespace pixo {

namespace {

constexpr size_t kResizeScratch = (size_t)256 << 20;
constexpr int kThreads = 128;

// The intermediate's cap in bytes.  PIXO_B200_RESIZE_SCRATCH, read on each call, replaces it (test hook: a
// small cap drives small frames through the row bands, the column chunks and the frame passes).
size_t scratch_cap()
{
    if (const char *e = getenv("PIXO_B200_RESIZE_SCRATCH")) return std::max<size_t>(1, strtoull(e, nullptr, 10));
    return kResizeScratch;
}

__device__ __forceinline__ uint8_t to_u8(float v)
{
    return (uint8_t)fminf(fmaxf(roundf(v), 0.0f), 255.0f);
}

// ((d as f32 + 0.5) * ratio - 0.5).round().max(0.0).min((src - 1) as f32) as usize
__device__ __forceinline__ uint32_t nearest_index(uint32_t d, float ratio, uint32_t src)
{
    const float f = __fadd_rn(__fmul_rn(__fadd_rn((float)d, 0.5f), ratio), -0.5f);
    return (uint32_t)fminf(fmaxf(roundf(f), 0.0f), (float)(src - 1));
}

// BPP bytes of a pixel; W > 1: the batch's frames, strides and rows allow W-byte loads and stores
template <int BPP, int W>
__device__ __forceinline__ void copy_px(uint8_t *d, const uint8_t *s)
{
    if constexpr (W == 4) *reinterpret_cast<uint32_t *>(d) = __ldg(reinterpret_cast<const uint32_t *>(s));
    else if constexpr (W == 2) *reinterpret_cast<uint16_t *>(d) = __ldg(reinterpret_cast<const uint16_t *>(s));
    else
#pragma unroll
        for (int c = 0; c < BPP; ++c) d[c] = __ldg(s + c);
}

// grid: x over destination columns, y over rows (strided), z over frames
template <int BPP, int W>
__global__ void __launch_bounds__(kThreads) k_resize_nearest(const uint8_t *__restrict__ src, size_t src_stride,
                                                             uint32_t sw, uint32_t sh, uint8_t *__restrict__ dst,
                                                             size_t dst_stride, uint32_t dw, uint32_t dh, float xr,
                                                             float yr)
{
    const uint8_t *s = src + (size_t)blockIdx.z * src_stride;
    uint8_t *d = dst + (size_t)blockIdx.z * dst_stride;
    for (uint32_t y = blockIdx.y; y < dh; y += gridDim.y) {
        const uint8_t *srow = s + (size_t)nearest_index(y, yr, sh) * sw * BPP;
        uint8_t *drow = d + (size_t)y * dw * BPP;
        for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < dw; x += gridDim.x * blockDim.x)
            copy_px<BPP, W>(drow + (size_t)x * BPP, srow + (size_t)nearest_index(x, xr, sw) * BPP);
    }
}

// src_f.floor() as usize, clamped to src - 1 (pixo would index past the row there, which f32 rounding
// allows only for a side above 2^23), and the fraction src_f - i as f32
__device__ __forceinline__ void bilinear_tap(uint32_t d, float ratio, uint32_t src, uint32_t &i0, uint32_t &i1,
                                             float &frac)
{
    const float f = __fmul_rn((float)d, ratio);
    i0 = min((uint32_t)floorf(f), src - 1);
    i1 = min(i0 + 1, src - 1);
    frac = __fadd_rn(f, -(float)i0);
}

template <int BPP>
__global__ void __launch_bounds__(kThreads) k_resize_bilinear(const uint8_t *__restrict__ src, size_t src_stride,
                                                              uint32_t sw, uint32_t sh, uint8_t *__restrict__ dst,
                                                              size_t dst_stride, uint32_t dw, uint32_t dh, float xr,
                                                              float yr)
{
    const uint8_t *s = src + (size_t)blockIdx.z * src_stride;
    uint8_t *d = dst + (size_t)blockIdx.z * dst_stride;
    for (uint32_t y = blockIdx.y; y < dh; y += gridDim.y) {
        uint32_t y0, y1;
        float yf;
        bilinear_tap(y, yr, sh, y0, y1, yf);
        const float yf1 = __fadd_rn(1.0f, -yf);
        const uint8_t *r0 = s + (size_t)y0 * sw * BPP, *r1 = s + (size_t)y1 * sw * BPP;
        uint8_t *drow = d + (size_t)y * dw * BPP;
        for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < dw; x += gridDim.x * blockDim.x) {
            uint32_t x0, x1;
            float xf;
            bilinear_tap(x, xr, sw, x0, x1, xf);
            const float xf1 = __fadd_rn(1.0f, -xf);
            const uint8_t *p00 = r0 + (size_t)x0 * BPP, *p01 = r0 + (size_t)x1 * BPP;
            const uint8_t *p10 = r1 + (size_t)x0 * BPP, *p11 = r1 + (size_t)x1 * BPP;
#pragma unroll
            for (int c = 0; c < BPP; ++c) {
                const float top = __fadd_rn(__fmul_rn((float)__ldg(p00 + c), xf1), __fmul_rn((float)__ldg(p01 + c), xf));
                const float bot = __fadd_rn(__fmul_rn((float)__ldg(p10 + c), xf1), __fmul_rn((float)__ldg(p11 + c), xf));
                drow[(size_t)x * BPP + c] = to_u8(__fadd_rn(__fmul_rn(top, yf1), __fmul_rn(bot, yf)));
            }
        }
    }
}

// Lanczos3 horizontal pass: source rows r0..r1-1, destination columns x0..x0+cw-1 -> the u8 intermediate
// (row r at tmp + (r - r0) * cw * BPP); one sequential sum per channel in tap order
template <int BPP>
__global__ void __launch_bounds__(kThreads) k_resize_lanczos_h(const uint8_t *__restrict__ src, size_t src_stride,
                                                               uint32_t sw, uint32_t r0, uint32_t r1, uint32_t x0,
                                                               uint32_t cw, const uint32_t *__restrict__ start,
                                                               const uint32_t *__restrict__ count,
                                                               const uint64_t *__restrict__ offset,
                                                               const float *__restrict__ weight,
                                                               uint8_t *__restrict__ tmp, size_t tmp_stride)
{
    const uint8_t *s = src + (size_t)blockIdx.z * src_stride;
    uint8_t *t = tmp + (size_t)blockIdx.z * tmp_stride;
    for (uint32_t r = r0 + blockIdx.y; r < r1; r += gridDim.y) {
        const uint8_t *row = s + (size_t)r * sw * BPP;
        uint8_t *trow = t + (size_t)(r - r0) * cw * BPP;
        for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cw; j += gridDim.x * blockDim.x) {
            const uint32_t x = x0 + j, n = __ldg(count + x);
            const uint8_t *p = row + (size_t)__ldg(start + x) * BPP;
            const float *w = weight + __ldg(offset + x);
            float acc[BPP];
#pragma unroll
            for (int c = 0; c < BPP; ++c) acc[c] = 0.0f;
            for (uint32_t i = 0; i < n; ++i, p += BPP) {
                const float wi = __ldg(w + i);
#pragma unroll
                for (int c = 0; c < BPP; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn((float)__ldg(p + c), wi));
            }
#pragma unroll
            for (int c = 0; c < BPP; ++c) trow[(size_t)j * BPP + c] = to_u8(acc[c]);
        }
    }
}

// Lanczos3 vertical pass: destination rows y0..y1-1, columns x0..x0+cw-1, from the intermediate that holds
// source rows from rs on
template <int BPP>
__global__ void __launch_bounds__(kThreads) k_resize_lanczos_v(const uint8_t *__restrict__ tmp, size_t tmp_stride,
                                                               uint32_t rs, uint32_t cw, uint32_t y0, uint32_t y1,
                                                               uint32_t x0, const uint32_t *__restrict__ start,
                                                               const uint32_t *__restrict__ count,
                                                               const uint64_t *__restrict__ offset,
                                                               const float *__restrict__ weight,
                                                               uint8_t *__restrict__ dst, size_t dst_stride,
                                                               uint32_t dw)
{
    const uint8_t *t = tmp + (size_t)blockIdx.z * tmp_stride;
    uint8_t *d = dst + (size_t)blockIdx.z * dst_stride;
    const size_t pitch = (size_t)cw * BPP;
    for (uint32_t y = y0 + blockIdx.y; y < y1; y += gridDim.y) {
        const uint32_t n = __ldg(count + y);
        const float *w = weight + __ldg(offset + y);
        const uint8_t *col = t + (n ? (size_t)(__ldg(start + y) - rs) * pitch : 0);
        uint8_t *drow = d + (size_t)y * dw * BPP + (size_t)x0 * BPP;
        for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cw; j += gridDim.x * blockDim.x) {
            const uint8_t *p = col + (size_t)j * BPP;
            float acc[BPP];
#pragma unroll
            for (int c = 0; c < BPP; ++c) acc[c] = 0.0f;
            for (uint32_t i = 0; i < n; ++i, p += pitch) {
                const float wi = __ldg(w + i);
#pragma unroll
                for (int c = 0; c < BPP; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn((float)__ldg(p + c), wi));
            }
#pragma unroll
            for (int c = 0; c < BPP; ++c) drow[(size_t)j * BPP + c] = to_u8(acc[c]);
        }
    }
}

// x blocks over cols columns, y blocks over rows (a grid-stride loop covers the rest), z = frames
dim3 grid_for(const pixo_b200_ctx *ctx, uint32_t cols, uint32_t rows, uint32_t frames)
{
    const uint32_t gx = std::min<uint32_t>((cols + kThreads - 1) / kThreads, 256);
    const uint64_t want = (uint64_t)std::max(ctx->sm_count, 1) * 32;
    const uint64_t gy = std::min<uint64_t>({rows, 65535, std::max<uint64_t>(1, want / ((uint64_t)gx * frames))});
    return dim3(gx, (uint32_t)gy, frames);
}

template <int BPP>
int launch_simple(pixo_b200_ctx *ctx, const uint8_t *src, size_t src_stride, uint32_t n, uint32_t sw, uint32_t sh,
                  uint8_t *dst, size_t dst_stride, uint32_t dw, uint32_t dh, uint32_t alg)
{
    const float xn = (float)sw / (float)dw, yn = (float)sh / (float)dh;
    const float xb = dw > 1 ? (float)(sw - 1) / (float)(dw - 1) : 0.0f;
    const float yb = dh > 1 ? (float)(sh - 1) / (float)(dh - 1) : 0.0f;
    // pixel-wide loads when every frame's base, every row and every pixel are aligned to them
    const uintptr_t al = (uintptr_t)src | (uintptr_t)dst | (n > 1 ? (src_stride | dst_stride) : 0);
    const bool wide = (BPP == 2 || BPP == 4) && al % BPP == 0;
    const auto kern = alg == 1 ? k_resize_bilinear<BPP>
                      : wide   ? k_resize_nearest<BPP, (BPP == 2 || BPP == 4) ? BPP : 1>
                               : k_resize_nearest<BPP, 1>;
    const float xr = alg == 1 ? xb : xn, yr = alg == 1 ? yb : yn;
    for (uint32_t f0 = 0; f0 < n; f0 += 65535) {
        const uint32_t nf = std::min<uint32_t>(n - f0, 65535);
        const uint8_t *s = src + (size_t)f0 * src_stride;
        uint8_t *d = dst + (size_t)f0 * dst_stride;
        PIXO_TRY(launch(ctx, kern, grid_for(ctx, dw, dh, nf), kThreads, 0, s, src_stride, sw, sh, d, dst_stride, dw, dh,
                        xr, yr));
    }
    return 0;
}

// one piece of Lanczos3 work: destination rows y0..y1-1 and columns x0..x0+cw-1, which need source rows
// rs..re-1 of the intermediate
struct Band {
    uint32_t y0, y1, rs, re, x0, cw;
};

std::vector<Band> lanczos_bands(const ResizeAxis &v, uint32_t sh, uint32_t dw, uint32_t dh, int bpp, size_t cap)
{
    std::vector<Band> bands;
    const size_t row = (size_t)dw * bpp;
    if ((size_t)sh * row <= cap) {
        bands.push_back({0, dh, 0, sh, 0, dw});
        return bands;
    }
    auto end = [&](uint32_t y) { return v.start[y] + v.count[y]; };
    for (uint32_t y0 = 0; y0 < dh;) {
        uint32_t rs = v.count[y0] ? v.start[y0] : UINT32_MAX, re = v.count[y0] ? end(y0) : 0, y1 = y0 + 1;
        const size_t rows1 = re > rs ? re - rs : 0;
        if (rows1 * row > cap) {  // one destination row's taps alone: split its columns
            const uint32_t cw = (uint32_t)std::max<size_t>(1, cap / (rows1 * bpp));
            for (uint32_t x0 = 0; x0 < dw; x0 += cw) bands.push_back({y0, y1, rs, re, x0, std::min(cw, dw - x0)});
            y0 = y1;
            continue;
        }
        for (; y1 < dh; ++y1) {
            if (!v.count[y1]) continue;
            const uint32_t nrs = std::min(rs, v.start[y1]), nre = std::max(re, end(y1));
            if ((size_t)(nre - nrs) * row > cap) break;
            rs = nrs;
            re = nre;
        }
        if (re <= rs) rs = re = 0;  // rows without taps read nothing
        bands.push_back({y0, y1, rs, re, 0, dw});
        y0 = y1;
    }
    return bands;
}

template <int BPP>
int launch_lanczos(pixo_b200_ctx *ctx, const uint8_t *src, size_t src_stride, uint32_t n, uint32_t sw, uint32_t sh,
                   uint8_t *dst, size_t dst_stride, uint32_t dw, uint32_t dh)
{
    ResizeAxis h, v;
    resize_axis(sw, dw, true, h);
    resize_axis(sh, dh, true, v);
    // tables: h start/count, v start/count (u32), h/v offsets (u64), h/v weights (f32), laid out alike in the
    // pinned upload buffer (H) and on the device (T)
    struct Tables {
        uint32_t *hs, *hc, *vs, *vc;
        uint64_t *ho, *vo;
        float *hw, *vw;
        size_t bytes;
    } T, H;
    auto tables = [&](Tables &t) {
        return [&](Layout &L) {
            t.hs = L.take<uint32_t>(dw), t.hc = L.take<uint32_t>(dw), t.vs = L.take<uint32_t>(dh), t.vc = L.take<uint32_t>(dh);
            t.ho = L.take<uint64_t>(dw), t.vo = L.take<uint64_t>(dh);
            t.hw = L.take<float>(h.w.size() + 1), t.vw = L.take<float>(v.w.size() + 1);
            t.bytes = L.end();
        };
    };
    PIXO_TRY(bind(ctx, ctx->d_resize, tables(T)));
    // One copy from one of the context's two pinned buffers, in turn.  A copy from the pageable vectors
    // lets the driver wait for the stream before the call returns (it does for some MB of tables); a
    // pinned one is only queued.  A buffer is rewritten once the copy out of it, two uploads back, has run.
    const int slot = (int)(ctx->resize_uploads % 2);
    PIXO_CUDA(ctx, cudaEventSynchronize(ctx->resize_events[slot]));
    PIXO_TRY(bind(ctx, ctx->h_resize[slot], tables(H)));
    const struct { void *dst; const void *src; size_t bytes; } up[] = {
        {H.hs, h.start.data(), 4 * (size_t)dw}, {H.hc, h.count.data(), 4 * (size_t)dw},
        {H.vs, v.start.data(), 4 * (size_t)dh}, {H.vc, v.count.data(), 4 * (size_t)dh},
        {H.ho, h.offset.data(), 8 * (size_t)dw}, {H.vo, v.offset.data(), 8 * (size_t)dh},
        {H.hw, h.w.data(), 4 * h.w.size()},      {H.vw, v.w.data(), 4 * v.w.size()}};
    for (const auto &u : up)
        if (u.bytes) memcpy(u.dst, u.src, u.bytes);
    PIXO_CUDA(ctx, cudaMemcpyAsync(T.hs, H.hs, T.bytes, cudaMemcpyHostToDevice, ctx->stream));
    PIXO_CUDA(ctx, cudaEventRecord(ctx->resize_events[slot], ctx->stream));
    ctx->resize_uploads++;
    const uint32_t *hs = T.hs, *hc = T.hc, *vs = T.vs, *vc = T.vc;
    const uint64_t *ho = T.ho, *vo = T.vo;
    const float *hw = T.hw, *vw = T.vw;

    const size_t cap = scratch_cap();
    const std::vector<Band> bands = lanczos_bands(v, sh, dw, dh, BPP, cap);
    size_t most = 1;  // intermediate bytes of the largest band
    for (const Band &b : bands) most = std::max(most, (size_t)(b.re - b.rs) * b.cw * BPP);
    // frames per pass: as many whole intermediates as the cap holds (only when one band covers the frame)
    const uint32_t per_pass = bands.size() == 1 ? (uint32_t)std::min<size_t>({n, 65535, std::max<size_t>(1, cap / most)}) : 1;
    const size_t tstride = Layout::round(most);
    PIXO_TRY(ctx->d_resize_tmp.ensure(ctx, tstride * per_pass));
    uint8_t *tmp = reinterpret_cast<uint8_t *>(ctx->d_resize_tmp.ptr);
    for (uint32_t f0 = 0; f0 < n; f0 += per_pass) {
        const uint32_t nf = std::min(per_pass, n - f0);
        const uint8_t *s = src + (size_t)f0 * src_stride;
        uint8_t *d = dst + (size_t)f0 * dst_stride;
        for (const Band &b : bands) {
            if (b.re > b.rs)
                PIXO_TRY(launch(ctx, k_resize_lanczos_h<BPP>, grid_for(ctx, b.cw, b.re - b.rs, nf), kThreads, 0, s,
                                src_stride, sw, b.rs, b.re, b.x0, b.cw, hs, hc, ho, hw, tmp, tstride));
            PIXO_TRY(launch(ctx, k_resize_lanczos_v<BPP>, grid_for(ctx, b.cw, b.y1 - b.y0, nf), kThreads, 0, tmp,
                            tstride, b.rs, b.cw, b.y0, b.y1, b.x0, vs, vc, vo, vw, d, dst_stride, dw));
        }
    }
    return 0;
}

template <int BPP>
int launch_bpp(pixo_b200_ctx *ctx, const uint8_t *src, size_t src_stride, uint32_t n, uint32_t sw, uint32_t sh,
               uint8_t *dst, size_t dst_stride, uint32_t dw, uint32_t dh, uint32_t alg)
{
    if (alg == 2) return launch_lanczos<BPP>(ctx, src, src_stride, n, sw, sh, dst, dst_stride, dw, dh);
    return launch_simple<BPP>(ctx, src, src_stride, n, sw, sh, dst, dst_stride, dw, dh, alg);
}

}  // namespace

int launch_resize(pixo_b200_ctx *ctx, const uint8_t *d_src, size_t src_stride, uint32_t n, uint32_t sw, uint32_t sh,
                  uint32_t dw, uint32_t dh, uint32_t bpp, uint32_t algorithm, uint8_t *d_dst, size_t dst_stride)
{
    switch (bpp) {
    case 1: return launch_bpp<1>(ctx, d_src, src_stride, n, sw, sh, d_dst, dst_stride, dw, dh, algorithm);
    case 2: return launch_bpp<2>(ctx, d_src, src_stride, n, sw, sh, d_dst, dst_stride, dw, dh, algorithm);
    case 3: return launch_bpp<3>(ctx, d_src, src_stride, n, sw, sh, d_dst, dst_stride, dw, dh, algorithm);
    default: return launch_bpp<4>(ctx, d_src, src_stride, n, sw, sh, d_dst, dst_stride, dw, dh, algorithm);
    }
}

}  // namespace pixo
