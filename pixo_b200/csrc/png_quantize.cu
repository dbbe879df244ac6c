// png_quantize.cu — pixo's lossy PNG path: palette quantisation ahead of the PNG filter.
//
// Restates
//   encode_into's quantisation branch     src/png/mod.rs:469-511
//   should_quantize_auto                  src/png/mod.rs:1708-1762  (sample stride max(N/20000, 1))
//   quantize_image                        src/png/mod.rs:1505-1701  (histogram stride max(N/50000, 1))
//   refine_palette_kmeans                 src/png/mod.rs:1346-1390
//   perceptual_distance_sq / nearest_palette_index / PaletteLut   src/png/mod.rs:1405-1500
// Median cut and maybe_trim_transparency are host work on <= 8192 colours (png_host.cpp).
//
// Design (H100):
//   k_quant_sample: both of pixo's strided sample sets of every image as 64-bit keys
//     (image << 33 | set << 32 | r<<24|g<<16|b<<8|a), sorted by CUB's radix sort and run-length counted
//     by CUB's run-length encoder, so the host receives only each image's distinct colours and counts.
//   k_quant_kmeans / k_quant_update: the two k-means passes.  One thread per histogram colour, the palette
//     in shared memory, first minimum wins; the sums are u64 and integer, so the order of the atomics
//     does not matter.
//   k_quant_lut: PaletteLut::new, one thread per 6-6-6 cell, palette in shared memory.
//   k_quant_map: the plain map and the early-out map (exact binary search over the key-sorted palette).
//   k_quant_dither: Floyd-Steinberg as a wavefront (see the kernel).
//   Pixels that need a full nearest-entry search (alpha < 255, early-out misses) are searched by the
//   whole warp: the 32 lanes split the entries and a min-reduction of (distance << 8 | index) gives the
//   first minimum.
// The index rows then go through png_filter.cu's filter kernels with bpp 1.
#include <string.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <vector>

#include "common.cuh"
#include "png_host.hpp"

namespace pixo {
namespace {

constexpr int Q_THREADS = 256;
constexpr uint32_t DECISION_CAP = 20000, HISTOGRAM_CAP = 50000, MAX_HIST_COLORS = 8192;
constexpr uint32_t LUT_CELLS = 64 * 64 * 64;
constexpr uint32_t SAMPLE_CHUNK = 64;            // images per sort (6 bits of the key)
constexpr int DITHER_WARPS = 4;                  // warps per CTA of k_quant_dither
constexpr uint32_t SPIN_LIMIT = 1u << 22;        // polls (with back-off) before a wait is a fault
constexpr size_t QUANT_PASS = 4096;              // quantised images per pass of k-means, tables, map and filter

__device__ __forceinline__ uint32_t redmean(uint32_t c, uint32_t p)
{
    // perceptual_distance_sq on keys r<<24|g<<16|b<<8|a
    const int r1 = c >> 24, g1 = (c >> 16) & 255, b1 = (c >> 8) & 255, a1 = c & 255;
    const int r2 = p >> 24, g2 = (p >> 16) & 255, b2 = (p >> 8) & 255, a2 = p & 255;
    const int dr = r1 - r2, dg = g1 - g2, db = b1 - b2, da = a1 - a2;
    const int rm = (r1 + r2) >> 1;
    const int d = ((512 + rm) * dr * dr + 1024 * dg * dg + (767 - rm) * db * db) >> 8;
    return (uint32_t)(d + da * da);
}

// first nearest entry of pal[0..n) to c, searched by one thread
__device__ __forceinline__ uint32_t nearest_seq(const uint32_t *pal, uint32_t n, uint32_t c)
{
    uint32_t best = 0xFFFFFFFFu;
    for (uint32_t i = 0; i < n; ++i) best = min(best, (redmean(c, pal[i]) << 8) | i);
    return best & 255u;
}

// Warp-cooperative nearest search for every lane in `need` (all 32 lanes call it): each lane's colour
// `c` is broadcast in turn, the lanes split the entries and reduce (distance << 8 | index).
__device__ __forceinline__ uint32_t nearest_warp(const uint32_t *pal, uint32_t n, uint32_t c, unsigned need,
                                                 uint32_t lane, uint32_t mine)
{
    while (need) {
        const int l = __ffs(need) - 1;
        need &= need - 1;
        const uint32_t q = __shfl_sync(0xffffffffu, c, l);
        uint32_t best = 0xFFFFFFFFu;
        for (uint32_t i = lane; i < n; i += 32) best = min(best, (redmean(q, pal[i]) << 8) | i);
        best = __reduce_min_sync(0xffffffffu, best);
        if ((int)lane == l) mine = best & 255u;
    }
    return mine;
}

__device__ __forceinline__ uint32_t pixel_key(const uint8_t *src, uint64_t p, uint32_t bpp)
{
    if (bpp == 4 && (reinterpret_cast<uintptr_t>(src) & 3) == 0) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(src) + p);
        return __byte_perm(v, 0, 0x0123);   // r g b a bytes -> r<<24|g<<16|b<<8|a
    }
    const uint8_t *q = src + p * bpp;
    return ((uint32_t)__ldg(q) << 24) | ((uint32_t)__ldg(q + 1) << 16) | ((uint32_t)__ldg(q + 2) << 8) |
           (bpp == 4 ? (uint32_t)__ldg(q + 3) : 255u);
}

// ---- k_quant_sample --------------------------------------------------------------------------------
struct SampleParams {
    const uint8_t *data;
    size_t in_stride;
    uint32_t n_images, bpp;
    uint64_t nd, nh, sd, sh;     // samples and strides of the decision and histogram sets
    unsigned long long *keys;
};

__global__ void __launch_bounds__(Q_THREADS) k_quant_sample(SampleParams P)
{
    const uint64_t per = P.nd + P.nh, total = per * P.n_images;
    for (uint64_t t = (uint64_t)blockIdx.x * Q_THREADS + threadIdx.x; t < total; t += (uint64_t)gridDim.x * Q_THREADS) {
        const uint64_t img = t / per, s = t - img * per;
        const bool hist = s >= P.nd;
        const uint64_t p = hist ? (s - P.nd) * P.sh : s * P.sd;
        const uint32_t key = pixel_key(P.data + img * P.in_stride, p, P.bpp);
        P.keys[t] = (img << 33) | ((unsigned long long)hist << 32) | key;
    }
}

// ---- k-means ---------------------------------------------------------------------------------------
struct KmeansJob {
    const uint32_t *colors;         // keys, key order
    const uint32_t *counts;
    uint32_t ncolors, npal;
    uint32_t *pal;                  // npal keys, updated in place
    unsigned long long *acc;        // 256 x 5 (r, g, b, a, count), zeroed before each pass
};

__global__ void __launch_bounds__(Q_THREADS) k_quant_kmeans(const KmeansJob *jobs)
{
    __shared__ uint32_t pal[256];
    __shared__ unsigned long long acc[256 * 5];
    const KmeansJob &J = jobs[blockIdx.y];
    const uint32_t n = J.npal;
    if (blockIdx.x * Q_THREADS >= J.ncolors) return;
    for (uint32_t i = threadIdx.x; i < n; i += Q_THREADS) pal[i] = J.pal[i];
    for (uint32_t i = threadIdx.x; i < 256 * 5; i += Q_THREADS) acc[i] = 0;
    __syncthreads();
    const uint32_t c = blockIdx.x * Q_THREADS + threadIdx.x;
    if (c < J.ncolors) {
        const uint32_t key = J.colors[c], cnt = J.counts[c];
        const uint32_t b = nearest_seq(pal, n, key);
        atomicAdd(&acc[b * 5 + 0], (unsigned long long)(key >> 24) * cnt);
        atomicAdd(&acc[b * 5 + 1], (unsigned long long)((key >> 16) & 255) * cnt);
        atomicAdd(&acc[b * 5 + 2], (unsigned long long)((key >> 8) & 255) * cnt);
        atomicAdd(&acc[b * 5 + 3], (unsigned long long)(key & 255) * cnt);
        atomicAdd(&acc[b * 5 + 4], (unsigned long long)cnt);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n * 5; i += Q_THREADS)
        if (acc[i]) atomicAdd(J.acc + i, acc[i]);
}

// centroid update (an entry with no members keeps its colour), then zero the sums for the next pass
__global__ void __launch_bounds__(256) k_quant_update(const KmeansJob *jobs)
{
    const KmeansJob &J = jobs[blockIdx.x];
    const uint32_t i = threadIdx.x;
    if (i >= J.npal) return;
    unsigned long long *a = J.acc + i * 5;
    const unsigned long long t = a[4];
    if (t) J.pal[i] = ((uint32_t)(a[0] / t) << 24) | ((uint32_t)(a[1] / t) << 16) | ((uint32_t)(a[2] / t) << 8) |
                      (uint32_t)(a[3] / t);
    for (int k = 0; k < 5; ++k) a[k] = 0;
}

// ---- k_quant_lut -----------------------------------------------------------------------------------
struct LutJob {
    const uint32_t *pal;
    uint32_t npal;
    uint8_t *lut;
};

__global__ void __launch_bounds__(Q_THREADS) k_quant_lut(const LutJob *jobs)
{
    __shared__ uint32_t pal[256];
    const LutJob &J = jobs[blockIdx.y];
    for (uint32_t i = threadIdx.x; i < J.npal; i += Q_THREADS) pal[i] = J.pal[i];
    __syncthreads();
    const uint32_t cell = blockIdx.x * Q_THREADS + threadIdx.x;
    const uint32_t r6 = cell >> 12, g6 = (cell >> 6) & 63, b6 = cell & 63;
    const uint32_t key = (((r6 << 2) | (r6 >> 4)) << 24) | (((g6 << 2) | (g6 >> 4)) << 16) |
                         (((b6 << 2) | (b6 >> 4)) << 8) | 255u;
    J.lut[cell] = (uint8_t)nearest_seq(pal, J.npal, key);
}

// ---- k_quant_map -----------------------------------------------------------------------------------
struct MapJob {
    const uint8_t *src;
    uint8_t *idx;
    const uint8_t *lut;         // null: early-out map (exact lookup)
    const uint32_t *pal;        // npal keys (early out: key order)
    uint32_t npal;
};

constexpr int MAP_PX = 4;   // pixels per thread and step

__global__ void __launch_bounds__(Q_THREADS) k_quant_map(const MapJob *jobs, uint64_t npix, uint32_t bpp)
{
    __shared__ uint32_t pal[256];
    const MapJob &J = jobs[blockIdx.y];
    const uint32_t n = J.npal, lane = threadIdx.x & 31;
    for (uint32_t i = threadIdx.x; i < n; i += Q_THREADS) pal[i] = J.pal[i];
    __syncthreads();
    const uint8_t *lut = J.lut;
    const bool rgba_words = bpp == 4 && (reinterpret_cast<uintptr_t>(J.src) & 15) == 0;
    const bool idx_words = (reinterpret_cast<uintptr_t>(J.idx) & 3) == 0;
    const uint64_t step = (uint64_t)gridDim.x * Q_THREADS * MAP_PX;
    // the loop bound is warp-uniform: the warp stays together for the cooperative search
    for (uint64_t wbase = ((uint64_t)blockIdx.x * Q_THREADS + (threadIdx.x & ~31u)) * MAP_PX; wbase < npix; wbase += step) {
        const uint64_t base = wbase + lane * MAP_PX;
        uint32_t key[MAP_PX];
        if (rgba_words && base + MAP_PX <= npix) {
            const uint4 v = __ldg(reinterpret_cast<const uint4 *>(J.src) + base / 4);
            key[0] = __byte_perm(v.x, 0, 0x0123); key[1] = __byte_perm(v.y, 0, 0x0123);
            key[2] = __byte_perm(v.z, 0, 0x0123); key[3] = __byte_perm(v.w, 0, 0x0123);
        } else {
#pragma unroll
            for (int k = 0; k < MAP_PX; ++k) key[k] = base + k < npix ? pixel_key(J.src, base + k, bpp) : 0xFFFFFFFFu;
        }
        uint32_t out[MAP_PX];
#pragma unroll
        for (int k = 0; k < MAP_PX; ++k) {
            const bool valid = base + k < npix;
            bool search = false;
            out[k] = 0;
            if (valid) {
                const uint32_t c = key[k];
                if (lut) {
                    if ((c & 255u) == 255u) out[k] = __ldg(lut + (((c >> 26) << 12) | (((c >> 18) & 63) << 6) | ((c >> 10) & 63)));
                    else search = true;
                } else {
                    uint32_t lo = 0, hi = n;
                    while (hi - lo > 1) {
                        const uint32_t mid = (lo + hi) >> 1;
                        if (pal[mid] <= c) lo = mid; else hi = mid;
                    }
                    if (pal[lo] == c) out[k] = lo; else search = true;
                }
            }
            out[k] = nearest_warp(pal, n, key[k], __ballot_sync(0xffffffffu, search), lane, out[k]);
        }
        if (idx_words && base + MAP_PX <= npix) {
            *reinterpret_cast<uint32_t *>(J.idx + base) = out[0] | (out[1] << 8) | (out[2] << 16) | (out[3] << 24);
        } else {
#pragma unroll
            for (int k = 0; k < MAP_PX; ++k) if (base + k < npix) J.idx[base + k] = (uint8_t)out[k];
        }
    }
}

// ---- k_quant_dither --------------------------------------------------------------------------------
// Floyd-Steinberg as pixo runs it (f32, row by row), computed exactly in integers: every error term
// er*k/16 is a multiple of 1/16 below 256 in magnitude, so pixo's f32 sums are exact and the kernel
// carries E16 = sum k*er and takes adj = clamp(16 v + E16, 0, 4080) >> 4.
// Pixel (x, y) receives 7 e(x-1, y) + 1 e(x-1, y-1) + 5 e(x, y-1) + 3 e(x+1, y-1).
// A warp owns 32 consecutive rows of one image, one lane per row; lane k handles pixel s - 1 - 2k at step s,
// so lane k-1 has finished pixel x+1 of the row above one step before lane k needs it, and passes that
// error down with a shuffle (the two before it stay in registers).  Row groups are handed out through
// a ticket counter in order; lane 0 of a group waits for the previous group's last row, which publishes
// its errors with a progress word every 32 pixels.  A group only waits on one a running warp claimed
// earlier, so the wavefront cannot deadlock; every wait is bounded and a timeout sets a status bit.
struct DitherJob {
    const uint8_t *src;
    uint8_t *idx;
    const uint8_t *lut;
    const uint32_t *pal;
    uint32_t npal;
    uint32_t *edge;         // (groups - 1) * width packed errors of each group's last row
    uint32_t *progress;     // groups - 1 words: pixels of that row published
};

struct DitherParams {
    const DitherJob *jobs;
    uint32_t n_jobs, width, height, bpp, groups;
    uint32_t *ticket;       // [0] next ticket, [1] status (bit 0: a wait timed out)
};

__device__ __forceinline__ uint32_t pack_err(int r, int g, int b)
{
    return ((uint32_t)r & 1023u) | (((uint32_t)g & 1023u) << 10) | (((uint32_t)b & 1023u) << 20);
}
__device__ __forceinline__ int err_ch(uint32_t e, int c) { return ((int)(e << (22 - 10 * c))) >> 22; }

__global__ void __launch_bounds__(DITHER_WARPS * 32) k_quant_dither(DitherParams P)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t W = P.width, total = P.n_jobs * P.groups;
    volatile uint32_t *status = P.ticket + 1;
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(P.ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= total) return;
        const uint32_t g = t / P.n_jobs;
        const DitherJob &J = P.jobs[t - g * P.n_jobs];
        const uint32_t y = g * 32 + lane;
        const bool row_ok = y < P.height;
        const uint8_t *row = J.src + (uint64_t)y * W * P.bpp;
        uint8_t *irow = J.idx + (uint64_t)y * W;
        const bool publish = lane == 31 && g + 1 < P.groups;
        const uint32_t *above = g ? J.edge + (uint64_t)(g - 1) * W : nullptr;
        uint32_t *mine = J.edge + (uint64_t)g * W;
        uint32_t seen = 0;                         // lane 0: pixels of the row above known published
        uint32_t carry = 0, up1 = 0, up0 = 0, last = 0;
        // lane 0 starts one step before its first pixel, to take e(0, y-1) in as every other lane does
        for (uint32_t s = 0; s < W + 63; ++s) {
            const int x = (int)s - 1 - 2 * (int)lane;
            uint32_t up = __shfl_up_sync(0xffffffffu, last, 1);
            if (lane == 0) {
                up = 0;
                const uint32_t xn = (uint32_t)(x + 1);   // x >= -1 for lane 0
                if (above && xn < W) {
                    if (seen <= xn) {
                        const volatile uint32_t *pw = J.progress + (g - 1);
                        uint32_t spins = 0;
                        while ((seen = *pw) <= xn) {
                            if (*status || ++spins > SPIN_LIMIT) { atomicOr(P.ticket + 1, 1u); seen = W; break; }
                            if (spins > 64) __nanosleep(128);
                        }
                        __threadfence();
                    }
                    up = __ldcg(above + xn);
                }
            }
            const bool active = row_ok && x >= 0 && x < (int)W;
            uint32_t c = 0xFFu, a = 255;
            int adj[3] = {0, 0, 0};
            if (active) {
                const uint32_t key = pixel_key(row, (uint64_t)x, P.bpp);
                a = key & 255u;
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) {
                    const int v = (key >> (24 - 8 * ch)) & 255;
                    const int e16 = 7 * err_ch(carry, ch) + err_ch(up1, ch) + 5 * err_ch(up0, ch) + 3 * err_ch(up, ch);
                    adj[ch] = min(max(16 * v + e16, 0), 4080) >> 4;
                }
                c = ((uint32_t)adj[0] << 24) | ((uint32_t)adj[1] << 16) | ((uint32_t)adj[2] << 8) | a;
            }
            uint32_t id = 0;
            if (active && a == 255u)
                id = __ldg(J.lut + (((uint32_t)(adj[0] >> 2) << 12) | ((uint32_t)(adj[1] >> 2) << 6) | (uint32_t)(adj[2] >> 2)));
            id = nearest_warp(J.pal, J.npal, c, __ballot_sync(0xffffffffu, active && a != 255u), lane, id);
            last = 0;
            if (active) {
                const uint32_t p = __ldg(J.pal + id);
                last = pack_err(adj[0] - (int)(p >> 24), adj[1] - (int)((p >> 16) & 255), adj[2] - (int)((p >> 8) & 255));
                irow[x] = (uint8_t)id;
                if (publish) {
                    __stcg(mine + x, last);
                    if ((x & 31) == 31 || x == (int)W - 1) {
                        __threadfence();
                        *(volatile uint32_t *)(J.progress + g) = (uint32_t)x + 1;
                    }
                }
            }
            carry = last;
            up1 = up0;
            up0 = up;
        }
    }
}

bool remapped_none(uint32_t s)
{
    return s == PIXO_B200_FILTER_ADAPTIVE || s == PIXO_B200_FILTER_ADAPTIVE_FAST || s == PIXO_B200_FILTER_MINSUM ||
           s == PIXO_B200_FILTER_BIGRAMS;
}

}  // namespace

int png_quantize_filter(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                        uint32_t width, uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                        uint32_t max_colors_u16, const uint8_t *palettes, const uint32_t *palette_lens,
                        pixo_b200_png_reduced *info, uint8_t *d_out, size_t out_stride, uint32_t *d_adler)
{
    const uint32_t bpp = color_type + 1;
    const uint64_t npix = (uint64_t)width * height;
    const bool force = strategy_and_flags & PIXO_B200_PNG_QUANTIZE_FORCE;
    const bool autom = strategy_and_flags & PIXO_B200_PNG_QUANTIZE_AUTO;
    const bool dither = strategy_and_flags & PIXO_B200_PNG_DITHER;
    const uint32_t max_colors = std::min<uint32_t>(max_colors_u16, 256);
    const uint32_t lossless_word = strategy_and_flags & ~(PIXO_B200_PNG_QUANTIZE_AUTO | PIXO_B200_PNG_QUANTIZE_FORCE |
                                                          PIXO_B200_PNG_DITHER);
    const bool rgbish = color_type == PIXO_B200_RGB || color_type == PIXO_B200_RGBA;

    // what each image becomes
    enum Kind { LOSSLESS, EARLY_OUT, LUT };
    std::vector<Kind> kind(n_images, LOSSLESS);
    std::vector<std::vector<uint32_t>> pal(n_images);          // palette keys r<<24|g<<16|b<<8|a
    std::vector<std::vector<uint32_t>> hcol(n_images), hcnt(n_images);

    if (rgbish && (force || autom)) {
        // 1. pixo's two sample sets of every image, sorted and counted on the device
        const uint64_t sd = std::max<uint64_t>(npix / DECISION_CAP, 1), sh = std::max<uint64_t>(npix / HISTOGRAM_CAP, 1);
        const uint64_t nd = (npix + sd - 1) / sd, nh = (npix + sh - 1) / sh, per = nd + nh;
        const uint32_t chunk = std::min<uint32_t>(n_images, SAMPLE_CHUNK);
        const size_t maxk = (size_t)chunk * per;
        size_t tmp_sort = 0, tmp_rle = 0;
        PIXO_CUDA(ctx, cub::DeviceRadixSort::SortKeys(nullptr, tmp_sort, (const unsigned long long *)nullptr,
                                                      (unsigned long long *)nullptr, (int)maxk, 0, 39, ctx->stream));
        PIXO_CUDA(ctx, cub::DeviceRunLengthEncode::Encode(nullptr, tmp_rle, (const unsigned long long *)nullptr,
                                                          (unsigned long long *)nullptr, (uint32_t *)nullptr,
                                                          (uint32_t *)nullptr, (int)maxk, ctx->stream));
        // d_quant: the sample keys, sorted, the runs' keys and counts, the run count, cub's temporary storage;
        // h_quant: the runs' keys and counts, the run count
        unsigned long long *ka, *kb, *uq, *h_uq;
        uint32_t *cn, *nr, *h_cn, *h_nr;
        uint8_t *tmp;
        PIXO_TRY(bind(ctx, ctx->d_quant, [&](Layout &L) {
            ka = L.take<unsigned long long>(maxk), kb = L.take<unsigned long long>(maxk);
            uq = L.take<unsigned long long>(maxk), cn = L.take<uint32_t>(maxk), nr = L.take<uint32_t>(1);
            tmp = L.take(std::max(tmp_sort, tmp_rle));
        }));
        PIXO_TRY(bind(ctx, ctx->h_quant, [&](Layout &L) {
            h_uq = L.take<unsigned long long>(maxk), h_cn = L.take<uint32_t>(maxk), h_nr = L.take<uint32_t>(1);
        }, 8));
        for (uint32_t i0 = 0; i0 < n_images; i0 += chunk) {
            const uint32_t nb = std::min(chunk, n_images - i0);
            const int nk = (int)(nb * per);
            SampleParams S;
            S.data = d_data + (size_t)i0 * in_stride; S.in_stride = in_stride; S.n_images = nb; S.bpp = bpp;
            S.nd = nd; S.nh = nh; S.sd = sd; S.sh = sh; S.keys = ka;
            const uint32_t ctas = (uint32_t)std::min<uint64_t>(((uint64_t)nk + Q_THREADS - 1) / Q_THREADS, (uint64_t)ctx->sm_count * 16);
            PIXO_TRY(launch(ctx, k_quant_sample, ctas, Q_THREADS, 0, S));
            size_t tb = tmp_sort;
            PIXO_CUDA(ctx, cub::DeviceRadixSort::SortKeys(tmp, tb, ka, kb, nk, 0, 39, ctx->stream));
            tb = tmp_rle;
            PIXO_CUDA(ctx, cub::DeviceRunLengthEncode::Encode(tmp, tb, kb, uq, cn, nr, nk, ctx->stream));
            PIXO_CUDA(ctx, cudaMemcpyAsync(h_nr, nr, 4, cudaMemcpyDeviceToHost, ctx->stream));
            PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            const uint32_t runs = *h_nr;
            PIXO_CUDA(ctx, cudaMemcpyAsync(h_uq, uq, (size_t)runs * 8, cudaMemcpyDeviceToHost, ctx->stream));
            PIXO_CUDA(ctx, cudaMemcpyAsync(h_cn, cn, (size_t)runs * 4, cudaMemcpyDeviceToHost, ctx->stream));
            PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            std::vector<uint64_t> unique(nb, 0);
            for (uint32_t r = 0; r < runs; ++r) {
                const unsigned long long k = h_uq[r];
                const uint32_t img = i0 + (uint32_t)(k >> 33);
                if (!((k >> 32) & 1)) { ++unique[img - i0]; continue; }
                hcol[img].push_back((uint32_t)k);
                hcnt[img].push_back((uint32_t)std::min<uint64_t>((uint64_t)h_cn[r] * sh, 0xFFFFFFFFull));
            }
            // 2. decisions (encode_into, should_quantize_auto) and the palette of each image
            for (uint32_t j = 0; j < nb; ++j) {
                const uint32_t i = i0 + j;
                const bool q = force || (unique[j] > max_colors && unique[j] <= (uint64_t)max_colors * 32);
                if (!q) { hcol[i].clear(); hcnt[i].clear(); continue; }
                const uint32_t given = palettes && palette_lens ? palette_lens[i] : 0;
                if (given) {
                    kind[i] = LUT;
                    const uint8_t *pp = palettes + (size_t)i * 1024;
                    for (uint32_t e = 0; e < given; ++e)
                        pal[i].push_back(((uint32_t)pp[4 * e] << 24) | ((uint32_t)pp[4 * e + 1] << 16) |
                                         ((uint32_t)pp[4 * e + 2] << 8) | pp[4 * e + 3]);
                    hcol[i].clear(); hcnt[i].clear();
                } else if (hcol[i].size() > MAX_HIST_COLORS) {
                    return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED,
                                     "image %u: %zu distinct colours among the histogram samples exceed 8192; pixo keeps "
                                     "the 8192 most frequent with an unstable sort whose tie order this library does "
                                     "not restate - pass the palette pixo's median_cut_palette produced", i, hcol[i].size());
                } else if (hcol[i].size() <= max_colors) {
                    kind[i] = EARLY_OUT;
                    pal[i] = hcol[i];
                    hcol[i].clear(); hcnt[i].clear();
                } else {
                    kind[i] = LUT;
                    pal[i] = median_cut_palette(hcol[i], hcnt[i], max_colors);
                }
            }
        }
    }

    std::vector<uint32_t> qall;
    for (uint32_t i = 0; i < n_images; ++i) if (kind[i] != LOSSLESS) qall.push_back(i);
    const size_t idx_stride = Layout::round(npix);
    // steps 3-5 in passes of at most QUANT_PASS quantised images: every grid.y stays within CUDA's limit
    // and the scratch (about 330 KB per image besides its indices) does not grow with the batch
    for (size_t q0 = 0; q0 < qall.size(); q0 += QUANT_PASS) {
        const std::vector<uint32_t> qids(qall.begin() + q0, qall.begin() + std::min(qall.size(), q0 + QUANT_PASS));
        const size_t nq = qids.size();
        // 3. k-means, tables, map / dither on the device
        const size_t jobs_bytes = nq * (sizeof(KmeansJob) + sizeof(LutJob) + sizeof(MapJob) + sizeof(DitherJob)) + 1024;
        const size_t groups = (height + 31) / 32;
        // d_quant_img: the jobs, palettes, k-means sums, histogram colours, tables, dither edges and progress, the
        // dither ticket, the indices
        uint8_t *d_jobs, *d_lut, *d_idx;
        uint32_t *d_pal, *d_col, *d_edge, *d_prog, *d_tick;
        unsigned long long *d_acc;
        PIXO_TRY(bind(ctx, ctx->d_quant_img, [&](Layout &L) {
            d_jobs = L.take(jobs_bytes);
            d_pal = L.take<uint32_t>(nq * 256);
            d_acc = L.take<unsigned long long>(nq * 256 * 5);
            d_col = L.take<uint32_t>(nq * MAX_HIST_COLORS * 2);
            d_lut = L.take(nq * LUT_CELLS);
            d_edge = L.take<uint32_t>(nq * groups * width);
            d_prog = L.take<uint32_t>(nq * groups);
            d_tick = L.take<uint32_t>(1);
            d_idx = L.take(nq * idx_stride);
        }));
        std::vector<uint32_t> h_pal(nq * 256, 0);
        std::vector<uint32_t> h_col;   // each k-means job's histogram colours then counts, packed
        std::vector<KmeansJob> km;
        std::vector<LutJob> lj;
        std::vector<MapJob> mj;
        std::vector<DitherJob> dj;
        uint32_t max_cols = 0;
        for (size_t k = 0; k < nq; ++k) {
            const uint32_t i = qids[k];
            std::copy(pal[i].begin(), pal[i].end(), h_pal.begin() + k * 256);
            uint32_t *dp = d_pal + k * 256;
            if (!hcol[i].empty()) {   // median cut ran: two k-means passes over its histogram
                const uint32_t *cc = d_col + h_col.size();
                h_col.insert(h_col.end(), hcol[i].begin(), hcol[i].end());
                h_col.insert(h_col.end(), hcnt[i].begin(), hcnt[i].end());
                km.push_back({cc, cc + hcol[i].size(), (uint32_t)hcol[i].size(), (uint32_t)pal[i].size(), dp, d_acc + k * 256 * 5});
                max_cols = std::max(max_cols, (uint32_t)hcol[i].size());
            }
            uint8_t *lut = d_lut + k * LUT_CELLS;
            if (kind[i] == LUT) lj.push_back({dp, (uint32_t)pal[i].size(), lut});
            MapJob M{d_data + (size_t)i * in_stride, d_idx + k * idx_stride, kind[i] == LUT ? lut : nullptr, dp,
                     (uint32_t)pal[i].size()};
            if (kind[i] == LUT && dither)
                dj.push_back({M.src, M.idx, lut, dp, M.npal, d_edge + k * groups * width,
                              d_prog + k * groups});
            else
                mj.push_back(M);
        }
        auto *d_km = reinterpret_cast<KmeansJob *>(d_jobs);
        auto *d_lj = reinterpret_cast<LutJob *>(d_km + km.size());
        auto *d_mj = reinterpret_cast<MapJob *>(d_lj + lj.size());
        auto *d_dj = reinterpret_cast<DitherJob *>(d_mj + mj.size());
        std::vector<uint8_t> jobs(jobs_bytes);
        size_t o = 0;
        auto put = [&](const void *p, size_t n) { memcpy(jobs.data() + o, p, n); o += n; };
        put(km.data(), km.size() * sizeof(KmeansJob));
        put(lj.data(), lj.size() * sizeof(LutJob));
        put(mj.data(), mj.size() * sizeof(MapJob));
        put(dj.data(), dj.size() * sizeof(DitherJob));
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_jobs, jobs.data(), o, cudaMemcpyHostToDevice, ctx->stream));
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_pal, h_pal.data(), nq * 256 * 4, cudaMemcpyHostToDevice, ctx->stream));
        if (!km.empty()) {
            PIXO_CUDA(ctx, cudaMemcpyAsync(d_col, h_col.data(), h_col.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
            PIXO_CUDA(ctx, cudaMemsetAsync(d_acc, 0, nq * 256 * 5 * 8, ctx->stream));
            for (int pass = 0; pass < 2; ++pass) {
                PIXO_TRY(launch(ctx, k_quant_kmeans, dim3((max_cols + Q_THREADS - 1) / Q_THREADS, (uint32_t)km.size()),
                                Q_THREADS, 0, d_km));
                PIXO_TRY(launch(ctx, k_quant_update, (uint32_t)km.size(), 256, 0, d_km));
            }
        }
        if (!lj.empty())
            PIXO_TRY(launch(ctx, k_quant_lut, dim3(LUT_CELLS / Q_THREADS, (uint32_t)lj.size()), Q_THREADS, 0, d_lj));
        PIXO_CUDA(ctx, cudaMemcpyAsync(h_pal.data(), d_pal, nq * 256 * 4, cudaMemcpyDeviceToHost, ctx->stream));
        if (!mj.empty()) {
            const uint64_t want = (uint64_t)ctx->sm_count * 8 / mj.size() + 1;
            const uint32_t ctas = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(want, (npix + Q_THREADS * MAP_PX - 1) / (Q_THREADS * MAP_PX)));
            PIXO_TRY(launch(ctx, k_quant_map, dim3(ctas, (uint32_t)mj.size()), Q_THREADS, 0, d_mj, npix, bpp));
        }
        if (!dj.empty()) {
            PIXO_CUDA(ctx, cudaMemsetAsync(d_prog, 0, nq * groups * 4, ctx->stream));
            PIXO_CUDA(ctx, cudaMemsetAsync(d_tick, 0, 8, ctx->stream));
            bool &carveout_set = ctx->kernels[reinterpret_cast<const void *>(k_quant_dither)].carveout_set;
            if (!carveout_set) {
                PIXO_CUDA(ctx, cudaFuncSetAttribute(k_quant_dither, cudaFuncAttributePreferredSharedMemoryCarveout, 0));
                carveout_set = true;
            }
            DitherParams D{d_dj, (uint32_t)dj.size(), width, height, bpp, (uint32_t)groups, d_tick};
            const uint64_t warps = std::min<uint64_t>((uint64_t)dj.size() * groups, (uint64_t)ctx->sm_count * 32);
            PIXO_TRY(launch(ctx, k_quant_dither, (uint32_t)((warps + DITHER_WARPS - 1) / DITHER_WARPS), DITHER_WARPS * 32,
                            0, D));
        }
        uint32_t h_tick[2] = {0, 0};
        PIXO_CUDA(ctx, cudaMemcpyAsync(h_tick, d_tick, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (!dj.empty() && (h_tick[1] & 1u))
            return set_error(ctx, PIXO_B200_ERR_CUDA, "k_quant_dither: a row group's wait for the rows above timed out");

        // 4. what encode_indexed_into writes: PLTE, trimmed tRNS, 8-bit indices
        for (size_t k = 0; k < nq; ++k) {
            const uint32_t i = qids[k], n = (uint32_t)pal[i].size();
            pixo_b200_png_reduced &r = info[i];
            memset(&r, 0, sizeof r);
            r.color_type_byte = 3; r.bit_depth = 8; r.effective_color_type = PIXO_B200_RGB; r.bytes_per_pixel = 1;
            r.row_bytes = width;
            r.palette_len = n;
            uint32_t alpha[256];
            for (uint32_t e = 0; e < n; ++e) {
                const uint32_t key = h_pal[k * 256 + e];
                r.palette[e][0] = (uint8_t)(key >> 24); r.palette[e][1] = (uint8_t)(key >> 16);
                r.palette[e][2] = (uint8_t)(key >> 8); r.palette[e][3] = (uint8_t)key;
                alpha[e] = key & 255u;
            }
            r.trns_len = trimmed_trns_len(alpha, n);
        }
        // 5. the index rows through the filter: one launch per run of consecutive quantised images
        const uint32_t strat = strategy_and_flags & 0xFFu;
        const uint32_t fs = remapped_none(strat) ? (uint32_t)PIXO_B200_FILTER_NONE : strat;
        for (size_t k0 = 0; k0 < nq;) {
            size_t k1 = k0 + 1;
            while (k1 < nq && qids[k1] == qids[k1 - 1] + 1) ++k1;
            const uint32_t i0 = qids[k0];
            PIXO_TRY(launch_png_filter_rows(ctx, d_idx + k0 * idx_stride, idx_stride, (uint32_t)(k1 - k0), width, height,
                                            width, 1, fs, d_out + (size_t)i0 * out_stride, out_stride,
                                            d_adler ? d_adler + i0 : nullptr, nullptr, height));
            k0 = k1;
        }
    }

    // 6. frames pixo does not quantise take the lossless path unchanged
    for (uint32_t i0 = 0; i0 < n_images;) {
        if (kind[i0] != LOSSLESS) { ++i0; continue; }
        uint32_t i1 = i0 + 1;
        while (i1 < n_images && kind[i1] == LOSSLESS) ++i1;
        PIXO_TRY(png_reduce_filter(ctx, d_data + (size_t)i0 * in_stride, in_stride, i1 - i0, width, height, color_type,
                                   lossless_word, info + i0, d_out + (size_t)i0 * out_stride, out_stride,
                                   d_adler ? d_adler + i0 : nullptr));
        i0 = i1;
    }
    return 0;
}

}  // namespace pixo
