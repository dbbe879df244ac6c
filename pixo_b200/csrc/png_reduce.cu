// png_reduce.cu — pixo's lossless colour-type / palette reduction ahead of the PNG filter.
//
// Restates
//   maybe_reduce_color_type          src/png/mod.rs:683-836
//   build_palette                    src/png/mod.rs:838-900   (key r<<24|g<<16|b<<8|a, sorted unique)
//   build_co_occurrence_matrix       src/png/mod.rs:940-977
//   all_gray_rgb / analyze_rgba      src/png/mod.rs:1122-1147
//   reduce_gray_bit_depth, palette_bit_depth, pack_bits_rows   src/png/bit_depth.rs
// The palette ordering itself (mzeng_reindex, apply_most_popular_first) is host work on <= 256
// colours, png_host.cpp.
//
// Design (H100): three kernels, then the filter kernels of png_filter.cu on the reduced rows.
//   k_reduce_analyze: one launch for the batch, grid (CTAs, images), each CTA a contiguous run of
//     pixels.  Gray / opaque / max(channel 0) are OR / max reductions.  The distinct colours go into a
//     1024-slot hash set in shared memory (64-bit slots, 0 = empty, so every 32-bit key - transparent
//     black included - is storable), after a warp-level de-duplication with __match_any_sync; at the end
//     the CTA merges its set into the image's global set of the same shape.  Past 256 colours an
//     overflow flag is raised, and a CTA stops as soon as nothing the image could still need is open
//     (no palette possible, not gray, not opaque): photographic frames leave after a few CTAs' work.
//   k_reduce_index (palette images only): the pre-remap index of every pixel against the sorted palette
//     (binary search in shared memory), written as a byte, plus the per-index counts and the
//     off-diagonal co-occurrence counts of right and below neighbours.  The index below is looked up
//     from the raw row below, so the kernel does not read its own output.  The counters are privatised
//     in shared memory (n(n-1)/2 + 256 u32, 129 KB at 256 colours) with warp-aggregated increments and
//     flushed with one global atomic per non-zero counter: a flat image hammers one counter, which
//     global atomics serialise in L2, while a shared counter absorbs it inside the SM.
//   k_reduce_pack: every byte of the reduced rows from the raw pixels or the indices: palette byte map
//     + 1/2/4/8-bit packing, gray extraction + packing, RGB or GrayAlpha extraction.  An image that
//     does not reduce is not copied: the filter reads the caller's pixels.
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "png_host.hpp"

namespace pixo {
namespace {

constexpr int RED_THREADS = 256;
constexpr int SET_SLOTS = 1024;        // hash-set slots (shared per CTA, and global per image)
constexpr int AN_UNROLL = 4;           // pixels per thread per step of k_reduce_analyze
constexpr uint32_t AN_PIXELS = 16384;  // pixels per CTA of k_reduce_analyze
constexpr uint32_t TRI_MAX = 256 * 255 / 2;

// per-image result of k_reduce_analyze (zeroed before it)
struct ReduceStat {
    uint32_t not_gray, not_opaque, max0, overflow, count, pad[3];
    unsigned long long slot[SET_SLOTS];
};

struct AnalyzeParams {
    const uint8_t *data;
    size_t in_stride;
    uint64_t npix;
    uint32_t bpp, want_pal, want_ct, per_cta;
    ReduceStat *stat;
};

__device__ __forceinline__ uint32_t mix32(uint32_t k)   // murmur3 finaliser
{
    k ^= k >> 16; k *= 0x85ebca6bu; k ^= k >> 13; k *= 0xc2b2ae35u; k ^= k >> 16;
    return k;
}

// Insert into a set of SET_SLOTS 64-bit slots.  Returns 1 if the key was new, 0 if present, -1 if the
// set is full (only possible with far more than 256 keys, which is an overflow anyway).
__device__ __forceinline__ int set_insert(unsigned long long *set, uint32_t key)
{
    const unsigned long long v = (1ull << 32) | key;
    uint32_t h = mix32(key) & (SET_SLOTS - 1);
    for (int probe = 0; probe < SET_SLOTS; ++probe) {
        const unsigned long long old = atomicCAS(set + h, 0ull, v);
        if (old == 0ull) return 1;
        if (old == v) return 0;
        h = (h + 1) & (SET_SLOTS - 1);
    }
    return -1;
}

__device__ __forceinline__ void load_px(const uint8_t *src, uint64_t p, uint32_t bpp, bool word,
                                        uint32_t &r, uint32_t &g, uint32_t &b, uint32_t &a)
{
    if (word) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(src) + p);
        r = v & 255u; g = (v >> 8) & 255u; b = (v >> 16) & 255u; a = v >> 24;
    } else {
        const uint8_t *q = src + p * bpp;
        r = __ldg(q); g = __ldg(q + 1); b = __ldg(q + 2); a = bpp == 4 ? __ldg(q + 3) : 255u;
    }
}

__global__ void __launch_bounds__(RED_THREADS) k_reduce_analyze(AnalyzeParams P)
{
    __shared__ unsigned long long set[SET_SLOTS];
    __shared__ uint32_t s_count, s_flags, s_max, s_stop;   // s_flags: 1 overflow, 2 not gray, 4 not opaque
    const uint32_t img = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
    ReduceStat *st = P.stat + img;
    const uint8_t *src = P.data + (size_t)img * P.in_stride;
    const bool word = P.bpp == 4 && (reinterpret_cast<uintptr_t>(src) & 3) == 0;
    const uint64_t p0 = (uint64_t)blockIdx.x * P.per_cta;
    const uint64_t p1 = min(p0 + P.per_cta, P.npix);
    for (int s = tid; s < SET_SLOTS; s += RED_THREADS) set[s] = 0ull;
    if (tid == 0) { s_count = 0; s_flags = 0; s_max = 0; s_stop = 0; }
    __syncthreads();

    uint32_t published = 0;   // thread 0: flags already raised in the image's state
    bool ng = false, no = false;
    uint32_t mx = 0;
    for (uint64_t base = p0; base < p1; base += RED_THREADS * AN_UNROLL) {
        if (tid == 0) {
            const uint32_t f = *(volatile uint32_t *)&s_flags;
            if ((f & 1) && !(published & 1)) atomicExch(&st->overflow, 1u);
            if ((f & 2) && !(published & 2)) atomicExch(&st->not_gray, 1u);
            if ((f & 4) && !(published & 4)) atomicExch(&st->not_opaque, 1u);
            published = f;
            const volatile ReduceStat *vs = st;
            const bool pal_open = P.want_pal && !(f & 1) && !vs->overflow;
            const bool gray_open = P.want_ct && !(f & 2) && !vs->not_gray;
            const bool opaque_open = P.want_ct && P.bpp == 4 && !(f & 4) && !vs->not_opaque;
            s_stop = !(pal_open || gray_open || opaque_open);
        }
        __syncthreads();
        if (s_stop) break;
        const bool pal = P.want_pal && !(s_flags & 1);
        __syncthreads();   // everyone has read s_flags before it changes in this step
#pragma unroll
        for (int u = 0; u < AN_UNROLL; ++u) {
            const uint64_t p = base + (uint64_t)u * RED_THREADS + tid;
            const bool valid = p < p1;
            uint32_t r = 0, g = 0, b = 0, a = 255;
            if (valid) {
                load_px(src, p, P.bpp, word, r, g, b, a);
                ng |= !(r == g && g == b);
                no |= a != 255u;
                mx = max(mx, r);
            }
            if (pal) {
                const uint32_t key = (r << 24) | (g << 16) | (b << 8) | a;
                const unsigned vm = __ballot_sync(0xffffffffu, valid);
                if (valid) {
                    const unsigned peers = __match_any_sync(vm, key);
                    if (lane == (unsigned)__ffs(peers) - 1 && *(volatile uint32_t *)&s_count <= 256u) {
                        const int ins = set_insert(set, key);
                        if (ins < 0 || (ins > 0 && atomicAdd(&s_count, 1u) >= 256u)) atomicOr(&s_flags, 1u);
                    }
                }
            }
        }
        const unsigned any_ng = __ballot_sync(0xffffffffu, ng), any_no = __ballot_sync(0xffffffffu, no);
        if (lane == 0 && (any_ng || any_no)) atomicOr(&s_flags, (any_ng ? 2u : 0u) | (any_no ? 4u : 0u));
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    const unsigned any_ng = __ballot_sync(0xffffffffu, ng), any_no = __ballot_sync(0xffffffffu, no);
    if (lane == 0) {
        atomicMax(&s_max, mx);
        if (any_ng || any_no) atomicOr(&s_flags, (any_ng ? 2u : 0u) | (any_no ? 4u : 0u));
    }
    __syncthreads();
    const uint32_t f = s_flags;
    if (tid == 0) {
        if (f & 1) atomicExch(&st->overflow, 1u);
        if (f & 2) atomicExch(&st->not_gray, 1u);
        if (f & 4) atomicExch(&st->not_opaque, 1u);
        atomicMax(&st->max0, s_max);
    }
    if (!P.want_pal || (f & 1)) return;
    // merge the CTA's colours into the image's set
    for (int s = tid; s < SET_SLOTS; s += RED_THREADS) {
        const unsigned long long v = set[s];
        if (!v || *(volatile uint32_t *)&st->overflow) continue;
        const int ins = set_insert(st->slot, (uint32_t)v);
        if (ins < 0 || (ins > 0 && atomicAdd(&st->count, 1u) >= 256u)) atomicExch(&st->overflow, 1u);
    }
}

// ---- k_reduce_index --------------------------------------------------------------------------------
struct IndexJob {
    const uint8_t *src;    // the image's raw pixels
    uint8_t *idx;          // pre-remap index per pixel
    uint32_t *counts;      // 256 + TRI_MAX u32 (zeroed): counts, then the upper triangle
    uint32_t n, stats;     // palette entries; statistics wanted (n > 2)
    uint32_t keys[256];    // sorted palette keys
};

struct IndexParams {
    const IndexJob *jobs;
    uint32_t width, height, bpp, per_cta;
    uint64_t npix;
};

__device__ __forceinline__ uint32_t key_at(const uint8_t *src, uint64_t p, uint32_t bpp, bool word)
{
    uint32_t r, g, b, a;
    load_px(src, p, bpp, word, r, g, b, a);
    return (r << 24) | (g << 16) | (b << 8) | a;
}

__device__ __forceinline__ uint32_t lookup(const uint32_t *keys, uint32_t n, uint32_t key)
{
    uint32_t lo = 0, hi = n;   // keys[lo..hi) holds key
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (keys[mid] <= key) lo = mid; else hi = mid;
    }
    return lo;
}

// warp-aggregated shared-memory increment of counter[c] for the active lanes in `mask`
__device__ __forceinline__ void warp_count(uint32_t *counter, uint32_t c, unsigned mask, uint32_t lane)
{
    const unsigned peers = __match_any_sync(mask, c);
    if (lane == (unsigned)__ffs(peers) - 1) atomicAdd(counter + c, (uint32_t)__popc(peers));
}

__global__ void __launch_bounds__(RED_THREADS) k_reduce_index(IndexParams P)
{
    extern __shared__ uint32_t sm[];   // keys[256], counts[256], tri[n(n-1)/2]
    const IndexJob &J = P.jobs[blockIdx.y];
    const uint32_t tid = threadIdx.x, lane = tid & 31, n = J.n;
    uint32_t *keys = sm, *cnt = sm + 256, *tri = sm + 512;
    const uint32_t ncnt = J.stats ? 256 + n * (n - 1) / 2 : 0;
    for (uint32_t i = tid; i < n; i += RED_THREADS) keys[i] = J.keys[i];
    for (uint32_t i = tid; i < ncnt; i += RED_THREADS) cnt[i] = 0;
    __syncthreads();
    const bool word = P.bpp == 4 && (reinterpret_cast<uintptr_t>(J.src) & 3) == 0;
    const uint64_t p0 = (uint64_t)blockIdx.x * P.per_cta, p1 = min(p0 + P.per_cta, P.npix);
    for (uint64_t base = p0; base < p1; base += RED_THREADS) {
        const uint64_t p = base + tid;
        const bool valid = p < p1;
        uint32_t i = 0;
        if (valid) {
            i = lookup(keys, n, key_at(J.src, p, P.bpp, word));
            J.idx[p] = (uint8_t)i;
        }
        if (!J.stats) continue;
        const unsigned vm = __ballot_sync(0xffffffffu, valid);
        // the right neighbour's index: the next lane's, or looked up at the warp's end
        const uint32_t nb = __shfl_down_sync(0xffffffffu, i, 1);
        if (!valid) continue;
        warp_count(cnt, i, vm, lane);
        const uint32_t x = (uint32_t)(p % P.width), y = (uint32_t)(p / P.width);
        uint32_t pr = 0xffffffffu, pb = 0xffffffffu;   // pair codes, none = all ones
        if (x + 1 < P.width) {
            const uint32_t j = (lane < 31 && p + 1 < p1) ? nb : lookup(keys, n, key_at(J.src, p + 1, P.bpp, word));
            if (j != i) pr = (uint32_t)tri_index(min(i, j), max(i, j), n);
        }
        if (y + 1 < P.height) {
            const uint32_t j = lookup(keys, n, key_at(J.src, p + P.width, P.bpp, word));
            if (j != i) pb = (uint32_t)tri_index(min(i, j), max(i, j), n);
        }
        const unsigned mr = __ballot_sync(vm, pr != 0xffffffffu);
        if (pr != 0xffffffffu) warp_count(tri, pr, mr, lane);
        const unsigned mb = __ballot_sync(vm, pb != 0xffffffffu);
        if (pb != 0xffffffffu) warp_count(tri, pb, mb, lane);
    }
    __syncthreads();
    for (uint32_t k = tid; k < ncnt; k += RED_THREADS)
        if (const uint32_t v = cnt[k]) atomicAdd(J.counts + k, v);
}

// ---- k_reduce_pack ---------------------------------------------------------------------------------
enum PackMode : uint32_t { PACK_PALETTE = 0, PACK_GRAY = 1, PACK_RGB = 2, PACK_GRAY_ALPHA = 3 };

struct PackJob {
    const uint8_t *src;    // indices (palette) or raw pixels
    uint8_t *dst;          // height * row_bytes
    uint32_t mode, bits;
    uint64_t row_bytes;
    uint8_t map[256];      // palette: pre-remap index -> PLTE index
};

struct PackParams {
    const PackJob *jobs;
    uint32_t width, height, bpp;
};

__global__ void __launch_bounds__(RED_THREADS) k_reduce_pack(PackParams P)
{
    __shared__ uint8_t map[256];
    const PackJob &J = P.jobs[blockIdx.y];
    const uint32_t mode = J.mode, bits = J.bits;
    if (mode == PACK_PALETTE) {
        map[threadIdx.x] = J.map[threadIdx.x];
        __syncthreads();
    }
    const uint64_t total = J.row_bytes * P.height, w = P.width;
    for (uint64_t o = (uint64_t)blockIdx.x * RED_THREADS + threadIdx.x; o < total; o += (uint64_t)gridDim.x * RED_THREADS) {
        const uint64_t y = o / J.row_bytes, c = o - y * J.row_bytes;
        uint32_t v;
        if (mode == PACK_RGB) {
            const uint64_t px = y * w + c / 3;
            v = J.src[px * 4 + c % 3];
        } else if (mode == PACK_GRAY_ALPHA) {
            const uint64_t px = y * w + c / 2;
            v = J.src[px * 4 + ((c & 1) ? 3 : 0)];
        } else {
            const uint32_t per = 8 / bits;
            v = 0;
            for (uint32_t k = 0; k < per; ++k) {
                const uint64_t x = c * per + k;
                uint32_t s = 0;
                if (x < w) s = mode == PACK_PALETTE ? map[J.src[y * w + x]] : J.src[(y * w + x) * P.bpp];
                v = (v << bits) | s;
            }
        }
        J.dst[o] = (uint8_t)v;
    }
}

uint32_t palette_bits(uint32_t n) { return n <= 2 ? 1 : n <= 4 ? 2 : n <= 16 ? 4 : 8; }
uint32_t gray_bits(uint32_t vmax) { return vmax <= 1 ? 1 : vmax <= 3 ? 2 : vmax <= 15 ? 4 : 8; }

}  // namespace

int png_reduce_filter(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride, uint32_t n_images,
                      uint32_t width, uint32_t height, uint32_t color_type, uint32_t strategy_and_flags,
                      pixo_b200_png_reduced *info, uint8_t *d_out, size_t out_stride, uint32_t *d_adler)
{
    const uint32_t bpp = color_type + 1;
    const uint64_t npix = (uint64_t)width * height;
    const bool rgbish = color_type == PIXO_B200_RGB || color_type == PIXO_B200_RGBA;
    const bool want_pal = (strategy_and_flags & PIXO_B200_PNG_REDUCE_PALETTE) && rgbish;
    const bool want_ct = (strategy_and_flags & PIXO_B200_PNG_REDUCE_COLOR_TYPE) && rgbish;
    const bool opt_alpha = strategy_and_flags & PIXO_B200_PNG_OPTIMIZE_ALPHA;
    const uint32_t strategy = strategy_and_flags & 0xFFu;

    // what each image becomes; start from "unchanged"
    enum Kind { UNCHANGED, PALETTE, GRAY, RGB, GRAY_ALPHA };
    std::vector<Kind> kind(n_images, UNCHANGED);
    std::vector<uint32_t> bits(n_images, 8);
    std::vector<std::vector<uint32_t>> keys(n_images);
    for (uint32_t i = 0; i < n_images; ++i) {
        pixo_b200_png_reduced &r = info[i];
        memset(&r, 0, sizeof r);
        r.color_type_byte = (uint8_t)(color_type == PIXO_B200_GRAY ? 0 : color_type == PIXO_B200_GRAY_ALPHA ? 4
                                      : color_type == PIXO_B200_RGB ? 2 : 6);
        r.bit_depth = 8;
        r.effective_color_type = (uint8_t)color_type;
        r.bytes_per_pixel = (uint8_t)bpp;
        r.row_bytes = (uint64_t)width * bpp;
    }

    if (want_pal || want_ct) {
        // 1. analysis of the whole batch
        const size_t stat_bytes = (size_t)n_images * sizeof(ReduceStat);
        PIXO_TRY(ctx->d_red.ensure(ctx, stat_bytes));
        PIXO_TRY(ctx->h_red.ensure(ctx, stat_bytes));
        auto *d_stat = reinterpret_cast<ReduceStat *>(ctx->d_red.ptr);
        auto *h_stat = reinterpret_cast<ReduceStat *>(ctx->h_red.ptr);
        PIXO_CUDA(ctx, cudaMemsetAsync(d_stat, 0, stat_bytes, ctx->stream));
        AnalyzeParams A;
        A.data = d_data; A.in_stride = in_stride; A.npix = npix; A.bpp = bpp;
        A.want_pal = want_pal; A.want_ct = want_ct; A.per_cta = AN_PIXELS; A.stat = d_stat;
        const uint32_t ctas = (uint32_t)((npix + AN_PIXELS - 1) / AN_PIXELS);
        for (uint32_t i0 = 0; i0 < n_images; i0 += 65535) {
            const uint32_t nb = std::min(n_images - i0, 65535u);
            AnalyzeParams Ai = A;
            Ai.data = d_data + (size_t)i0 * in_stride; Ai.stat = d_stat + i0;
            PIXO_TRY(launch(ctx, k_reduce_analyze, dim3(ctas, nb), RED_THREADS, 0, Ai));
        }
        PIXO_CUDA(ctx, cudaMemcpyAsync(h_stat, d_stat, stat_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

        // 2. decisions (maybe_reduce_color_type's order: palette first, then the colour type)
        for (uint32_t i = 0; i < n_images; ++i) {
            const ReduceStat &s = h_stat[i];
            const bool gray = !s.not_gray, opaque = color_type == PIXO_B200_RGB || !s.not_opaque;
            if (want_pal && !s.overflow) {
                kind[i] = PALETTE;
                for (int k = 0; k < SET_SLOTS; ++k)
                    if (s.slot[k]) keys[i].push_back((uint32_t)s.slot[k]);
                std::sort(keys[i].begin(), keys[i].end());
                bits[i] = palette_bits((uint32_t)keys[i].size());
            } else if (want_ct) {
                if (gray && opaque) { kind[i] = GRAY; bits[i] = gray_bits(s.max0); }
                else if (color_type == PIXO_B200_RGBA && opaque) kind[i] = RGB;
                else if (color_type == PIXO_B200_RGBA && gray) kind[i] = GRAY_ALPHA;
            }
        }
    }

    // 3. palette images: indices and statistics on the GPU, the ordering on the host
    std::vector<uint32_t> pal_ids;
    for (uint32_t i = 0; i < n_images; ++i) if (kind[i] == PALETTE) pal_ids.push_back(i);
    std::vector<PackJob> pack;   // one per reduced image, in image order
    std::vector<uint32_t> pack_img;
    size_t red_stride = 0;
    for (uint32_t i = 0; i < n_images; ++i) {
        if (kind[i] == UNCHANGED) continue;
        const uint32_t b = kind[i] == PALETTE || kind[i] == GRAY ? bits[i] : 8;
        const uint32_t ch = kind[i] == RGB ? 3 : kind[i] == GRAY_ALPHA ? 2 : 1;
        const uint64_t rb = b < 8 ? ((uint64_t)width * b + 7) / 8 : (uint64_t)width * ch;
        red_stride = std::max(red_stride, (size_t)((rb * height + 15) & ~15ull));
    }
    const size_t cnt_words = 256 + TRI_MAX;
    std::vector<uint8_t> maps(pal_ids.size() * 256, 0);
    uint8_t *d_idx = nullptr;   // every palette image's indices, npix each
    if (!pal_ids.empty()) {
        const size_t np = pal_ids.size();
        // d_red_idx: the indices, the jobs, the counts
        IndexJob *d_jobs;
        uint32_t *d_cnt;
        PIXO_TRY(bind(ctx, ctx->d_red_idx, [&](Layout &L) {
            d_idx = L.take(np * npix), d_jobs = L.take<IndexJob>(np), d_cnt = L.take<uint32_t>(np * cnt_words);
        }));
        std::vector<IndexJob> jobs(np);
        uint32_t nmax = 0;
        bool any_stats = false;
        for (size_t k = 0; k < np; ++k) {
            const uint32_t i = pal_ids[k];
            IndexJob &J = jobs[k];
            memset(&J, 0, sizeof J);
            J.src = d_data + (size_t)i * in_stride;
            J.idx = d_idx + k * npix;
            J.counts = d_cnt + k * cnt_words;
            J.n = (uint32_t)keys[i].size();
            J.stats = J.n > 2;
            any_stats |= J.n > 2;
            std::copy(keys[i].begin(), keys[i].end(), J.keys);
            nmax = std::max(nmax, J.stats ? J.n : 0u);
        }
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_jobs, jobs.data(), np * sizeof(IndexJob), cudaMemcpyHostToDevice, ctx->stream));
        if (any_stats) PIXO_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, np * cnt_words * 4, ctx->stream));
        const Smem smem{(512 + (size_t)nmax * (nmax > 0 ? nmax - 1 : 0) / 2) * 4, (512 + (size_t)TRI_MAX) * 4};
        // about two waves of CTAs over the whole batch, at least 8192 pixels each
        const uint64_t want_ctas = (uint64_t)ctx->sm_count * 2;
        uint64_t per = (npix * np + want_ctas - 1) / want_ctas;
        per = std::max<uint64_t>(per, 8192);
        per = (per + RED_THREADS - 1) / RED_THREADS * RED_THREADS;
        IndexParams I;
        I.width = width; I.height = height; I.bpp = bpp; I.per_cta = (uint32_t)std::min<uint64_t>(per, npix + RED_THREADS);
        I.npix = npix;
        const uint32_t ctas = (uint32_t)((npix + I.per_cta - 1) / I.per_cta);
        for (size_t k0 = 0; k0 < np; k0 += 65535) {
            const uint32_t nb = (uint32_t)std::min<size_t>(np - k0, 65535);
            I.jobs = d_jobs + k0;
            PIXO_TRY(launch(ctx, k_reduce_index, dim3(ctas, nb), RED_THREADS, smem, I));
        }
        std::vector<uint32_t> h_cnt;
        if (any_stats) {
            h_cnt.resize(np * cnt_words);
            PIXO_CUDA(ctx, cudaMemcpyAsync(h_cnt.data(), d_cnt, np * cnt_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
            PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
        for (size_t k = 0; k < np; ++k) {
            const uint32_t i = pal_ids[k], n = jobs[k].n;
            uint8_t order[256];
            if (jobs[k].stats) {
                const uint32_t *c = h_cnt.data() + k * cnt_words;
                palette_order(n, c, c + 256, npix, order);
            } else {
                for (uint32_t e = 0; e < n; ++e) order[e] = (uint8_t)e;
            }
            pixo_b200_png_reduced &r = info[i];
            bool trns = false;
            for (uint32_t e = 0; e < n; ++e) {
                const uint32_t key = keys[i][order[e]];
                maps[k * 256 + order[e]] = (uint8_t)e;
                r.palette[e][0] = (uint8_t)(key >> 24); r.palette[e][1] = (uint8_t)(key >> 16);
                r.palette[e][2] = (uint8_t)(key >> 8); r.palette[e][3] = (uint8_t)key;
                trns |= (key & 255u) != 255u;
            }
            r.palette_len = n;
            r.trns_len = trns ? n : 0;
        }
    }

    // 4. the reduced rows
    uint8_t *d_red_img = nullptr;
    size_t pal_k = 0;
    for (uint32_t i = 0; i < n_images; ++i) {
        if (kind[i] == UNCHANGED) continue;
        pixo_b200_png_reduced &r = info[i];
        PackJob J;
        memset(&J, 0, sizeof J);
        J.bits = 8;
        switch (kind[i]) {
        case PALETTE:
            J.mode = PACK_PALETTE; J.bits = bits[i];
            J.src = d_idx + pal_k * npix;
            memcpy(J.map, &maps[pal_k * 256], 256);
            ++pal_k;
            r.color_type_byte = 3; r.effective_color_type = PIXO_B200_RGB; r.bytes_per_pixel = 1;
            break;
        case GRAY:
            J.mode = PACK_GRAY; J.bits = bits[i];
            r.color_type_byte = 0; r.effective_color_type = PIXO_B200_GRAY; r.bytes_per_pixel = 1;
            break;
        case RGB:
            J.mode = PACK_RGB;
            r.color_type_byte = 2; r.effective_color_type = PIXO_B200_RGB; r.bytes_per_pixel = 3;
            break;
        default:
            J.mode = PACK_GRAY_ALPHA;
            r.color_type_byte = 4; r.effective_color_type = PIXO_B200_GRAY_ALPHA; r.bytes_per_pixel = 2;
            break;
        }
        if (kind[i] != PALETTE) J.src = d_data + (size_t)i * in_stride;
        r.bit_depth = (uint8_t)J.bits;
        r.row_bytes = J.bits < 8 ? ((uint64_t)width * J.bits + 7) / 8 : (uint64_t)width * r.bytes_per_pixel;
        J.row_bytes = r.row_bytes;
        pack.push_back(J);
        pack_img.push_back(i);
    }
    if (!pack.empty()) {
        const size_t jobs_bytes = pack.size() * sizeof(PackJob);
        // d_red_img: the jobs, the reduced rows
        PackJob *d_jobs;
        PIXO_TRY(bind(ctx, ctx->d_red_img, [&](Layout &L) {
            d_jobs = L.take<PackJob>(pack.size()), d_red_img = L.take((size_t)n_images * red_stride);
        }));
        for (size_t k = 0; k < pack.size(); ++k) pack[k].dst = d_red_img + (size_t)pack_img[k] * red_stride;
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_jobs, pack.data(), jobs_bytes, cudaMemcpyHostToDevice, ctx->stream));
        PackParams K;
        K.jobs = d_jobs;
        K.width = width; K.height = height; K.bpp = bpp;
        uint64_t most = 0;
        for (const PackJob &J : pack) most = std::max<uint64_t>(most, J.row_bytes * height);
        uint32_t ctas = (uint32_t)std::min<uint64_t>((most + RED_THREADS * 8 - 1) / (RED_THREADS * 8),
                                                     std::max<uint64_t>(1, (uint64_t)ctx->sm_count * 8 / pack.size() + 1));
        ctas = std::max(ctas, 1u);
        for (size_t k0 = 0; k0 < pack.size(); k0 += 65535) {
            const uint32_t nb = (uint32_t)std::min<size_t>(pack.size() - k0, 65535);
            K.jobs = d_jobs + k0;
            PIXO_TRY(launch(ctx, k_reduce_pack, dim3(ctas, nb), RED_THREADS, 0, K));
        }
    }
    // the host vectors copied asynchronously above must outlive the copies
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

    // 5. filter + Adler-32: one launch per run of consecutive images with the same reduced geometry
    for (uint32_t i0 = 0; i0 < n_images;) {
        const bool reduced = kind[i0] != UNCHANGED;
        const pixo_b200_png_reduced &r0 = info[i0];
        uint32_t i1 = i0 + 1;
        while (i1 < n_images && (kind[i1] != UNCHANGED) == reduced && info[i1].row_bytes == r0.row_bytes &&
               info[i1].bytes_per_pixel == r0.bytes_per_pixel && info[i1].effective_color_type == r0.effective_color_type)
            ++i1;
        const bool oa = opt_alpha && (r0.effective_color_type == PIXO_B200_RGBA ||
                                      r0.effective_color_type == PIXO_B200_GRAY_ALPHA);
        const uint8_t *src = reduced ? d_red_img + (size_t)i0 * red_stride : d_data + (size_t)i0 * in_stride;
        PIXO_TRY(launch_png_filter_rows(ctx, src, reduced ? red_stride : in_stride, i1 - i0, width, height,
                                        r0.row_bytes, r0.bytes_per_pixel, strategy | (oa ? PIXO_B200_PNG_OPTIMIZE_ALPHA : 0u),
                                        d_out + (size_t)i0 * out_stride, out_stride, d_adler ? d_adler + i0 : nullptr,
                                        nullptr, height));
        i0 = i1;
    }
    return 0;
}

}  // namespace pixo
