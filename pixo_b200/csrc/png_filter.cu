// png_filter.cu — PNG per-row predictive-filter selection with fused Adler-32, and the
// standalone Adler-32 kernel.
//
// Restates pixo's
//   filter_{sub,up,average,paeth}   src/simd/fallback.rs:100-159 (normative scalar semantics;
//                                   dispatch src/simd/mod.rs:159-236)
//   score_filter                    src/simd/fallback.rs:93-98  (sum |i8|)
//   adaptive_filter / minsum        src/png/filter.rs:302-404
//   adaptive_filter_fast            src/png/filter.rs:474-527
//   filter_row / apply_filters*     src/png/filter.rs:64-206,529-608
//   adler32                         src/compress/adler32.rs:26-47
//
// Design (H100): two kernels.
//   k_png_band (the default): a CTA walks a band of 16 consecutive rows with a 3-deep ring of row
//     buffers in shared memory (previous / current / next, filled by 16-byte cp.async), so every
//     raw byte is read from HBM once and the next row streams in under the current row's
//     arithmetic.  Candidates are scored on 4-byte words, four consecutive words per thread
//     (|i8(x - pred)| = 128 - ||x - pred| - 128|: two VABSDIFF4 per candidate; Paeth is a
//     byte-SIMD predictor), the scores are reduced (REDUX + one shared-memory
//     step) and the reference's decision ladder is replayed.  Paeth - most of the scoring
//     arithmetic - is scored only while the ladder is still open: in the same pass as the others when
//     the row above needed it, in a second pass otherwise.  Only the winner is re-derived, 16 bytes
//     per thread, shifted to the output stream's byte phase through a per-warp staging array and
//     written as aligned 16-byte stores.  The row's Adler-32 contribution
//     (A = sum d, B = sum (n-i) d, position-weighted to the end of the image) rides along; the last
//     CTA of an image folds the accumulators into the checksum.
//   k_png_filter (one CTA per row, rows staged in 32 KB segments): Bigrams (65 536-bit "seen"
//     bitmaps per candidate), the sticky small-image AdaptiveFast rule, and rows too long for three
//     shared-memory buffers.
// A band of rows of a taller image (one image over several GPUs) takes the raw row above it as an
// extra input (`above`); nothing else crosses a band.
#include <type_traits>

#include "common.cuh"

namespace pixo {
namespace {

constexpr uint32_t ADLER_MOD = 65521u;
constexpr int PNG_THREADS = 256;
constexpr int SEG_BYTES = 32768;  // bytes of a row staged per pass segment

__device__ __forceinline__ uint32_t sum_abs_s8x4(uint32_t v)
{
    // sum over bytes of |(i8)byte|: sign mask via PRMT sign-replicate, then dp4a with +-1
    uint32_t neg;  // 0xFF where byte < 0 (prmt selector msb = replicate the byte's sign)
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(neg) : "r"(v), "r"(0u), "r"(0xBA98u));
    const uint32_t sgn = neg | 0x01010101u;           // -1 / +1 as s8
    return (uint32_t)__dp4a((int)v, (int)sgn, 0);
}

__device__ __forceinline__ uint32_t sel4(uint32_t mask, uint32_t x, uint32_t y)
{
    return (x & mask) | (y & ~mask);
}
// every byte -> 0xFF if its bit 7 is set, else 0 (PRMT sign replication: one instruction)
__device__ __forceinline__ uint32_t signrep4(uint32_t v)
{
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(v), "r"(0u), "r"(0xBA98u));
    return r;
}
// bit 7 of every byte = (y >= x), unsigned per byte; the other bits are garbage.  (y | H) - (x & ~H)
// is 128 + y7 - x7 per byte (y7, x7 = low seven bits), so it never borrows across bytes and its bit
// 7 says y7 >= x7; the top bits decide unless they are equal.  Two LOP3, one IADD, one LOP3.
__device__ __forceinline__ uint32_t ge7(uint32_t y, uint32_t x)
{
    const uint32_t t = (y | 0x80808080u) - (x & 0x7F7F7F7Fu);
    return (y & ~x) | (~(y ^ x) & t);
}

// fallback_paeth_predictor (src/simd/fallback.rs:143-159) for four byte lanes at once.
// With pa=|b-c|, pb=|a-c|, dab=|a-b|:  c lies within [min(a,b), max(a,b)]  <=>  max(pa,pb) <= dab,
// in which case pc = |pa-pb|, otherwise pc = pa+pb >= max(pa,pb).  The reference's ladder
// (a if pa<=pb && pa<=pc, else b if pb<=pc, else c) therefore reduces to: take the nearer of a/b
// (a on ties) unless c is within the range and that nearer distance exceeds |pa-pb|, then c.
// The three byte-wise comparisons are carried in bit 7 only (ge7) and widened to byte masks with
// two PRMTs: 23 instructions for four bytes (the __vcmp* intrinsics version took 29).
// Checked against the scalar definition for all 2^24 (a, b, c): tools/verify_paeth.c.
__device__ __forceinline__ uint32_t paeth_pred4(uint32_t a, uint32_t b, uint32_t c)
{
    const uint32_t pa = __vabsdiffu4(b, c), pb = __vabsdiffu4(a, c), dab = __vabsdiffu4(a, b);
    const uint32_t m1 = signrep4(ge7(pb, pa));       // 0xFF where pa <= pb: a is the nearer endpoint
    const uint32_t near = sel4(m1, a, b);
    const uint32_t mn = sel4(m1, pa, pb), mx = sel4(m1, pb, pa);
    const uint32_t adiff = mx - mn;                  // per byte, mx >= mn: no borrow
    // c wins iff it lies within the range (dab >= mx) and the nearer endpoint does not beat it
    // (NOT adiff >= mn)
    const uint32_t cw = signrep4(ge7(dab, mx) & ~ge7(adiff, mn));
    return sel4(cw, c, near);
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// The reference's decision ladders over a row's score_filter sums s[] (sum |i8|), up to Paeth:
// adaptive_filter (src/png/filter.rs:302-393) goes through None, Sub, Up, Average and
// adaptive_filter_fast (:474-527) through Sub, Up.  A candidate replaces the best on a strict <,
// and the ladder ends early once the best scores <= early.  When it has not ended, Paeth then
// replaces the best on a strict < (the callers decide when to score Paeth).
struct LadderPick {
    int filter;
    unsigned long long score;
    bool done;   // the ladder ended early: Paeth is out
};
template <typename Scores>
__device__ __forceinline__ LadderPick cheap_ladder(Scores s, bool fast, uint32_t row_bytes)
{
    LadderPick p;
    if (fast) {
        const unsigned long long early = (unsigned long long)row_bytes / 8 + 1;
        p.filter = 1; p.score = s[1];
        p.done = p.score <= early;
        if (!p.done) {
            if (s[2] < p.score) { p.score = s[2]; p.filter = 2; }
            p.done = p.score <= early;
        }
    } else {
        const unsigned long long early = (unsigned long long)row_bytes / 4 + 1;
        p.filter = 0; p.score = s[0];
        p.done = p.score <= early;
        for (int f = 1; f < 4 && !p.done; ++f)
            if (s[f] < p.score) {
                p.score = s[f]; p.filter = f;
                if (p.score == 0 || p.score <= early) p.done = true;
            }
    }
    return p;
}

// Copy `len` bytes src[0..len) to dst (shared, 16-byte aligned) with the widest loads the
// source alignment allows.  lo/hi bound the readable allocation for the word path.
__device__ __forceinline__ void stage_bytes(uint8_t *__restrict__ dst,
                                            const uint8_t *__restrict__ src, int len,
                                            const uint8_t *lo_bound, const uint8_t *hi_bound,
                                            int tid)
{
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const int nv = len >> 4;
        for (int k = tid; k < nv; k += PNG_THREADS)
            reinterpret_cast<uint4 *>(dst)[k] = __ldg(reinterpret_cast<const uint4 *>(src) + k);
        for (int i = (nv << 4) + tid; i < len; i += PNG_THREADS) dst[i] = src[i];
        return;
    }
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3) * 8;
    const int nw = len >> 2;
    for (int k = tid; k < nw; k += PNG_THREADS) {
        const uint8_t *p = src + 4 * k;
        const uint8_t *a0 = p - (sh >> 3);
        uint32_t val;
        if (a0 >= lo_bound && a0 + 8 <= hi_bound) {
            const uint32_t lo = __ldg(reinterpret_cast<const uint32_t *>(a0));
            const uint32_t hi = sh ? __ldg(reinterpret_cast<const uint32_t *>(a0) + 1) : 0u;
            val = __funnelshift_r(lo, hi, sh);
        } else {
            val = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) |
                  ((uint32_t)p[3] << 24);
        }
        reinterpret_cast<uint32_t *>(dst)[k] = val;
    }
    for (int i = (nw << 2) + tid; i < len; i += PNG_THREADS) dst[i] = src[i];
}

// maybe_optimize_alpha (src/png/mod.rs:633-671) on one little-endian word of a row: Rgba (one
// pixel per word, alpha = byte 3) or GrayAlpha (two pixels per word, alpha = bytes 1 and 3):
// a pixel whose alpha is 0 becomes all-zero.
template <int BPP>
__device__ __forceinline__ uint32_t zero_transparent(uint32_t w)
{
    if (BPP == 4) return (w & 0xFF000000u) ? w : 0u;
    const uint32_t keep = ((w & 0x0000FF00u) ? 0x0000FFFFu : 0u) | ((w & 0xFF000000u) ? 0xFFFF0000u : 0u);
    return w & keep;
}
__device__ __forceinline__ uint32_t zero_transparent(uint32_t w, int oa /* 0, 2 or 4 */)
{
    return oa == 4 ? zero_transparent<4>(w) : oa == 2 ? zero_transparent<2>(w) : w;
}

struct PngParams {
    const uint8_t *data;
    size_t in_stride;
    uint8_t *out;
    size_t out_stride;
    uint32_t height;
    uint32_t row0;         // first row handled by this launch
    uint32_t row_bytes_lo; // row_bytes (rows < 4 GiB)
    uint32_t bpp;
    uint32_t strategy;     // 0..4 fixed, 5/6 adaptive ladder, 7 adaptive-fast ladder
    uint32_t opt_alpha;    // 0, or the pixel size (2 / 4) whose transparent pixels are zeroed first
    const uint8_t *forced; // per-image filter type decided earlier (sticky AdaptiveFast), or null
    uint8_t *decided;      // per-image: row0's decision is written here when non-null
    unsigned long long *acc; // per-image {A, B} accumulators (may be null)
    uint32_t *counter;     // per-image CTA completion counter
    uint32_t *adler_out;   // per-image checksum
    uint32_t rows_total_for_adler; // rows contributing before finalisation
    const uint8_t *above;  // raw row above row 0 (a row band of a taller image), or null = zeros
};

// smem layout (dynamic): cur[16 + SEGP] prev[16 + SEGP] sbuf[SEGP + 32]
__global__ void __launch_bounds__(PNG_THREADS) k_png_filter(const PngParams P)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const int tid = threadIdx.x;
    const uint32_t y = P.row0 + blockIdx.x;
    const uint32_t img = blockIdx.y;
    const size_t rb = P.row_bytes_lo;
    const int segcap = (int)min((size_t)SEG_BYTES, (rb + 15) & ~(size_t)15);
    uint8_t *cur = smem;
    uint8_t *prev = smem + 16 + segcap;
    uint8_t *sbuf = smem + 2 * (16 + segcap);
    __shared__ unsigned long long red[5][PNG_THREADS / 32];
    __shared__ unsigned long long red2[2][PNG_THREADS / 32];
    __shared__ int s_filter;

    const uint8_t *image = P.data + (size_t)img * P.in_stride;
    const uint8_t *row = image + (size_t)y * rb;
    const uint8_t *prow = y ? row - rb : P.above;
    const uint8_t *lo_b = image, *hi_b = image + (size_t)P.height * rb;
    const uint8_t *plo_b = y ? lo_b : P.above, *phi_b = y ? hi_b : P.above + rb;   // bounds of the row above
    const uint32_t bpp = P.bpp;
    const uint32_t ashift = (4 - bpp) * 8;
    const int nseg = (int)((rb + segcap - 1) / segcap);
    // Stage bytes [s0, s0 + slen) of the row and of the row above into cur / prev; callers first
    // wait at a barrier for the previous segment's readers.  A 16-byte front halo holds the bytes
    // left of the segment (zeros at row start), and the tail of the last word is zeroed so masked
    // lanes read defined data.  Then optimize_alpha rewrites the staged words (halo included;
    // segments start on 16-byte multiples, so words never straddle pixels) before anyone reads them.
    auto stage_segment = [&](size_t s0, int slen) {
        if (tid < 16) {
            const long long gi = (long long)s0 - 16 + tid;
            cur[tid] = gi >= 0 ? row[gi] : 0;
            prev[tid] = (gi >= 0 && prow) ? prow[gi] : 0;
        }
        stage_bytes(cur + 16, row + s0, slen, lo_b, hi_b, tid);
        if (prow) stage_bytes(prev + 16, prow + s0, slen, plo_b, phi_b, tid);
        else for (int i = tid; i < slen; i += PNG_THREADS) prev[16 + i] = 0;
        for (int i = slen + tid; i < ((slen + 3) & ~3); i += PNG_THREADS) { cur[16 + i] = 0; prev[16 + i] = 0; }
        __syncthreads();
        if (!P.opt_alpha) return;
        const int nwords = (16 + slen + 3) >> 2;
        for (int k = tid; k < nwords; k += PNG_THREADS) {
            reinterpret_cast<uint32_t *>(cur)[k] = zero_transparent(reinterpret_cast<uint32_t *>(cur)[k], (int)P.opt_alpha);
            reinterpret_cast<uint32_t *>(prev)[k] = zero_transparent(reinterpret_cast<uint32_t *>(prev)[k], (int)P.opt_alpha);
        }
        __syncthreads();
    };

    int filter = (int)P.strategy;
    if (P.forced) filter = P.forced[img];
    const bool need_scores = filter >= 5;

    uint8_t *orow = P.out + (size_t)img * P.out_stride + (size_t)y * (rb + 1);
    const uint32_t n_out = (uint32_t)rb + 1;
    unsigned long long adlA = 0, adlB = 0;

    if (filter == PIXO_B200_FILTER_BIGRAMS) {
        // bigrams_filter / score_bigrams (src/png/filter.rs:410-471,635-649): the candidate with
        // the fewest DISTINCT adjacent byte pairs wins (strict <, order None,Sub,Up,Avg,Paeth).
        // One 65 536-bit "seen" bitmap in shared memory per candidate; a thread counts the bits
        // it is the first to set.
        uint32_t *bitmap = reinterpret_cast<uint32_t *>(sbuf + segcap + 32);
        __shared__ uint32_t bg_cnt[PNG_THREADS / 32];
        __shared__ uint32_t bg_last;
        unsigned long long best_score = ~0ull;
        int best = 0;
        for (int f = 0; f < 5; ++f) {
            for (int i = tid; i < 2048; i += PNG_THREADS) bitmap[i] = 0;
            uint32_t cnt = 0;
            for (int seg = 0; seg < nseg; ++seg) {
                const size_t s0 = (size_t)seg * segcap;
                const int slen = (int)min((size_t)segcap, rb - s0);
                __syncthreads();
                if (nseg > 1 || f == 0) stage_segment(s0, slen);
                const uint32_t *c32 = reinterpret_cast<const uint32_t *>(cur) + 4;
                const uint32_t *p32 = reinterpret_cast<const uint32_t *>(prev) + 4;
                const int nw = (slen + 3) >> 2;
                for (int k = tid; k < nw; k += PNG_THREADS) {
                    const uint32_t x = c32[k], b = p32[k];
                    const uint32_t a = __funnelshift_r(c32[k - 1], x, ashift);
                    const uint32_t c = __funnelshift_r(p32[k - 1], b, ashift);
                    uint32_t v;
                    switch (f) {
                    case 0: v = x; break;
                    case 1: v = __vsub4(x, a); break;
                    case 2: v = __vsub4(x, b); break;
                    case 3: v = __vsub4(x, __vhaddu4(a, b)); break;
                    default: v = __vsub4(x, paeth_pred4(a, b, c)); break;
                    }
                    reinterpret_cast<uint32_t *>(sbuf)[k] = v;
                }
                __syncthreads();
                // windows(2) over this segment's bytes, plus the pair straddling the previous segment
                for (int i = tid; i < slen; i += PNG_THREADS) {
                    uint32_t key;
                    if (i + 1 < slen) key = ((uint32_t)sbuf[i] << 8) | sbuf[i + 1];
                    else continue;
                    const uint32_t bit = 1u << (key & 31);
                    if (!(atomicOr(&bitmap[key >> 5], bit) & bit)) ++cnt;
                }
                if (seg > 0 && tid == 0) {
                    const uint32_t key = (bg_last << 8) | sbuf[0];
                    const uint32_t bit = 1u << (key & 31);
                    if (!(atomicOr(&bitmap[key >> 5], bit) & bit)) ++cnt;
                }
                __syncthreads();
                if (tid == 0) bg_last = sbuf[slen - 1];
            }
            uint32_t v = cnt;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if ((tid & 31) == 0) bg_cnt[tid >> 5] = v;
            __syncthreads();
            unsigned long long score = 0;
            for (int w = 0; w < PNG_THREADS / 32; ++w) score += bg_cnt[w];
            if (score < best_score) { best_score = score; best = f; }
            __syncthreads();
        }
        filter = best;
    }

    for (int pass = (need_scores && filter >= 5) ? 0 : 1; pass < 2; ++pass) {
        unsigned long long sc[5] = {0, 0, 0, 0, 0};
        for (int seg = 0; seg < nseg; ++seg) {
            const size_t s0 = (size_t)seg * segcap;
            const int slen = (int)min((size_t)segcap, rb - s0);
            const bool restage = !(nseg == 1 && pass == 1 && need_scores && P.strategy != PIXO_B200_FILTER_BIGRAMS) ||
                                 (nseg > 1);
            if (restage) {
                __syncthreads();
                stage_segment(s0, slen);
            }
            const uint32_t *c32 = reinterpret_cast<const uint32_t *>(cur) + 4;
            const uint32_t *p32 = reinterpret_cast<const uint32_t *>(prev) + 4;
            const int nw = (slen + 3) >> 2;
            for (int k = tid; k < nw; k += PNG_THREADS) {
                const uint32_t x = c32[k], b = p32[k];
                const uint32_t a = __funnelshift_r(c32[k - 1], x, ashift);
                const uint32_t c = __funnelshift_r(p32[k - 1], b, ashift);
                const int valid = slen - 4 * k;
                const uint32_t mask = valid >= 4 ? 0xFFFFFFFFu : (0xFFFFFFFFu >> (8 * (4 - valid)));
                if (pass == 0) {
                    const bool fast = P.strategy == PIXO_B200_FILTER_ADAPTIVE_FAST;
                    if (!fast) sc[0] += sum_abs_s8x4(x & mask);
                    sc[1] += sum_abs_s8x4(__vsub4(x, a) & mask);
                    sc[2] += sum_abs_s8x4(__vsub4(x, b) & mask);
                    if (!fast) sc[3] += sum_abs_s8x4(__vsub4(x, __vhaddu4(a, b)) & mask);
                    sc[4] += sum_abs_s8x4(__vsub4(x, paeth_pred4(a, b, c)) & mask);
                } else {
                    uint32_t f;
                    switch (filter) {
                    case 0: f = x; break;
                    case 1: f = __vsub4(x, a); break;
                    case 2: f = __vsub4(x, b); break;
                    case 3: f = __vsub4(x, __vhaddu4(a, b)); break;
                    default: f = __vsub4(x, paeth_pred4(a, b, c)); break;
                    }
                    f &= mask;
                    // Adler terms: stream index q = 1 + s0 + 4k + j, weight (n_out - q)
                    const uint32_t s4 = __dp4a(f, 0x01010101u, 0u);
                    const uint32_t j4 = __dp4a(f, 0x03020100u, 0u);
                    adlA += s4;
                    adlB += (unsigned long long)(rb - s0 - 4 * (size_t)k) * s4 - j4;
                    // place the bytes at their position in the output stream image
                    const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(orow + 1 + s0) & 3);
                    uint8_t *d = sbuf + off + 4 * k;
                    d[0] = (uint8_t)f; d[1] = (uint8_t)(f >> 8); d[2] = (uint8_t)(f >> 16); d[3] = (uint8_t)(f >> 24);
                }
            }
            if (pass == 1) {
                __syncthreads();
                // copy this segment's bytes out: stream bytes [1+s0, 1+s0+slen) live at
                // sbuf[off ...]; aligned words in the middle, bytes at the two ends.
                uint8_t *g0 = orow + 1 + s0;
                const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(g0) & 3);
                uint8_t *gal = g0 - off;  // 4-byte aligned
                const int total = (int)off + slen;
                const int nwords = (total + 3) >> 2;
                const uint32_t *s32 = reinterpret_cast<const uint32_t *>(sbuf);
                for (int t = tid; t < nwords; t += PNG_THREADS) {
                    const int lo = 4 * t, hi = 4 * t + 4;
                    if (lo >= (int)off && hi <= total) {
                        reinterpret_cast<uint32_t *>(gal)[t] = s32[t];
                    } else {
                        for (int i = max(lo, (int)off); i < min(hi, total); ++i) gal[i] = sbuf[i];
                    }
                }
                if (seg == 0 && tid == 0) orow[0] = (uint8_t)filter;
            }
        }
        if (pass == 0) {
            // CTA reduction of the candidate scores, then the reference's decision ladder
#pragma unroll
            for (int f = 0; f < 5; ++f) {
                const unsigned long long v = warp_sum(sc[f]);
                if ((tid & 31) == 0) red[f][tid >> 5] = v;
            }
            __syncthreads();
            if (tid == 0) {
                unsigned long long s[5];
                for (int f = 0; f < 5; ++f) {
                    unsigned long long t = 0;
                    for (int w = 0; w < PNG_THREADS / 32; ++w) t += red[f][w];
                    s[f] = t;
                }
                const LadderPick p = cheap_ladder(s, P.strategy == PIXO_B200_FILTER_ADAPTIVE_FAST, P.row_bytes_lo);
                s_filter = !p.done && s[4] < p.score ? 4 : p.filter;   // Paeth replaces on strict <
            }
            __syncthreads();
            filter = s_filter;
        }
    }
    if (P.decided && blockIdx.x == 0 && tid == 0) P.decided[img] = (uint8_t)filter;

    if (P.acc) {
        // row contribution, weighted to the end of the image:
        //   A_r = sum d ;  B_r + n_out * (H-1-y) * A_r   (see DESIGN.md, Adler combine)
        adlA = warp_sum(adlA);
        adlB = warp_sum(adlB);
        if ((tid & 31) == 0) { red2[0][tid >> 5] = adlA; red2[1][tid >> 5] = adlB; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long A = (unsigned long long)filter, B = (unsigned long long)filter * n_out;
            for (int w = 0; w < PNG_THREADS / 32; ++w) { A += red2[0][w]; B += red2[1][w]; }
            const unsigned long long after = (unsigned long long)(P.height - 1 - y) % ADLER_MOD;
            const unsigned long long Am = A % ADLER_MOD;
            const unsigned long long Bm = (B % ADLER_MOD + (((n_out % ADLER_MOD) * after) % ADLER_MOD) * Am) % ADLER_MOD;
            atomicAdd(&P.acc[2 * img], Am);
            atomicAdd(&P.acc[2 * img + 1], Bm);
            __threadfence();
            const uint32_t done = atomicAdd(&P.counter[img], 1u) + 1;
            if (done == P.rows_total_for_adler) {
                __threadfence();
                const unsigned long long At = atomicAdd(&P.acc[2 * img], 0ull);
                const unsigned long long Bt = atomicAdd(&P.acc[2 * img + 1], 0ull);
                const unsigned long long N = ((unsigned long long)P.height % ADLER_MOD) * (n_out % ADLER_MOD) % ADLER_MOD;
                const uint32_t s1 = (uint32_t)((1 + At) % ADLER_MOD);
                const uint32_t s2 = (uint32_t)((N + Bt) % ADLER_MOD);
                P.adler_out[img] = (s2 << 16) | s1;
            }
        }
    }
}

// =========================================================================================
// K4 (band kernel): a CTA walks a band of consecutive rows with a 3-deep ring of row buffers —
// previous / current / next — so every raw byte is read from HBM exactly once and the next row
// streams in (cp.async, 16-byte) under the current row's arithmetic.  Lane l of warp w owns
// words w*C + 32*i + l of the row, so shared-memory and global accesses are fully coalesced.
//   scores   : |i8(x - pred)| = 128 - | |x - pred| - 128 |  per byte, hence per word
//              score = 512 - SAD(|x - pred|, 0x80808080): two native VABSDIFF4 per candidate
//   paeth    : branch-free byte-SIMD predictor (see paeth_pred4)
//   output   : winner re-derived, shifted to the row's byte phase in the output stream with one
//              funnel shift against the neighbouring lane's word, aligned 32-bit stores
//   adler    : per-thread sums folded with the row's distance to the end of the image; one block
//              reduction per band
// Used for every strategy except the sticky small-image AdaptiveFast case and rows too long for
// three shared-memory row buffers, which stay on the row kernel above.
// =========================================================================================
// 3, not 4: at 64 registers k_png_band<0> spills; on the H100 64 4K RGBA frames take 2.32-2.34 ms
// (Adaptive) / 2.19-2.20 ms (AdaptiveFast) at 80 registers against 2.61-2.62 / 2.49 ms at 64.
constexpr int PNG_BAND_MIN_BLOCKS = 3;
constexpr int BAND_ROWS = 16;

struct BandParams {
    const uint8_t *data;
    size_t in_stride;
    uint8_t *out;
    size_t out_stride;
    uint32_t height, row_bytes, bpp, strategy;
    unsigned long long *acc;   // per-image {A, B} (may be null)
    uint32_t *counter;         // per-image band completion counter
    uint32_t *adler_out;
    uint32_t nbands;
    uint32_t async16;          // rows are 16-byte aligned: cp.async path
    const uint8_t *above;      // raw row above row 0 (a row band of a taller image), or null = zeros
};


// explicit shared-space loads with 32-bit addresses: the ring's row buffers are picked by r % 3, and
// through generic pointers the compiler emits LD.E with 64-bit address arithmetic for every operand
__device__ __forceinline__ uint32_t lds32(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint4 lds128(uint32_t a)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}

__device__ __forceinline__ void cp_async16(void *dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src)
                 : "memory");
}

// OA: 0, or the pixel size (2 / 4) whose transparent pixels are zeroed as the rows are read
template <int OA>
__global__ void __launch_bounds__(PNG_THREADS, PNG_BAND_MIN_BLOCKS) k_png_band(const BandParams P)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ uint32_t red[5][PNG_THREADS / 32];
    __shared__ unsigned long long red64[3][PNG_THREADS / 32];
    __shared__ int s_filter, s_need_paeth;
    __shared__ unsigned long long s_score[5], s_best;
    __shared__ uint4 vstage[PNG_THREADS / 32][33];   // emit_vec: a warp's filtered vectors, slot l + 1 = lane l, slot 0 = carry
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t img = blockIdx.y;
    const uint32_t rb = P.row_bytes;
    const uint32_t pitch = 16 + ((rb + 15) & ~15u) + 16;   // [16 B zero halo][row][slack]
    uint8_t *bufs[3] = {smem, smem + pitch, smem + 2 * pitch};
    const uint32_t smem_u = (uint32_t)__cvta_generic_to_shared(smem);
    const uint8_t *image = P.data + (size_t)img * P.in_stride;
    const uint8_t *lo_b = image, *hi_b = image + (size_t)P.height * rb;
    const uint32_t r0 = blockIdx.x * BAND_ROWS;
    const uint32_t r1 = min(P.height, r0 + BAND_ROWS);
    const uint32_t n_out = rb + 1;
    const uint32_t nw = (rb + 3) >> 2;
    const uint32_t ashift = (4 - P.bpp) * 8;
    // each warp owns a contiguous chunk of output words (a multiple of 32)
    const uint32_t nj = (rb + 3 + 3) / 4 + 1;                       // output words incl. phase slack
    const uint32_t chunk = (((nj + 7) / 8) + 31) & ~31u;
    const uint32_t j_lo = warp * chunk, j_hi = min(nj, j_lo + chunk);

    auto load_row = [&](uint32_t r, uint8_t *buf) {
        const uint8_t *src = image + (size_t)r * rb;
        if (P.async16) {
            const uint32_t nv = rb >> 4;
            for (uint32_t k = tid; k < nv; k += PNG_THREADS) cp_async16(buf + 16 + 16 * k, src + 16 * (size_t)k);
            for (uint32_t i = (nv << 4) + tid; i < rb; i += PNG_THREADS) buf[16 + i] = src[i];
        } else {
            stage_bytes(buf + 16, src, (int)rb, lo_b, hi_b, tid);
        }
    };
    // halos are zero for the whole band ("left" of the first pixel is 0)
    if (tid < 12) reinterpret_cast<uint32_t *>(bufs[tid >> 2])[tid & 3] = 0;
    // previous row of the band's first row (zeros above row 0), then the first row
    if (r0 == 0) {
        for (uint32_t i = tid; i < (pitch - 16) / 4; i += PNG_THREADS)
            reinterpret_cast<uint32_t *>(bufs[(r0 + 2) % 3] + 16)[i] = 0;
        if (P.above) {
            __syncthreads();
            stage_bytes(bufs[(r0 + 2) % 3] + 16, P.above, (int)rb, P.above, P.above + rb, tid);
        }
    } else {
        load_row(r0 - 1, bufs[(r0 + 2) % 3]);
    }
    load_row(r0, bufs[r0 % 3]);
    asm volatile("cp.async.commit_group;" ::: "memory");

    unsigned long long accA = 0, accBpos = 0, accBneg = 0;
    const unsigned long long Ntot = (unsigned long long)P.height * n_out;

    bool prev_needed_paeth = false;   // the band's first row takes the two-phase route
    for (uint32_t r = r0; r < r1; ++r) {
        if (r + 1 < r1) load_row(r + 1, bufs[(r + 1) % 3]);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");   // everything but the newest group
        __syncthreads();
        const uint32_t cs = smem_u + (r % 3) * pitch + 16u;          // shared address of the row's word 0
        const uint32_t ps = smem_u + ((r + 2) % 3) * pitch + 16u;    // ... of the row above

        // words before `full` hold four row bytes; the last word's missing bytes are masked off
        const uint32_t full = rb >> 2;
        const uint32_t tailmask = (rb & 3u) ? (0xFFFFFFFFu >> (8 * (4 - (rb & 3u)))) : 0u;
        auto operands = [&](uint32_t k, uint32_t &x, uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &mask) {
            x = lds32(cs + 4u * k); b = lds32(ps + 4u * k);
            uint32_t xl = lds32(cs + 4u * k - 4u), bl = lds32(ps + 4u * k - 4u);
            if (OA) {
                x = zero_transparent<OA ? OA : 4>(x); b = zero_transparent<OA ? OA : 4>(b);
                xl = zero_transparent<OA ? OA : 4>(xl); bl = zero_transparent<OA ? OA : 4>(bl);
            }
            a = __funnelshift_r(xl, x, ashift);
            c = __funnelshift_r(bl, b, ashift);
            mask = k < full ? 0xFFFFFFFFu : tailmask;
        };

        int filter = (int)P.strategy;
        if (filter >= 5) {
            uint32_t T[5] = {0, 0, 0, 0, 0};
            const bool fast = P.strategy == PIXO_B200_FILTER_ADAPTIVE_FAST;
            // every word below `full` is whole: no masking there; the ragged last word (rows whose
            // length is not a multiple of 4) is scored by one thread with its mask
            // Two phases, like the reference's ladder: the cheap candidates first (None, Sub, Up, Average:
            // 12 of the 37 arithmetic instructions a word costs), and Paeth (25) only for rows whose
            // ladder has not ended by then ("immediately wins if <= early", src/png/filter.rs:338-372 /
            // :492-511) - on smooth rows Sub or Up ends it.  The result is identical; only the time is
            // data dependent, as it is in the reference.
            // mode 0: the cheap candidates, 1: Paeth alone, 2: all of them in one pass
            auto score = [&](uint32_t k, uint32_t mask, bool all_five, int mode) {
                uint32_t x, a, b, c, unused;
                operands(k, x, a, b, c, unused);
                if (mode) T[4] += __vsadu4(__vabsdiffu4(x, paeth_pred4(a, b, c)) & mask, 0x80808080u);
                if (mode == 1) return;
                if (all_five) {
                    T[0] += __vsadu4(x & mask, 0x80808080u);
                    T[3] += __vsadu4(__vabsdiffu4(x, __vhaddu4(a, b)) & mask, 0x80808080u);
                }
                T[1] += __vsadu4(__vabsdiffu4(x, a) & mask, 0x80808080u);
                T[2] += __vsadu4(__vabsdiffu4(x, b) & mask, 0x80808080u);
            };
            // Four consecutive words per thread (one LDS.128 per row buffer): the left neighbours of
            // words 1-3 are already in registers, word 0's comes from the previous lane by shuffle,
            // so a word costs half a shared-memory load instead of four; pixels of four bytes need
            // no funnel shift at all (left = the previous word).
            const uint32_t nv = full >> 2;
            auto score4 = [&](auto a0tag, auto fivetag, auto modetag) {
                constexpr bool A0 = decltype(a0tag)::value, FIVE = decltype(fivetag)::value;
                constexpr int MODE = decltype(modetag)::value;
                for (uint32_t vb = (uint32_t)tid & ~31u; vb < nv; vb += PNG_THREADS) {
                    const uint32_t v = vb + lane;
                    const bool valid = v < nv;
                    const uint32_t vv = valid ? v : nv - 1;
                    const uint4 X4 = lds128(cs + 16u * vv), B4 = lds128(ps + 16u * vv);
                    uint32_t x[5] = {0, X4.x, X4.y, X4.z, X4.w}, b[5] = {0, B4.x, B4.y, B4.z, B4.w};
                    x[0] = __shfl_up_sync(0xffffffffu, X4.w, 1);
                    b[0] = __shfl_up_sync(0xffffffffu, B4.w, 1);
                    if (lane == 0) { x[0] = lds32(cs + 16u * vv - 4u); b[0] = lds32(ps + 16u * vv - 4u); }
                    if (OA) {
#pragma unroll
                        for (int i = 0; i < 5; ++i) { x[i] = zero_transparent<OA ? OA : 4>(x[i]); b[i] = zero_transparent<OA ? OA : 4>(b[i]); }
                    }
                    if (valid) {
#pragma unroll
                        for (int i = 1; i < 5; ++i) {
                            const uint32_t a = A0 ? x[i - 1] : __funnelshift_r(x[i - 1], x[i], ashift);
                            if (MODE) {
                                const uint32_t c = A0 ? b[i - 1] : __funnelshift_r(b[i - 1], b[i], ashift);
                                T[4] += __vsadu4(__vabsdiffu4(x[i], paeth_pred4(a, b[i], c)), 0x80808080u);
                            }
                            if (MODE != 1) {
                                if (FIVE) {
                                    T[0] += __vsadu4(x[i], 0x80808080u);
                                    T[3] += __vsadu4(__vabsdiffu4(x[i], __vhaddu4(a, b[i])), 0x80808080u);
                                }
                                T[1] += __vsadu4(__vabsdiffu4(x[i], a), 0x80808080u);
                                T[2] += __vsadu4(__vabsdiffu4(x[i], b[i]), 0x80808080u);
                            }
                        }
                    }
                }
            };
            using std::true_type; using std::false_type;
            auto score_row = [&](auto modetag) {
                constexpr int MODE = decltype(modetag)::value;
                if (ashift == 0) { if (fast) score4(true_type{}, false_type{}, modetag); else score4(true_type{}, true_type{}, modetag); }
                else { if (fast) score4(false_type{}, false_type{}, modetag); else score4(false_type{}, true_type{}, modetag); }
                // the up-to-three whole words after the last vector, and the ragged last word
                for (uint32_t k = nv * 4 + tid; k < full; k += PNG_THREADS) score(k, 0xFFFFFFFFu, !fast, MODE);
                if (full < nw && tid == (int)(full % PNG_THREADS)) score(full, tailmask, !fast, MODE);
            };
            auto reduce_scores = [&](int f0, int f1) {   // scores f0..f1-1 -> s_score[] (sum |i8|)
#pragma unroll
                for (int f = 0; f < 5; ++f) {   // static indices: T[] stays in registers
                    if (f < f0 || f >= f1) continue;
                    const uint32_t v = __reduce_add_sync(0xffffffffu, T[f]);   // REDUX: one instruction per score
                    if (lane == 0) red[f][warp] = v;
                }
                __syncthreads();
                if (tid == 0)
                    for (int f = f0; f < f1; ++f) {
                        unsigned long long t = 0;
                        for (int w = 0; w < PNG_THREADS / 32; ++w) t += red[f][w];
                        s_score[f] = 512ull * nw - t;   // score_filter: sum |i8|
                    }
            };
            // Rows resemble their neighbours: when the row above needed Paeth, all candidates are scored
            // in one pass over the row (no second read, one reduction); when its ladder ended early,
            // the cheap ones go first.
            const bool fused = prev_needed_paeth;   // uniform
            if (fused) { score_row(std::integral_constant<int, 2>{}); reduce_scores(0, 5); }
            else { score_row(std::integral_constant<int, 0>{}); reduce_scores(0, 4); }
            if (tid == 0) {
                const volatile unsigned long long *sc = s_score;
                const LadderPick p = cheap_ladder(sc, fast, rb);
                int best = p.filter;
                if (fused && !p.done && sc[4] < p.score) best = 4;   // Paeth replaces on strict <
                s_filter = best;
                s_best = p.score;
                s_need_paeth = p.done ? 0 : 1;
            }
            __syncthreads();
            prev_needed_paeth = s_need_paeth != 0;
            if (!fused && prev_needed_paeth) {      // uniform
                score_row(std::integral_constant<int, 1>{});
                reduce_scores(4, 5);
                if (tid == 0) {   // (volatile: no other thread may read these words speculatively while thread 0 writes them)
                    const volatile unsigned long long *sc = s_score;
                    if (sc[4] < *(const volatile unsigned long long *)&s_best) s_filter = 4;
                }
                __syncthreads();
            }
            filter = s_filter;
        }

        // ---- emit the winner (the filter is chosen once per row: one straight-line loop per type) ----
        uint8_t *orow = P.out + (size_t)img * P.out_stride + (size_t)r * n_out;
        const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(orow + 1) & 3);
        uint32_t *gal = reinterpret_cast<uint32_t *>(orow + 1 - sh);   // aligned; word j = bytes 4j-sh..
        uint32_t S1 = 0, S2 = 0, S3 = 0;
        auto emit_row = [&](auto ftag) {
            constexpr int F = decltype(ftag)::value;
            auto filtered = [&](uint32_t k) -> uint32_t {
                if (k >= nw) return 0u;
                uint32_t x, a, b, c, mask;
                operands(k, x, a, b, c, mask);
                const uint32_t pred = F == 0 ? 0u : F == 1 ? a : F == 2 ? b : F == 3 ? __vhaddu4(a, b) : paeth_pred4(a, b, c);
                return __vsub4(x, pred) & mask;
            };
            uint32_t carry = j_lo ? filtered(j_lo - 1) : 0u;   // f[j-1] for this warp's first word
            for (uint32_t j0 = j_lo; j0 < j_hi; j0 += 32) {
                const uint32_t j = j0 + lane;
                const uint32_t f = filtered(j);
                if (j < nw) {
                    const uint32_t s4 = __dp4a(f, 0x01010101u, 0u);
                    S1 += s4; S2 += j * s4; S3 += __dp4a(f, 0x03020100u, 0u);
                }
                uint32_t fm1 = __shfl_up_sync(0xffffffffu, f, 1);
                if (lane == 0) fm1 = carry;
                carry = __shfl_sync(0xffffffffu, f, 31);
                if (j < j_hi) {
                    const uint32_t word = __funnelshift_l(fm1, f, 8 * sh);
                    const int i0 = 4 * (int)j - (int)sh;            // first filtered-byte index in this word
                    if (i0 >= 0 && i0 + 3 < (int)rb) {
                        gal[j] = word;
                    } else {
#pragma unroll
                        for (int t = 0; t < 4; ++t)
                            if (i0 + t >= 0 && i0 + t < (int)rb) reinterpret_cast<uint8_t *>(gal + j)[t] = (uint8_t)(word >> (8 * t));
                    }
                }
            }
        };
        // ---- the same, 16 filtered bytes per thread (rows of at least VEC_MIN_VECS vectors) ---------
        // Thread = vector v (four consecutive words, one LDS.128 per row buffer as in score4).  The
        // output stream is byte-shifted against the row (type bytes: row r starts at r * (rb + 1) + 1), so
        // the ALIGNED 16-byte chunk v of the output holds the last sh16 bytes of vector v-1 and the
        // first 16 - sh16 of vector v: the previous vector comes through a per-warp shared staging
        // array (the warp's first one is recomputed), eight words are funnel-shifted into four, and
        // the chunk leaves as one 16-byte store, 512 contiguous bytes per warp instruction.  Up to 15
        // bytes at either end of the row go out singly.  Adler: two dp4a chains per vector.
        uint32_t SWv = 0, SVv = 0;   // sum v * (byte sum of vector v); sum of (index within the vector) * byte
        auto emit_vec = [&](auto ftag, auto a0tag) {
            constexpr int F = decltype(ftag)::value;
            constexpr bool A0 = decltype(a0tag)::value;
            const uint32_t nv = (rb >> 2) >> 2;                       // whole 16-byte vectors in the row
            const uint32_t sh16 = (uint32_t)(reinterpret_cast<uintptr_t>(orow + 1) & 15);
            uint8_t *abase = orow + 1 - sh16;                          // 16-byte aligned; chunk v at abase + 16 v
            auto fvec = [&](uint32_t v, bool shfl, uint32_t (&f)[4]) {
                const uint4 X4 = lds128(cs + 16u * v), B4 = lds128(ps + 16u * v);
                uint32_t x[5] = {0, X4.x, X4.y, X4.z, X4.w}, b[5] = {0, B4.x, B4.y, B4.z, B4.w};
                if (shfl) {
                    x[0] = __shfl_up_sync(0xffffffffu, X4.w, 1);
                    b[0] = __shfl_up_sync(0xffffffffu, B4.w, 1);
                }
                if (!shfl || lane == 0) { x[0] = lds32(cs + 16u * v - 4u); b[0] = lds32(ps + 16u * v - 4u); }
                if (OA) {
#pragma unroll
                    for (int i = 0; i < 5; ++i) { x[i] = zero_transparent<OA ? OA : 4>(x[i]); b[i] = zero_transparent<OA ? OA : 4>(b[i]); }
                }
#pragma unroll
                for (int i = 1; i < 5; ++i) {
                    const uint32_t a = A0 ? x[i - 1] : __funnelshift_r(x[i - 1], x[i], ashift);
                    const uint32_t c = A0 ? b[i - 1] : __funnelshift_r(b[i - 1], b[i], ashift);
                    const uint32_t pred = F == 0 ? 0u : F == 1 ? a : F == 2 ? b[i] : F == 3 ? __vhaddu4(a, b[i]) : paeth_pred4(a, b[i], c);
                    f[i - 1] = F == 0 ? x[i] : __vsub4(x[i], pred);
                }
            };
            const uint32_t per = (((nv + PNG_THREADS / 32 - 1) / (PNG_THREADS / 32)) + 31) & ~31u;   // vectors per warp
            const uint32_t v_lo = warp * per, v_hi = min(nv, v_lo + per);
            uint4 *stg = vstage[warp];
            // the row's byte phase, uniform: chunk v = bytes [16 - o, 16) of vector v-1 ++ bytes [0, 16 - o) of v
            const uint32_t o = 16u - sh16, kq = o >> 2, bs = (o & 3u) * 8u;
            if (v_lo < v_hi) {
                if (lane == 0) {
                    uint32_t f[4] = {0, 0, 0, 0};
                    if (v_lo > 0 && sh16) fvec(v_lo - 1, false, f);
                    stg[0] = make_uint4(f[0], f[1], f[2], f[3]);
                }
                uint8_t *dst = abase + 16 * (size_t)(v_lo + lane);      // this lane's aligned chunk, 512 bytes on per round
                for (uint32_t vb = v_lo; vb < v_hi; vb += 32, dst += 512) {
                    const uint32_t v = vb + lane;
                    const bool valid = v < v_hi;
                    uint32_t f[4];
                    fvec(valid ? v : v_hi - 1, true, f);
                    if (valid) {
                        const uint32_t ssum = __dp4a(f[0], 0x01010101u, __dp4a(f[1], 0x01010101u, __dp4a(f[2], 0x01010101u, __dp4a(f[3], 0x01010101u, 0u))));
                        S1 += ssum;
                        SWv += v * ssum;
                        SVv += __dp4a(f[0], 0x03020100u, __dp4a(f[1], 0x07060504u, __dp4a(f[2], 0x0B0A0908u, __dp4a(f[3], 0x0F0E0D0Cu, 0u))));
                    }
                    stg[lane + 1] = make_uint4(f[0], f[1], f[2], f[3]);
                    __syncwarp();
                    const uint4 pv = stg[lane];                          // vector v - 1
                    __syncwarp();
                    if (lane == 31) stg[0] = make_uint4(f[0], f[1], f[2], f[3]);   // carry into the next round
                    if (valid) {
                        if (v > 0 || sh16 == 0) {
                            uint4 q;
                            // (an if-ladder on the uniform kq: a switch becomes an indirect branch through a
                            // constant-bank jump table, ~15 instructions per vector)
                            if (kq == 4) q = make_uint4(f[0], f[1], f[2], f[3]);
                            else if (kq == 3) q = make_uint4(__funnelshift_r(pv.w, f[0], bs), __funnelshift_r(f[0], f[1], bs), __funnelshift_r(f[1], f[2], bs), __funnelshift_r(f[2], f[3], bs));
                            else if (kq == 2) q = make_uint4(__funnelshift_r(pv.z, pv.w, bs), __funnelshift_r(pv.w, f[0], bs), __funnelshift_r(f[0], f[1], bs), __funnelshift_r(f[1], f[2], bs));
                            else if (kq == 1) q = make_uint4(__funnelshift_r(pv.y, pv.z, bs), __funnelshift_r(pv.z, pv.w, bs), __funnelshift_r(pv.w, f[0], bs), __funnelshift_r(f[0], f[1], bs));
                            else q = make_uint4(__funnelshift_r(pv.x, pv.y, bs), __funnelshift_r(pv.y, pv.z, bs), __funnelshift_r(pv.z, pv.w, bs), __funnelshift_r(pv.w, f[0], bs));
                            *reinterpret_cast<uint4 *>(dst) = q;
                        }
                        // The row's two ragged ends go out byte by byte, read back from the lane's own staging
                        // slot (indexing f[] with a run-time index would put it in local memory for every vector).
                        const bool head = v == 0 && sh16 != 0;            // first 16 - sh16 bytes share chunk 0 with the row before
                        const bool tail = v == nv - 1 && sh16 != 0;       // the last sh16 bytes start the chunk after the last
                        if (head || tail) {
                            const uint8_t *fb = reinterpret_cast<const uint8_t *>(&stg[lane + 1]);
                            if (head) for (uint32_t i = 0; i < o; ++i) orow[1 + i] = fb[i];
                            if (tail) for (uint32_t i = o; i < 16u; ++i) orow[1 + 16 * (size_t)v + i] = fb[i];
                        }
                    }
                    __syncwarp();
                }
            }
            // what is left of the row after the last whole vector: up to three words and a ragged one
            for (uint32_t k = nv * 4 + tid; k < nw; k += PNG_THREADS) {
                uint32_t x, a, b, c, mask;
                operands(k, x, a, b, c, mask);
                const uint32_t pred = F == 0 ? 0u : F == 1 ? a : F == 2 ? b : F == 3 ? __vhaddu4(a, b) : paeth_pred4(a, b, c);
                const uint32_t f = __vsub4(x, pred) & mask;
                const uint32_t s4 = __dp4a(f, 0x01010101u, 0u);
                S1 += s4; S2 += k * s4; S3 += __dp4a(f, 0x03020100u, 0u);
                for (uint32_t t = 0; t < 4 && 4 * k + t < rb; ++t) orow[1 + 4 * (size_t)k + t] = (uint8_t)(f >> (8 * t));
            }
        };
        const bool use_vec = (rb >> 4) >= 64;   // at least 64 vectors (1 KB rows)
        using std::integral_constant;
        if (use_vec) {
            if (ashift == 0) {
                switch (filter) {
                case 0: emit_vec(integral_constant<int, 0>{}, std::true_type{}); break;
                case 1: emit_vec(integral_constant<int, 1>{}, std::true_type{}); break;
                case 2: emit_vec(integral_constant<int, 2>{}, std::true_type{}); break;
                case 3: emit_vec(integral_constant<int, 3>{}, std::true_type{}); break;
                default: emit_vec(integral_constant<int, 4>{}, std::true_type{}); break;
                }
            } else {
                switch (filter) {
                case 0: emit_vec(integral_constant<int, 0>{}, std::false_type{}); break;
                case 1: emit_vec(integral_constant<int, 1>{}, std::false_type{}); break;
                case 2: emit_vec(integral_constant<int, 2>{}, std::false_type{}); break;
                case 3: emit_vec(integral_constant<int, 3>{}, std::false_type{}); break;
                default: emit_vec(integral_constant<int, 4>{}, std::false_type{}); break;
                }
            }
        } else {
            switch (filter) {
            case 0: emit_row(std::integral_constant<int, 0>{}); break;
            case 1: emit_row(std::integral_constant<int, 1>{}); break;
            case 2: emit_row(std::integral_constant<int, 2>{}); break;
            case 3: emit_row(std::integral_constant<int, 3>{}); break;
            default: emit_row(std::integral_constant<int, 4>{}); break;
            }
        }
        if (tid == 0) orow[0] = (uint8_t)filter;
        if (P.acc) {
            // distance-to-end weights: byte i of the row's filtered data weighs Wr - i, the type byte Wr + 1
            const unsigned long long Wr = (Ntot - (unsigned long long)r * n_out - 1) % ADLER_MOD;
            accA += S1;
            accBpos += Wr * S1;
            accBneg += 4ull * S2 + S3 + 16ull * SWv + SVv;
            if (tid == 0) { accA += (unsigned)filter; accBpos += ((Wr + 1) % ADLER_MOD) * (unsigned)filter; }
        }
        __syncthreads();   // all reads of this row's buffers are done before the ring advances
    }

    if (P.acc) {
        unsigned long long v[3] = {accA, accBpos, accBneg};
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            v[q] = warp_sum(v[q]);
            if (lane == 0) red64[q][warp] = v[q];
        }
        __syncthreads();
        if (tid == 0) {
            unsigned long long A = 0, Bp = 0, Bn = 0;
            for (int w = 0; w < PNG_THREADS / 32; ++w) { A += red64[0][w]; Bp += red64[1][w]; Bn += red64[2][w]; }
            const unsigned long long Bm = (Bp % ADLER_MOD + ADLER_MOD - Bn % ADLER_MOD) % ADLER_MOD;
            atomicAdd(&P.acc[2 * img], A % ADLER_MOD);
            atomicAdd(&P.acc[2 * img + 1], Bm);
            __threadfence();
            const uint32_t done = atomicAdd(&P.counter[img], 1u) + 1;
            if (done == P.nbands) {
                __threadfence();
                const unsigned long long At = atomicAdd(&P.acc[2 * img], 0ull);
                const unsigned long long Bt = atomicAdd(&P.acc[2 * img + 1], 0ull);
                const uint32_t s1 = (uint32_t)((1 + At) % ADLER_MOD);
                const uint32_t s2 = (uint32_t)((Ntot % ADLER_MOD + Bt) % ADLER_MOD);
                P.adler_out[img] = (s2 << 16) | s1;
            }
        }
    }
}

// Standalone Adler-32 (K5): grid-stride over 16-byte vectors; per-thread A and end-weighted B.
__global__ void __launch_bounds__(256)
k_adler32(const uint8_t *__restrict__ data, size_t len, unsigned long long *acc,
          uint32_t *counter, uint32_t *out)
{
    __shared__ unsigned long long red[2][8];
    const int tid = threadIdx.x;
    unsigned long long A = 0, B = 0;
    const uintptr_t mis = reinterpret_cast<uintptr_t>(data) & 15;
    const size_t head = mis ? min(len, (size_t)(16 - mis)) : 0;
    const size_t nvec = (len - head) >> 4;
    const uint4 *v = reinterpret_cast<const uint4 *>(data + head);
    const size_t gsz = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + tid; i < nvec; i += gsz) {
        const uint4 q = __ldg(v + i);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        const unsigned long long wt = (unsigned long long)(len - (head + (i << 4)));  // weight of byte 0
        uint32_t s = 0, js = 0;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const uint32_t s4 = __dp4a(w[m], 0x01010101u, 0u);
            s += s4;
            js += __dp4a(w[m], 0x03020100u, 0u) + 4 * m * s4;
        }
        A += s;
        B += (wt % ADLER_MOD) * s + (unsigned long long)ADLER_MOD * 4096 - js;  // keep positive
        if ((B >> 60) != 0) B %= ADLER_MOD;
    }
    // head and tail bytes (at most 15 each) by the first thread of the grid
    if (blockIdx.x == 0 && tid == 0) {
        for (size_t i = 0; i < head; ++i) { A += data[i]; B += ((len - i) % ADLER_MOD) * data[i]; }
        for (size_t i = head + (nvec << 4); i < len; ++i) { A += data[i]; B += ((len - i) % ADLER_MOD) * data[i]; }
    }
    A = warp_sum(A % ADLER_MOD);
    B = warp_sum(B % ADLER_MOD);
    if ((tid & 31) == 0) { red[0][tid >> 5] = A; red[1][tid >> 5] = B; }
    __syncthreads();
    if (tid == 0) {
        unsigned long long At = 0, Bt = 0;
        for (int w = 0; w < 8; ++w) { At += red[0][w]; Bt += red[1][w]; }
        atomicAdd(&acc[0], At % ADLER_MOD);
        atomicAdd(&acc[1], Bt % ADLER_MOD);
        __threadfence();
        const uint32_t done = atomicAdd(counter, 1u) + 1;
        if (done == gridDim.x) {
            __threadfence();
            const unsigned long long a = atomicAdd(&acc[0], 0ull), b = atomicAdd(&acc[1], 0ull);
            const uint32_t s1 = (uint32_t)((1 + a) % ADLER_MOD);
            const uint32_t s2 = (uint32_t)((len % ADLER_MOD + b) % ADLER_MOD);
            *out = (s2 << 16) | s1;
        }
    }
}

}  // namespace

// `height` rows starting at d_data; d_above (single image only): the raw row above them when they
// are a band of an image of `rule_height` rows (the strategy pre-rules look at the whole image).
int launch_png_filter_rows(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t in_stride,
                           uint32_t n_images, uint32_t width, uint32_t height, size_t row_bytes,
                           uint32_t bpp, uint32_t strategy, uint8_t *d_out, size_t out_stride,
                           uint32_t *d_adler, const uint8_t *d_above, uint32_t rule_height)
{
    if (row_bytes >= (1ull << 32) - 16)
        return set_error(ctx, PIXO_B200_ERR_IMAGE_TOO_LARGE, "row_bytes too large");
    if (d_above && n_images != 1)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "a row above is given for a single image only");
    // apply_filters_with_row_bytes pre-rules, src/png/filter.rs:72-86
    const size_t area = (size_t)width * (size_t)rule_height;
    uint32_t strat = strategy & 0xFFu;
    const uint32_t oa = ((strategy & PIXO_B200_PNG_OPTIMIZE_ALPHA) && (bpp == 2 || bpp == 4)) ? bpp : 0u;
    if (area <= 4096 && (strat == PIXO_B200_FILTER_ADAPTIVE || strat == PIXO_B200_FILTER_ADAPTIVE_FAST ||
                         strat == PIXO_B200_FILTER_BIGRAMS))
        strat = PIXO_B200_FILTER_SUB;
    // default-feature build: AdaptiveFast takes the sequential (sticky) loop when height <= 32
    const bool sticky = strat == PIXO_B200_FILTER_ADAPTIVE_FAST && rule_height <= 32;
    if (sticky && rule_height != height)
        return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED, "row bands of an image of 32 rows or fewer (sticky AdaptiveFast)");

    const size_t band_pitch = 16 + ((row_bytes + 15) & ~(size_t)15) + 16;
    const size_t band_smem = 3 * band_pitch;
    const bool use_band = !sticky && strat != PIXO_B200_FILTER_BIGRAMS && band_smem <= 200 * 1024 &&
                          row_bytes < (1u << 18);
    const size_t segcap = row_bytes + 15 < (size_t)SEG_BYTES ? ((row_bytes + 15) & ~(size_t)15) : (size_t)SEG_BYTES;
    const Smem smem{2 * (16 + segcap) + segcap + 32 + 8192,   // + bigram "seen" bitmap
                    2 * (16 + (size_t)SEG_BYTES) + SEG_BYTES + 32 + 8192};
    // misc scratch, cleared: per image {accA, accB}, a counter and the decided filter
    unsigned long long *acc;
    uint32_t *counter;
    uint8_t *decided;
    size_t misc_bytes;
    PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &L) {
        acc = L.take<unsigned long long>(2 * (size_t)n_images), counter = L.take<uint32_t>(n_images);
        decided = L.take(n_images), misc_bytes = L.end();
    }, 8));
    PIXO_CUDA(ctx, cudaMemsetAsync(acc, 0, misc_bytes, ctx->stream));

    if (use_band) {
        const auto band = oa == 4 ? k_png_band<4> : oa == 2 ? k_png_band<2> : k_png_band<0>;
        const uint32_t nbands = (height + BAND_ROWS - 1) / BAND_ROWS;
        for (uint32_t i0 = 0; i0 < n_images; i0 += 65535) {
            const uint32_t nb = n_images - i0 < 65535 ? n_images - i0 : 65535;
            BandParams B;
            B.data = d_data + (size_t)i0 * in_stride; B.in_stride = in_stride;
            B.out = d_out + (size_t)i0 * out_stride; B.out_stride = out_stride;
            B.height = height; B.row_bytes = (uint32_t)row_bytes; B.bpp = bpp; B.strategy = strat;
            B.acc = d_adler ? acc + 2 * (size_t)i0 : nullptr;
            B.counter = counter + i0;
            B.adler_out = d_adler ? d_adler + i0 : nullptr;
            B.nbands = nbands;
            B.above = d_above;
            B.async16 = (row_bytes % 16 == 0 && in_stride % 16 == 0 &&
                         (reinterpret_cast<uintptr_t>(d_data) & 15) == 0) ? 1u : 0u;
            PIXO_TRY(launch(ctx, band, dim3(nbands, nb), PNG_THREADS, {band_smem, 200 * 1024}, B));
        }
        return 0;
    }
    for (uint32_t i0 = 0; i0 < n_images; i0 += 65535) {
        const uint32_t nb = n_images - i0 < 65535 ? n_images - i0 : 65535;
        PngParams P;
        P.data = d_data + (size_t)i0 * in_stride;
        P.in_stride = in_stride;
        P.out = d_out + (size_t)i0 * out_stride;
        P.out_stride = out_stride;
        P.height = height;
        P.row_bytes_lo = (uint32_t)row_bytes;
        P.bpp = bpp;
        P.strategy = strat;
        P.opt_alpha = oa;
        P.acc = d_adler ? acc + 2 * (size_t)i0 : nullptr;
        P.counter = counter + i0;
        P.adler_out = d_adler ? d_adler + i0 : nullptr;
        P.rows_total_for_adler = height;
        P.above = d_above;
        if (sticky) {
            // row 0 decides (adaptive_filter_fast), every later row reuses that filter
            P.row0 = 0; P.forced = nullptr; P.decided = decided + i0;
            PIXO_TRY(launch(ctx, k_png_filter, dim3(1, nb), PNG_THREADS, smem, P));
            if (height > 1) {
                P.row0 = 1; P.forced = decided + i0; P.decided = nullptr;
                PIXO_TRY(launch(ctx, k_png_filter, dim3(height - 1, nb), PNG_THREADS, smem, P));
            }
        } else {
            P.row0 = 0; P.forced = nullptr; P.decided = nullptr;
            PIXO_TRY(launch(ctx, k_png_filter, dim3(height, nb), PNG_THREADS, smem, P));
        }
    }
    return 0;
}

int launch_adler32(pixo_b200_ctx *ctx, const uint8_t *d_data, size_t len, uint32_t *d_out)
{
    unsigned long long *acc;   // {accA, accB}, then the counter, cleared
    uint32_t *counter;
    PIXO_TRY(bind(ctx, ctx->d_misc, [&](Layout &L) { acc = L.take<unsigned long long>(2), counter = L.take<uint32_t>(1); }, 8));
    PIXO_CUDA(ctx, cudaMemsetAsync(acc, 0, 2 * sizeof *acc + sizeof *counter, ctx->stream));
    size_t nvec = len / 16 + 1;
    uint32_t grid = (uint32_t)((nvec + 256 * 8 - 1) / (256 * 8));
    const uint32_t cap = (uint32_t)ctx->sm_count * 8;
    if (grid > cap) grid = cap;
    if (grid == 0) grid = 1;
    return launch(ctx, k_adler32, grid, 256, 0, d_data, len, acc, counter, d_out);
}

}  // namespace pixo
