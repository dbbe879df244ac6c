// jpeg_progressive.cu — the progressive scans of pixo's max preset ON the GPU: the 7 scans of
// simple_progressive_script, each coded into a stuffed, 1-padded entropy-coded segment of its own.
//
// Restates, bit for bit (quirks included):
//   encode_progressive                  src/jpeg/mod.rs:872-927
//   encode_dc_scan / encode_ac_first_scan src/jpeg/mod.rs:1248-1365
//   simple_progressive_script           src/jpeg/progressive.rs:98-110
//   encode_ac_first / flush_eob_run     src/jpeg/progressive.rs:141-210, 313-345
//   get_code_from_table                 src/jpeg/progressive.rs:363-380 (a missing symbol is (0, 4))
//   BitWriterMsb                        src/bits.rs:195-278
//
// A scan is one bit stream over ONE component's blocks, in the order of its coefficient array (MCU
// order for 4:2:0 Y, as pixo writes it).  DC scans code each block's DC against the previous block of
// the array (never reset).  AC scans (Ss > 0) carry one dependency across blocks, the EOB run: with p the
// previous non-empty block (in the band [Ss, Se]) and init = 1 when p's last non-zero lies below Se,
// the run pending before block b is (init + empties between p and b) mod 0x7FFF, and an empty block
// emits a 0x7FFF run exactly where that count reaches a multiple of 0x7FFF.  "p and its init" is a
// running maximum over (index, init), so every block's bits follow from a prefix over tiles.
//
// One thread per block, tiles of PT blocks; a batch of frames is one launch of each kernel:
//   k_prog_measure  code length of the block's own symbols, its empty / init flags, the tile's last
//                   non-empty block; coefficients outside +-16383 set status bit 0
//   k_prog_carry    per stream: exclusive running maximum of the tiles' last non-empty blocks
//   k_prog_count    per block: the EOB-run flushes it emits, added to its length; tile bit totals
//   k_prog_offsets  per stream: exclusive prefix of the tile totals (u64) and the stream's bit count
//   k_prog_place    per frame: its 7 streams laid out byte-aligned in ONE zeroed raw string, whether the
//                   frame is coded (see the capacity below), the 1-padding of each stream's last byte
//   k_prog_emit_at  per block: its bit offset (stream start + tile prefix + CTA scan), its bits OR-ed into
//                   the frame's string (MSB first)
//   k_seg_*         (jpeg_entropy.cu) splice each frame's string into its 7 stuffed, 1-padded segments
//                   back to back in the caller's slot; k_seg_fit writes a frame whole or not at all
// The tables come from the frames' DHT blocks (k_prog_dht_tables) or from the host.  A frame's raw string
// is sized from the slot's capacity (out_cap + 16 bytes, nothing read back; k_prog_place leaves out a frame
// whose raw bytes exceed out_cap), or from the bit counts read back after k_prog_offsets, so that every
// frame is coded and k_seg_fit alone decides the fit.
// Nothing spins on another CTA, so no step can hang: a fault is a CUDA error.
// One band of a frame tiled over several GPUs (pixo_b200_jpeg_band_dev_progressive*) runs measure / carry / count /
// offsets / emit in their band mode (BAND = true, see ProgParams), each stream a string of its own, then
// k_prog_band_trailer; k_prog_band_last is the band's summary for the bands after it.
#include <string.h>

#include <algorithm>

#include "common.cuh"
#include "jpeg_host.hpp"

namespace pixo {
namespace {

constexpr int PT = 256;              // blocks per tile == threads per CTA
constexpr int NSCAN = 7;
constexpr uint32_t EOBRUN_MAX = 0x7FFF;
constexpr int kComp[NSCAN] = {0, 1, 2, 0, 0, 1, 2};   // (Ss, Se) of the scans: see scan_ss / scan_se

struct ProgParams {
    const int16_t *arr[3];           // Y, Cb, Cr: natural order, compute_all_coefficients' layout
    size_t stride[3];                // int16 elements between frames
    uint64_t nb[NSCAN];              // blocks of each scan's component
    uint32_t tile_base[NSCAN + 1];   // first tile of each scan inside a frame; [NSCAN] = tiles per frame
    uint64_t blk_base[NSCAN + 1];    // first block record of each scan inside a frame; [NSCAN] = per frame
    uint32_t n;                      // frames
    uint32_t *blen;                  // [n][blocks]: the block's own bits (measure), then with its flushes (count)
    uint8_t *flag;                   // [n][blocks]: bit 0 non-empty, bit 1 its last non-zero lies below Se
    uint32_t *tile_last;             // [n][tiles]: encoded last non-empty block of the tile (see enc_of), 0 = none
    uint32_t *tile_carry;            // [n][tiles]: ... of every earlier tile of the stream
    uint32_t *tile_bits;             // [n][tiles]
    unsigned long long *tile_off;    // [n][tiles]: bits of the stream before the tile
    unsigned long long *bits;        // [n * NSCAN]: bits of each stream
    uint32_t *raw;                   // big-endian words, zeroed before the emission: one string per frame (see
                                     // ProgPlace), or per stream of a band
    unsigned long long raw_words;    // words per string
    uint32_t *status;                // bit 0: a coefficient outside -16383..16383
    const ProgTables *tables;        // [n] per frame, or [1] for every frame
    uint32_t tables_per_frame;       // 1 or 0
    // band mode (the kernels' BAND = true, one frame): the band's blocks are a contiguous range of each scan's
    // array, and what the frame's earlier bands leave crosses into it
    uint64_t gbase[NSCAN];           // frame index of the band's first block of each scan
    uint64_t gnb[NSCAN];             // the frame's blocks of each scan
    uint32_t carry_in[NSCAN];        // AC scans: enc_of (frame index) of the last non-empty block before the band
    int dc_seed[3];                  // DC predictors before the band's first block, per component
};

// tile t of the batch -> frame, scan, tile inside the scan
struct TileId {
    uint32_t frame, scan, tile;
};
__device__ __forceinline__ TileId tile_id(const ProgParams &P, uint32_t t)
{
    TileId id;
    const uint32_t per = P.tile_base[NSCAN];
    id.frame = t / per;
    const uint32_t r = t - id.frame * per;
    id.scan = 0;
#pragma unroll
    for (int s = 1; s < NSCAN; ++s)
        if (r >= P.tile_base[s]) id.scan = s;
    id.tile = r - P.tile_base[id.scan];
    return id;
}

// frame index of the band's first block of scan s (0 for a whole frame)
template <bool BAND>
__device__ __forceinline__ uint64_t scan_base(const ProgParams &P, uint32_t s) { return BAND ? P.gbase[s] : 0; }

__device__ __forceinline__ int scan_comp(uint32_t s) { return s == 0 || s == 3 || s == 4 ? 0 : (s == 1 || s == 5 ? 1 : 2); }
__device__ __forceinline__ int scan_ss(uint32_t s) { return s < 3 ? 0 : (s == 4 ? 11 : 1); }
__device__ __forceinline__ int scan_se(uint32_t s) { return s < 3 ? 0 : (s == 3 ? 10 : 63); }

// (index + 1) << 1 | init of a non-empty block; larger == later, 0 == none
__device__ __forceinline__ uint32_t enc_of(uint64_t b, uint8_t flag)
{
    return (flag & 1u) ? (uint32_t)(((b + 1) << 1) | ((flag >> 1) & 1u)) : 0u;
}

template <typename T, typename Op>
__device__ __forceinline__ T cta_scan_excl(T x, T identity, T *sh, T *total, Op op)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc = op(inc, v);
    }
    T ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) ex = identity;
    __syncthreads();
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    T before = identity, all = identity;
    for (int w = 0; w < (int)(blockDim.x / 32); ++w) {
        const T v = sh[w];
        if (w < warp) before = op(before, v);
        all = op(all, v);
    }
    *total = all;
    return op(before, ex);
}

struct MaxOp {
    __device__ uint32_t operator()(uint32_t a, uint32_t b) const { return a > b ? a : b; }
};
struct AddOp {
    template <typename T>
    __device__ T operator()(T a, T b) const { return a + b; }
};

__device__ __forceinline__ void load_tables(const ProgParams &P, uint32_t frame, ProgTables &T)
{
    const uint32_t *src = reinterpret_cast<const uint32_t *>(P.tables + (P.tables_per_frame ? frame : 0));
    uint32_t *dst = reinterpret_cast<uint32_t *>(&T);
    for (int k = threadIdx.x; k < (int)(sizeof(ProgTables) / 4); k += blockDim.x) dst[k] = src[k];
    __syncthreads();
}

__device__ __forceinline__ uint32_t category(uint32_t a) { return 32u - (uint32_t)__clz((int)a); }

// One block's own symbols (no EOB-run flush), fed to put(value, nbits) with value's nbits <= 31:
// DC scans the DC difference, AC scans the (run, size) symbols of [ss, last] with their ZRLs.
// v: the block, natural order, two coefficients per word.  Returns false when a coefficient of the
// scan's band lies outside -16383..16383.
template <typename Put>
__device__ __forceinline__ bool code_own(const uint32_t (&v)[32], int prev_dc, int ss, int last, bool dc_scan,
                                         const uint32_t *dctab, const uint32_t *actab, Put put)
{
    auto coef = [&](int nat) { return (int)(int16_t)(v[nat >> 1] >> (16 * (nat & 1))); };
    if (dc_scan) {
        const int dc = coef(0);
        const int diff = (int)(int16_t)(dc - prev_dc);          // pixo's i16 difference
        const uint32_t a = (uint32_t)abs(diff), cat = category(a);
        const uint32_t e = dctab[min(cat, 15u)];   // (16 only for rejected input)
        const uint32_t amp = (diff < 0 ? (uint32_t)(diff - 1) : (uint32_t)diff) & ((1u << cat) - 1u);
        put(((e >> 8) << cat) | amp, (e & 0xFFu) + cat);
        return dc >= -16383 && dc <= 16383;
    }
    uint32_t run = 0;
    bool ok = true;
#pragma unroll
    for (int k = 1; k < 64; ++k) {
        if (k < ss || k > last) continue;
        const int c = coef(zz_nat(k));
        if (c == 0) { ++run; continue; }
        ok &= c >= -16383 && c <= 16383;
        while (run >= 16u) {
            const uint32_t z = actab[0xF0];
            put(z >> 8, z & 0xFFu);
            run -= 16u;
        }
        const uint32_t a = (uint32_t)abs(c), cat = category(a);
        const uint32_t e = actab[(run << 4) | min(cat, 15u)];
        const uint32_t amp = (c < 0 ? (uint32_t)(c - 1) : (uint32_t)c) & ((1u << cat) - 1u);
        put(((e >> 8) << cat) | amp, (e & 0xFFu) + cat);
        run = 0;
    }
    return ok;
}

// flush_eob_run of a run r (1..0x7FFF): symbol (log2 r) << 4, then the low log2 r bits of r
template <typename Put>
__device__ __forceinline__ void code_eobrun(uint32_t r, const uint32_t *actab, Put put)
{
    const uint32_t nb = 31u - (uint32_t)__clz((int)r);
    const uint32_t e = actab[nb << 4];
    put(((e >> 8) << nb) | (r - (1u << nb)), (e & 0xFFu) + nb);
}

// The EOB-run flushes block b emits, in order: `before` (a non-empty block: the pending run; an empty
// one: 0x7FFF when its count reaches it) and `after` (the stream's last block: whatever is still pending).
// excl: enc_of of the nearest earlier non-empty block of the stream, 0 = none.
struct Flushes {
    uint32_t before, after;
};
__device__ __forceinline__ Flushes flushes_of(uint64_t b, uint64_t nb, uint8_t flag, uint32_t excl)
{
    const uint64_t p1 = excl >> 1;               // index of p + 1, 0 = none
    const uint64_t init = excl & 1u;
    const uint64_t empties = b - p1;             // empty blocks between p and b
    Flushes f{0, 0};
    uint32_t pending;
    if (flag & 1u) {
        f.before = (uint32_t)((init + empties) % EOBRUN_MAX);
        pending = (flag >> 1) & 1u;
    } else {
        const uint64_t cnt = init + empties + 1;
        pending = (uint32_t)(cnt % EOBRUN_MAX);
        if (pending == 0) f.before = EOBRUN_MAX;
    }
    if (b + 1 == nb) f.after = pending;
    return f;
}

// Loads block b (16-byte aligned, natural order) and finds its last non-zero in [ss, se] (ss - 1: none).
__device__ __forceinline__ int load_block(const int16_t *blk, int ss, int se, bool dc_scan, uint32_t (&v)[32])
{
    if (dc_scan) {
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = 0;
        v[0] = (uint16_t)blk[0];
        return 0;
    }
    const uint4 *q = reinterpret_cast<const uint4 *>(blk);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint4 w = q[k];
        v[4 * k] = w.x; v[4 * k + 1] = w.y; v[4 * k + 2] = w.z; v[4 * k + 3] = w.w;
    }
    int last = ss - 1;
#pragma unroll
    for (int k = 1; k < 64; ++k) {
        const int nat = zz_nat(k);
        if (k >= ss && k <= se && (int16_t)(v[nat >> 1] >> (16 * (nat & 1))) != 0) last = k;
    }
    return last;
}

template <bool BAND>
__global__ void __launch_bounds__(PT) k_prog_measure(const __grid_constant__ ProgParams P)
{
    __shared__ ProgTables T;
    __shared__ uint32_t sh[PT / 32];
    const TileId id = tile_id(P, blockIdx.x);
    load_tables(P, id.frame, T);
    const int comp = scan_comp(id.scan), ss = scan_ss(id.scan), se = scan_se(id.scan);
    const bool dc_scan = ss == 0;
    const int lum = comp == 0 ? 0 : 1;
    const uint64_t nb = P.nb[id.scan];
    const uint64_t b = (uint64_t)id.tile * PT + threadIdx.x;
    uint32_t len = 0, enc = 0;
    uint8_t flag = 0;
    if (b < nb) {
        const int16_t *blk = P.arr[comp] + (size_t)id.frame * P.stride[comp] + b * 64;
        uint32_t v[32];
        const int last = load_block(blk, ss, se, dc_scan, v);
        const int prev = (dc_scan && b) ? blk[-64] : (BAND && dc_scan ? P.dc_seed[comp] : 0);
        bool ok = true;
        if (dc_scan || last >= ss)
            ok = code_own(v, prev, ss, last, dc_scan, T.dc[lum], T.ac[lum], [&](uint32_t, uint32_t n) { len += n; });
        if (!dc_scan && last >= ss) flag = (uint8_t)(1u | (last < se ? 2u : 0u));
        if (!ok) atomicOr(P.status, 1u);
        const size_t r = (size_t)id.frame * P.blk_base[NSCAN] + P.blk_base[id.scan] + b;
        P.blen[r] = len;
        P.flag[r] = flag;
        enc = enc_of(b + scan_base<BAND>(P, id.scan), flag);
    }
    uint32_t tot;
    cta_scan_excl<uint32_t>(enc, 0u, sh, &tot, MaxOp());
    if (threadIdx.x == 0) P.tile_last[(size_t)id.frame * P.tile_base[NSCAN] + P.tile_base[id.scan] + id.tile] = tot;
}

// One CTA per stream: exclusive running maximum of tile_last over the stream's tiles (from the band's carry)
template <bool BAND>
__global__ void __launch_bounds__(PT) k_prog_carry(const __grid_constant__ ProgParams P)
{
    __shared__ uint32_t sh[PT / 32];
    const uint32_t frame = blockIdx.x / NSCAN, s = blockIdx.x % NSCAN;
    const uint32_t nt = P.tile_base[s + 1] - P.tile_base[s];
    const size_t base = (size_t)frame * P.tile_base[NSCAN] + P.tile_base[s];
    uint32_t run = BAND ? P.carry_in[s] : 0u;
    for (uint32_t t0 = 0; t0 < nt; t0 += PT) {
        const uint32_t t = t0 + threadIdx.x;
        const uint32_t x = t < nt ? P.tile_last[base + t] : 0u;
        uint32_t tot;
        const uint32_t ex = cta_scan_excl<uint32_t>(x, 0u, sh, &tot, MaxOp());
        if (t < nt) P.tile_carry[base + t] = max(run, ex);
        run = max(run, tot);
    }
}

// Per block: own bits + its flushes (AC scans) -> blen; tile totals
template <bool BAND>
__global__ void __launch_bounds__(PT) k_prog_count(const __grid_constant__ ProgParams P)
{
    __shared__ ProgTables T;
    __shared__ uint32_t sh[PT / 32];
    const TileId id = tile_id(P, blockIdx.x);
    load_tables(P, id.frame, T);
    const int comp = scan_comp(id.scan);
    const bool dc_scan = scan_ss(id.scan) == 0;
    const int lum = comp == 0 ? 0 : 1;
    const uint64_t nb = P.nb[id.scan];
    const uint64_t b = (uint64_t)id.tile * PT + threadIdx.x;
    const size_t tix = (size_t)id.frame * P.tile_base[NSCAN] + P.tile_base[id.scan] + id.tile;
    const size_t r = (size_t)id.frame * P.blk_base[NSCAN] + P.blk_base[id.scan] + b;
    const bool live = b < nb;
    const uint8_t flag = live ? P.flag[r] : 0;
    uint32_t len = live ? P.blen[r] : 0u, tot;
    if (!dc_scan) {   // (uniform per CTA)
        const uint64_t gb = b + scan_base<BAND>(P, id.scan);
        const uint32_t ex = max(P.tile_carry[tix], cta_scan_excl<uint32_t>(enc_of(gb, flag), 0u, sh, &tot, MaxOp()));
        if (live) {
            const Flushes f = flushes_of(gb, BAND ? P.gnb[id.scan] : nb, flag, ex);
            auto add = [&](uint32_t, uint32_t n) { len += n; };
            if (f.before) code_eobrun(f.before, T.ac[lum], add);
            if (f.after) code_eobrun(f.after, T.ac[lum], add);
            P.blen[r] = len;
        }
    }
    uint32_t sum;
    cta_scan_excl<uint32_t>(len, 0u, sh, &sum, AddOp());
    if (threadIdx.x == 0) P.tile_bits[tix] = sum;
}

// One CTA per stream: exclusive prefix of the tile totals, the stream's bit count
__global__ void __launch_bounds__(PT) k_prog_offsets(const __grid_constant__ ProgParams P)
{
    __shared__ unsigned long long sh[PT / 32];
    const uint32_t frame = blockIdx.x / NSCAN, s = blockIdx.x % NSCAN;
    const uint32_t nt = P.tile_base[s + 1] - P.tile_base[s];
    const size_t base = (size_t)frame * P.tile_base[NSCAN] + P.tile_base[s];
    unsigned long long run = 0;
    for (uint32_t t0 = 0; t0 < nt; t0 += PT) {
        const uint32_t t = t0 + threadIdx.x;
        const unsigned long long x = t < nt ? P.tile_bits[base + t] : 0ull;
        unsigned long long tot;
        const unsigned long long ex = cta_scan_excl<unsigned long long>(x, 0ull, sh, &tot, AddOp());
        if (t < nt) P.tile_off[base + t] = run + ex;
        run += tot;
    }
    if (threadIdx.x == 0) P.bits[blockIdx.x] = run;
}

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// Where whole frames' 7 streams go: one string per frame in P.raw (P.raw_words words per frame), stream s
// from bit start[frame * 8 + s] on, each padded with 1s to a whole byte, so that the splice of the frame's
// string is its 7 segments back to back.  start[frame * 8 + 7]: the string's bits.
struct ProgPlace {
    unsigned long long *start;       // [n][8]
    unsigned long long *str_bits;    // [n]: the string's bits for the splice, 0 = the frame is skipped
    unsigned long long *str_tails;   // [n]: 0 (every string starts on a byte)
    const uint32_t *trellis_status;  // bit 0: COEF_TRELLIS rejected its input, or null
    unsigned long long out_cap;      // the raw bytes a coded frame may have, at most the string's
    unsigned long long *scan_len;    // [n][7] the caller's
    uint32_t *overflow;              // [n] the caller's
};

// Per block: flushes and symbols OR-ed into the zeroed raw words at the block's bit offset.  Whole frames:
// into the frame's string at the stream's start (ProgPlace), skipping frames that are not spliced.  BAND:
// one band of a frame (see ProgParams), each stream a string of its own.
template <bool BAND>
__device__ __forceinline__ void prog_emit(const ProgParams &P, const ProgPlace &Q)
{
    __shared__ ProgTables T;
    __shared__ uint32_t sh[PT / 32];
    __shared__ unsigned long long sh64[PT / 32];
    const TileId id = tile_id(P, blockIdx.x);
    if (!BAND && Q.str_bits[id.frame] == 0) return;   // (uniform per CTA)
    load_tables(P, id.frame, T);
    const int comp = scan_comp(id.scan), ss = scan_ss(id.scan), se = scan_se(id.scan);
    const bool dc_scan = ss == 0;
    const int lum = comp == 0 ? 0 : 1;
    const uint64_t nb = P.nb[id.scan];
    const uint64_t b = (uint64_t)id.tile * PT + threadIdx.x;
    const size_t tix = (size_t)id.frame * P.tile_base[NSCAN] + P.tile_base[id.scan] + id.tile;
    const size_t r = (size_t)id.frame * P.blk_base[NSCAN] + P.blk_base[id.scan] + b;
    const bool live = b < nb;
    const uint8_t flag = live ? P.flag[r] : 0;
    const uint64_t gb = b + scan_base<BAND>(P, id.scan);
    uint32_t ex = 0, tot;
    if (!dc_scan) ex = max(P.tile_carry[tix], cta_scan_excl<uint32_t>(enc_of(gb, flag), 0u, sh, &tot, MaxOp()));
    const unsigned long long len = live ? P.blen[r] : 0ull;
    unsigned long long all;
    unsigned long long pos = P.tile_off[tix] + cta_scan_excl<unsigned long long>(len, 0ull, sh64, &all, AddOp());
    if (!live || len == 0) return;
    uint32_t *words = P.raw + (size_t)(BAND ? id.frame * NSCAN + id.scan : id.frame) * P.raw_words;
    if (!BAND) pos += Q.start[(size_t)id.frame * 8 + id.scan];
    auto put = [&](uint32_t val, uint32_t n) {
        if (n == 0) return;
        const uint32_t al = val << (32u - n);
        const uint64_t w = pos >> 5;
        const uint32_t o = (uint32_t)(pos & 31u);
        atomicOr(words + w, bswap32(al >> o));
        if (o + n > 32u) atomicOr(words + w + 1, bswap32(al << (32u - o)));
        pos += n;
    };
    const int16_t *blk = P.arr[comp] + (size_t)id.frame * P.stride[comp] + b * 64;
    uint32_t v[32];
    const int last = load_block(blk, ss, se, dc_scan, v);
    const int prev = (dc_scan && b) ? blk[-64] : (BAND && dc_scan ? P.dc_seed[comp] : 0);
    Flushes f{0, 0};
    if (!dc_scan) f = flushes_of(gb, BAND ? P.gnb[id.scan] : nb, flag, ex);
    if (f.before) code_eobrun(f.before, T.ac[lum], put);
    if (dc_scan || last >= ss) code_own(v, prev, ss, last, dc_scan, T.dc[lum], T.ac[lum], put);
    if (f.after) code_eobrun(f.after, T.ac[lum], put);
}

// One band of a frame (its streams' strings, see launch_progressive_band); whole frames go through k_prog_emit_at
template <bool BAND>
__global__ void __launch_bounds__(PT) k_prog_emit(const __grid_constant__ ProgParams P)
{
    static_assert(BAND, "whole frames are coded by k_prog_emit_at");
    prog_emit<true>(P, ProgPlace{});
}

__global__ void __launch_bounds__(PT) k_prog_emit_at(const __grid_constant__ ProgParams P, const __grid_constant__ ProgPlace Q)
{
    prog_emit<false>(P, Q);
}

// Per frame (one thread): the streams' places in the frame's string (ProgPlace), whether the frame is coded,
// and the 1-padding of each stream's last byte (the raw area is zeroed, k_prog_emit_at ORs its bits in
// afterwards).  A string of more than Q.out_cap raw bytes is left out (overflow bit 0): with the caller's slot
// capacity there, raw bytes never exceed the stuffed ones, so it could not fit, and one that is not longer fits
// its raw area (out_cap + 16 bytes).  A frame of a pass whose coefficients the trellis or this stage rejected
// gets kOvfInput.  scan_len: each stream's bytes x 2, room for any stuffing; the splice overwrites it with the
// exact lengths of the frames it splices.
__global__ void __launch_bounds__(128) k_prog_place(const __grid_constant__ ProgParams P, const __grid_constant__ ProgPlace Q)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const bool bad = *P.status || (Q.trellis_status && *Q.trellis_status);
    const unsigned long long *bits = P.bits + (size_t)i * NSCAN;
    unsigned long long off = 0;
    for (int s = 0; s < NSCAN; ++s) {
        Q.start[(size_t)i * 8 + s] = off;
        Q.scan_len[(size_t)i * NSCAN + s] = 2 * ((bits[s] + 7) >> 3);
        off += (bits[s] + 7) & ~7ull;
    }
    Q.start[(size_t)i * 8 + NSCAN] = off;
    const bool fit = !bad && (off >> 3) <= Q.out_cap;
    Q.overflow[i] = bad ? kOvfInput : (fit ? 0u : kOvfNoFit);
    Q.str_bits[i] = fit ? off : 0ull;
    Q.str_tails[i] = 0;
    if (!fit) return;
    uint8_t *raw = reinterpret_cast<uint8_t *>(P.raw + (size_t)i * P.raw_words);
    for (int s = 0; s < NSCAN; ++s) {
        const uint32_t r = (uint32_t)(bits[s] & 7);
        if (r) raw[(Q.start[(size_t)i * 8 + s] + bits[s]) >> 3] |= (uint8_t)(0xFFu >> r);
    }
}

// Per frame (one CTA): a DHT block (kDhtBytes: per table 16 counts + 256 values) as prog_tables makes it on the
// host - get_code_from_table's (code << 8) | length, the first entry of a symbol winning, (0, 4) for a missing
// symbol.  The blocks come from k_huff_tables, so every table is well formed.
__global__ void __launch_bounds__(128) k_prog_dht_tables(const uint8_t *dht, ProgTables *out)
{
    __shared__ uint8_t seen[4][256];
    const uint8_t *d = dht + (size_t)blockIdx.x * kDhtBytes;
    ProgTables &T = out[blockIdx.x];
    uint32_t *w = reinterpret_cast<uint32_t *>(&T);
    for (int k = threadIdx.x; k < (int)(sizeof(ProgTables) / 4); k += blockDim.x) w[k] = 4u;
    for (int k = threadIdx.x; k < 4 * 256; k += blockDim.x) seen[k >> 8][k & 255] = 0;
    __syncthreads();
    if (threadIdx.x >= 4) return;
    const int k = threadIdx.x;
    uint32_t *dst = k < 2 ? T.dc[k] : T.ac[k - 2];
    const int nsym = k < 2 ? 16 : 256;
    const uint8_t *bits = d + k * 272, *vals = bits + 16;
    uint32_t code = 0;
    int idx = 0;
    for (int l = 0; l < 16; ++l) {
        for (int c = 0; c < bits[l] && idx < 256; ++c, ++idx, ++code) {
            const uint8_t sym = vals[idx];
            if (seen[k][sym]) continue;
            seen[k][sym] = 1;
            if (sym < nsym) dst[sym] = (code << 8) | (uint32_t)(l + 1);
        }
        code <<= 1;
    }
}

// ---- one band of a frame tiled over several GPUs (pixo_b200_jpeg_band_dev_progressive*) ----------------------------
// A band of whole MCU rows is a contiguous range of every scan's array, so the band mode of the kernels above codes
// it with frame indices (gbase), the frame's block counts (gnb: the end-of-scan flush falls in the band that holds
// the scan's last block) and what the earlier bands leave: the DC predictors and, per AC scan, the running maximum
// of enc_of over their non-empty blocks (carry_in).  The band's summary gives the later bands those values.

struct ProgBandLast {
    const int16_t *arr[3];
    uint64_t nb[3], base[3];         // the band's blocks of each component, the frame index of its first
    ProgBandSummary *out;            // zeroed by the caller
};

// One thread per block of the component blockIdx.y: the block's enc_of in each AC scan of its component (Y: 1-10 and
// 11-63, chroma: 1-63), the largest of the band to out->last_enc, the last block's DC to out->last_dc, status bit 0
// for a coefficient outside -16383..16383
__global__ void __launch_bounds__(PT) k_prog_band_last(const __grid_constant__ ProgBandLast A)
{
    const uint32_t comp = blockIdx.y;
    const uint64_t nb = A.nb[comp];
    const uint64_t b = (uint64_t)blockIdx.x * PT + threadIdx.x;
    if ((uint64_t)blockIdx.x * PT >= nb) return;   // (uniform per CTA)
    uint32_t lo = 0, hi = 0;   // Y: scans 1-10 and 11-63; chroma: scan 1-63 in lo
    bool ok = true;
    if (b < nb) {
        const uint4 *q = reinterpret_cast<const uint4 *>(A.arr[comp] + b * 64);
        uint32_t v[32];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint4 w = q[k];
            v[4 * k] = w.x; v[4 * k + 1] = w.y; v[4 * k + 2] = w.z; v[4 * k + 3] = w.w;
        }
        int last_a = 0, last_b = 0;   // last non-zero zig-zag position in 1..10, in 11..63 (0: none)
#pragma unroll
        for (int k = 0; k < 64; ++k) {
            const int nat = zz_nat(k);
            const int c = (int16_t)(v[nat >> 1] >> (16 * (nat & 1)));
            ok &= c >= -16383 && c <= 16383;
            if (k >= 1 && c != 0) (k <= 10 ? last_a : last_b) = k;
        }
        const uint64_t gb = b + A.base[comp];
        auto flag = [](int last, int se) { return (uint8_t)(last ? 1u | (last < se ? 2u : 0u) : 0u); };
        if (comp == 0) {
            lo = enc_of(gb, flag(last_a, 10));
            hi = enc_of(gb, flag(last_b, 63));
        } else {
            lo = enc_of(gb, flag(last_b ? last_b : last_a, 63));
        }
        if (b + 1 == nb) A.out->last_dc[comp] = (int16_t)v[0];
    }
    lo = __reduce_max_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    const bool bad = __any_sync(0xffffffffu, !ok);
    if ((threadIdx.x & 31) == 0) {
        if (lo) atomicMax(&A.out->last_enc[comp == 0 ? 0 : 1 + comp], lo);
        if (hi) atomicMax(&A.out->last_enc[1], hi);
        if (bad) atomicOr(&A.out->status, 1u);
    }
}

// Where a coded band's 7 strings live: scan s's string at P.raw + s * P.raw_words (a splice area of its own, see
// SegRaw), its bit count and tail to that area's trailer, the tails also to tail7 for the host
struct ProgBandRaw {
    unsigned long long *bits[NSCAN], *tails[NSCAN];
    unsigned long long *tail7;       // [NSCAN]
};

// Thread s: scan s's bit count and last (up to) 7 bits, the last one in bit 0
__global__ void __launch_bounds__(32) k_prog_band_trailer(const __grid_constant__ ProgParams P,
                                                          const __grid_constant__ ProgBandRaw R)
{
    const uint32_t s = threadIdx.x;
    if (s >= NSCAN) return;
    const unsigned long long n = P.bits[s];
    const uint8_t *raw = reinterpret_cast<const uint8_t *>(P.raw + (size_t)s * P.raw_words);
    unsigned long long t = 0;
    for (unsigned long long i = n > 7 ? n - 7 : 0; i < n; ++i) t = (t << 1) | ((raw[i >> 3] >> (7 - (i & 7))) & 1u);
    *R.bits[s] = n;
    *R.tails[s] = t;
    R.tail7[s] = t;
}

}  // namespace

// get_code_from_table over each table: (code << 8) | length per symbol, pixo's (0, 4) for a symbol the
// table does not hold.  False when a table holds more than 256 values or a code does not fit its length.
bool prog_tables(const uint8_t bits[4][16], const uint8_t *const vals[4], ProgTables *T)
{
    memset(T, 0, sizeof *T);
    for (int k = 0; k < 4; ++k) {
        uint32_t *dst = k < 2 ? T->dc[k] : T->ac[k - 2];
        const int nsym = k < 2 ? 16 : 256;
        for (int s = 0; s < nsym; ++s) dst[s] = 4u;
        int total = 0;
        for (int l = 0; l < 16; ++l) total += bits[k][l];
        if (total > 256) return false;
        uint32_t code = 0;
        int idx = 0;
        std::vector<bool> seen(256, false);
        for (int l = 0; l < 16; ++l) {
            for (int c = 0; c < bits[k][l]; ++c, ++idx, ++code) {
                if (code >= (1u << (l + 1))) return false;
                const uint8_t sym = vals[k][idx];
                if (seen[sym]) continue;   // the first entry of a symbol wins
                seen[sym] = true;
                if (sym < nsym) dst[sym] = (code << 8) | (uint32_t)(l + 1);
            }
            code <<= 1;
        }
    }
    return true;
}

// The scans' block and tile counts of one band of a frame into P (a whole frame is the band of all its blocks),
// and what the frame's earlier bands leave it
static void prog_counts(const ProgBand &B, ProgParams &P)
{
    uint32_t tb = 0;
    uint64_t bb = 0;
    for (int s = 0; s < NSCAN; ++s) {
        const bool y = kComp[s] == 0;
        P.nb[s] = y ? B.ny : B.nc;
        P.gbase[s] = y ? B.y_base : B.c_base;
        P.gnb[s] = y ? B.frame_ny : B.frame_nc;
        P.carry_in[s] = s >= 3 ? B.ac_carry[s - 3] : 0u;
        P.tile_base[s] = tb;
        P.blk_base[s] = bb;
        tb += (uint32_t)((P.nb[s] + PT - 1) / PT);
        bb += P.nb[s];
    }
    P.tile_base[NSCAN] = tb;
    P.blk_base[NSCAN] = bb;
    for (int k = 0; k < 3; ++k) P.dc_seed[k] = B.dc_seed[k];
}

// The per-block state of P.n frames (or of one band) in L, and room for P.n tables, which it returns
static ProgTables *take_state(Layout &L, ProgParams &P)
{
    const size_t tiles = (size_t)P.n * P.tile_base[NSCAN], blocks = (size_t)P.n * P.blk_base[NSCAN];
    P.status = L.take<uint32_t>(1);
    P.blen = L.take<uint32_t>(blocks);
    P.flag = L.take(blocks);
    P.tile_last = L.take<uint32_t>(tiles);
    P.tile_carry = L.take<uint32_t>(tiles);
    P.tile_bits = L.take<uint32_t>(tiles);
    P.tile_off = L.take<unsigned long long>(tiles);
    P.bits = L.take<unsigned long long>((size_t)P.n * NSCAN);
    ProgTables *tables = L.take<ProgTables>(P.n);
    P.tables = tables;
    return tables;
}

// The measuring half of a whole-frame pass: the per-block state and the streams' places in d_prog, the tables
// (from the frames' DHT blocks when d_dht is not null, else the host's T), k_prog_measure / carry / count / offsets
static int prog_measure(pixo_b200_ctx *ctx, ProgParams &P, ProgPlace &Q, const uint8_t *d_dht, const ProgTables *T,
                        bool per_frame)
{
    cudaStream_t st = ctx->stream;
    const uint32_t n = P.n;
    const unsigned tiles = n * P.tile_base[NSCAN];   // (every frame has a Y block)
    ProgTables *d_tables;
    PIXO_TRY(bind(ctx, ctx->d_prog, [&](Layout &L) {
        d_tables = take_state(L, P);
        Q.start = L.take<unsigned long long>((size_t)n * 8);
    }));
    PIXO_CUDA(ctx, cudaMemsetAsync(P.status, 0, 4, st));
    if (d_dht)
        PIXO_TRY(launch(ctx, k_prog_dht_tables, n, 128, 0, d_dht, d_tables));
    else
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_tables, T, (per_frame ? n : 1) * sizeof(ProgTables), cudaMemcpyHostToDevice, st));
    PIXO_TRY(launch(ctx, k_prog_measure<false>, tiles, PT, 0, P));
    PIXO_TRY(launch(ctx, k_prog_carry<false>, n * NSCAN, PT, 0, P));
    PIXO_TRY(launch(ctx, k_prog_count<false>, tiles, PT, 0, P));
    return launch(ctx, k_prog_offsets, n * NSCAN, PT, 0, P);
}

// The measuring half's status word and the bit counts of its P.n x 7 streams to h_prog, after one wait; a
// coefficient out of range is refused.  *h_bits: the counts, valid until h_prog is bound again.
static int prog_read_bits(pixo_b200_ctx *ctx, const ProgParams &P, uint64_t **h_bits)
{
    uint32_t *h_status;
    PIXO_TRY(bind(ctx, ctx->h_prog, [&](Layout &L) {
        h_status = L.take<uint32_t>(1);
        *h_bits = L.take<uint64_t>((size_t)P.n * NSCAN);
    }, 8));
    PIXO_CUDA(ctx, cudaMemcpyAsync(h_status, P.status, 4, cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaMemcpyAsync(*h_bits, P.bits, (size_t)P.n * NSCAN * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*h_status)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "coefficient out of the progressive range (-16383..16383)");
    return 0;
}

// The coding half: every frame's string of raw_each bytes in d_prog_raw, k_prog_place (a frame of more than
// place_cap raw bytes is left out), k_prog_emit_at and the splice into dst (launch_splice_bounded: five launches).
// dst.out null: slots of dst.cap bytes, their lengths and flags in d_prog_out, to dst.
static int prog_code(pixo_b200_ctx *ctx, ProgParams &P, ProgPlace &Q, size_t raw_each, uint64_t place_cap,
                     const uint32_t *d_trellis_status, ProgSlots &dst)
{
    const uint32_t n = P.n;
    const SegPlan sp = splice_plan(n, raw_each);
    const bool own = dst.out == nullptr;
    uint8_t *scratch;
    uint64_t *d_len;
    // d_prog_out: the splice's scratch, every frame's spliced length, and the slots the pass owns
    PIXO_TRY(bind(ctx, ctx->d_prog_out, [&](Layout &L) {
        scratch = L.take(seg_scratch_bytes(sp));
        d_len = L.take<uint64_t>(n);
        if (own) {
            dst.out = L.take((size_t)n * dst.cap);
            dst.scan_len = L.take<uint64_t>((size_t)n * NSCAN);
            dst.overflow = L.take<uint32_t>(n);
        }
    }));
    PIXO_TRY(ctx->d_prog_raw.ensure(ctx, seg_raw(sp, nullptr).total));
    const SegRaw raw = seg_raw(sp, ctx->d_prog_raw.ptr);
    P.raw = reinterpret_cast<uint32_t *>(raw.strings);
    P.raw_words = raw_each / 4;
    Q.str_bits = raw.bits;
    Q.str_tails = raw.tails;
    Q.trellis_status = d_trellis_status;
    Q.out_cap = place_cap;
    Q.scan_len = reinterpret_cast<unsigned long long *>(dst.scan_len);
    Q.overflow = dst.overflow;
    PIXO_CUDA(ctx, cudaMemsetAsync(raw.strings, 0, (size_t)n * raw_each, ctx->stream));
    PIXO_TRY(launch(ctx, k_prog_place, (n + 127) / 128, 128, 0, P, Q));
    PIXO_TRY(launch(ctx, k_prog_emit_at, n * P.tile_base[NSCAN], PT, 0, P, Q));
    return launch_splice_bounded(ctx, sp, scratch, raw.strings, dst.out, dst.cap, d_len, dst.overflow, Q.start, NSCAN,
                                 dst.scan_len);
}

int launch_progressive(pixo_b200_ctx *ctx, const int16_t *d_y, size_t y_stride, const int16_t *d_cb,
                       const int16_t *d_cr, size_t c_stride, uint32_t n, const FrameGeometry &g, const uint8_t *d_dht,
                       const ProgTables *T, bool per_frame, const uint32_t *d_trellis_status, ProgSlots *dst)
{
    ProgParams P;
    memset(&P, 0, sizeof P);
    prog_counts(ProgBand{g.ny, g.nc, 0, 0, g.ny, g.nc, {}, {}}, P);
    P.arr[0] = d_y; P.arr[1] = d_cb; P.arr[2] = d_cr;
    P.stride[0] = y_stride; P.stride[1] = P.stride[2] = c_stride;
    P.n = n;
    P.tables_per_frame = d_dht || per_frame ? 1u : 0u;
    if ((size_t)n * P.tile_base[NSCAN] > 0x7FFFFFFFull)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "progressive stage: too many blocks per call");
    ProgPlace Q;
    PIXO_TRY(prog_measure(ctx, P, Q, d_dht, T, per_frame));
    if (d_dht) return prog_code(ctx, P, Q, Layout::round(dst->cap + 16), dst->cap, d_trellis_status, *dst);

    uint64_t *h_bits;
    PIXO_TRY(prog_read_bits(ctx, P, &h_bits));
    if (!dst) return 0;
    uint64_t longest = 0;   // raw bytes of the longest frame string (its streams byte-aligned, see k_prog_place)
    for (uint32_t i = 0; i < n; ++i) {
        uint64_t bytes = 0;
        for (int s = 0; s < NSCAN; ++s) bytes += (h_bits[(size_t)i * NSCAN + s] + 7) / 8;
        longest = std::max(longest, bytes);
    }
    if (!dst->out) dst->cap = Layout::round(2 * longest);   // stuffing at most doubles a byte: every frame fits
    const size_t raw_each = Layout::round(longest + 16);
    return prog_code(ctx, P, Q, raw_each, raw_each, nullptr, *dst);
}

// The band summary: the last DC of each component, the largest enc_of (frame index) of each AC scan.  Waits for
// the device.
int launch_progressive_band_summary(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                                    uint64_t ny, uint64_t nc, uint64_t y_base, uint64_t c_base, ProgBandSummary *out)
{
    cudaStream_t st = ctx->stream;
    ProgBandLast A;
    A.arr[0] = d_y; A.arr[1] = d_cb; A.arr[2] = d_cr;
    A.nb[0] = ny; A.nb[1] = A.nb[2] = nc;
    A.base[0] = y_base; A.base[1] = A.base[2] = c_base;
    PIXO_TRY(bind(ctx, ctx->d_prog, [&](Layout &L) { A.out = L.take<ProgBandSummary>(1); }));
    ProgBandSummary *h;
    PIXO_TRY(bind(ctx, ctx->h_prog, [&](Layout &L) { h = L.take<ProgBandSummary>(1); }, 8));
    PIXO_CUDA(ctx, cudaMemsetAsync(A.out, 0, sizeof(ProgBandSummary), st));
    const uint64_t tiles = (std::max(ny, nc) + PT - 1) / PT;
    if (tiles > 0x7FFFFFFFull) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "progressive band: too many blocks");
    if (tiles) PIXO_TRY(launch(ctx, k_prog_band_last, dim3((unsigned)tiles, nc ? 3 : 1), PT, 0, A));
    PIXO_CUDA(ctx, cudaMemcpyAsync(h, A.out, sizeof(ProgBandSummary), cudaMemcpyDeviceToHost, st));
    PIXO_CUDA(ctx, cudaStreamSynchronize(st));
    if (h->status)
        return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "coefficient out of the progressive range (-16383..16383)");
    *out = *h;
    return 0;
}

// Code one band of a frame: its tables from d_hist (k_huff_tables, the standard ones when null; to d_dht_out when
// it is not null), the band mode of measure / carry / count / offsets, a wait for the bit counts, then the 7
// strings, each in a splice area of its own in d_raw (registered in ctx->bands, so launch_band_splice takes it),
// and their tails.  Nothing is written for a coefficient out of range or a raw_cap below *raw_need.
int launch_progressive_band(pixo_b200_ctx *ctx, const int16_t *d_y, const int16_t *d_cb, const int16_t *d_cr,
                            const ProgBand &B, const uint64_t *d_hist, uint8_t *d_dht_out, uint8_t *d_raw,
                            size_t raw_cap, size_t *raw_need, uint64_t nbits[NSCAN], uint32_t tail7[NSCAN])
{
    cudaStream_t st = ctx->stream;
    ProgParams P;
    memset(&P, 0, sizeof P);
    prog_counts(B, P);
    P.arr[0] = d_y; P.arr[1] = d_cb; P.arr[2] = d_cr;
    P.n = 1;
    const size_t tiles = P.tile_base[NSCAN], blocks = P.blk_base[NSCAN];
    if (tiles > 0x7FFFFFFFull) return set_error(ctx, PIXO_B200_ERR_INVALID_ARGUMENT, "progressive band: too many blocks");
    ProgTables *d_tables;
    uint8_t *dht;
    ProgBandRaw R;
    PIXO_TRY(bind(ctx, ctx->d_prog, [&](Layout &L) {
        d_tables = take_state(L, P);
        dht = L.take(kDhtBytes);
        R.tail7 = L.take<unsigned long long>(NSCAN);
    }));
    PIXO_CUDA(ctx, cudaMemsetAsync(P.status, 0, 4, st));
    PIXO_TRY(launch_huff_tables(ctx, d_hist, 1, B.frame_nc > 0, dht, nullptr));
    PIXO_TRY(launch(ctx, k_prog_dht_tables, 1, 128, 0, dht, d_tables));
    if (tiles) {
        PIXO_TRY(launch(ctx, k_prog_measure<true>, (unsigned)tiles, PT, 0, P));
        PIXO_TRY(launch(ctx, k_prog_carry<true>, NSCAN, PT, 0, P));
        PIXO_TRY(launch(ctx, k_prog_count<true>, (unsigned)tiles, PT, 0, P));
    }
    PIXO_TRY(launch(ctx, k_prog_offsets, NSCAN, PT, 0, P));
    uint64_t *h_bits;
    PIXO_TRY(prog_read_bits(ctx, P, &h_bits));
    // every scan's splice area as large as the longest string needs, so that scan s starts at s * stride
    uint64_t max_bytes = 0;
    for (int s = 0; s < NSCAN; ++s) max_bytes = std::max<uint64_t>(max_bytes, (h_bits[s] + 7) / 8);
    const SegPlan sp = splice_plan(1, Layout::round((size_t)max_bytes + 16));
    const size_t stride = seg_raw(sp, nullptr).total;
    *raw_need = blocks ? NSCAN * stride : 0;
    for (int s = 0; s < NSCAN; ++s) nbits[s] = h_bits[s], tail7[s] = 0;
    if (raw_cap < *raw_need)
        return set_error(ctx, PIXO_B200_ERR_OUTPUT_TOO_SMALL, "raw capacity %zu too small (need %zu)", raw_cap, *raw_need);
    if (d_dht_out) PIXO_CUDA(ctx, cudaMemcpyAsync(d_dht_out, dht, kDhtBytes, cudaMemcpyDeviceToDevice, st));
    if (!blocks) {   // an empty band: no string
        PIXO_CUDA(ctx, cudaStreamSynchronize(st));
        return 0;
    }
    PIXO_CUDA(ctx, cudaMemsetAsync(d_raw, 0, *raw_need, st));
    P.raw = reinterpret_cast<uint32_t *>(d_raw);
    P.raw_words = stride / 4;
    for (int s = 0; s < NSCAN; ++s) {
        uint8_t *area = d_raw + (size_t)s * stride;
        const SegRaw r = seg_raw(sp, area);
        R.bits[s] = r.bits;
        R.tails[s] = r.tails;
        ctx->bands[area] = sp;
    }
    ctx->prog_bands[d_raw] = stride;
    PIXO_TRY(launch(ctx, k_prog_emit<true>, (unsigned)tiles, PT, 0, P));
    PIXO_TRY(launch(ctx, k_prog_band_trailer, 1, 32, 0, P, R));
    uint64_t *h_tails = h_bits;   // in h_prog, over the bit counts, which nbits holds by now
    PIXO_CUDA(ctx, cudaMemcpyAsync(h_tails, R.tail7, NSCAN * 8, cudaMemcpyDeviceToHost, st));
    PIXO_CUDA(ctx, cudaStreamSynchronize(st));
    for (int s = 0; s < NSCAN; ++s) tail7[s] = (uint32_t)h_tails[s];
    return 0;
}

}  // namespace pixo
