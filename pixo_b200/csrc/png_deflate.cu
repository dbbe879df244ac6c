// png_deflate.cu — pixo's deflate_zlib_packed at levels 1-9 (src/compress/deflate.rs:1008-1079) for batches of
// device streams, byte-identical.  See DESIGN.md, "PNG encoding".
//
//   k_lz77          one warp per stream, longest first, from a ticket.  The warp resets its hash state, sums the
//                   Adler-32 and takes the 4 096-byte literal census; lane 0 runs pixo's parse
//                   (Lz77Compressor::compress_into_sink, src/compress/lz77.rs:403-591) and counts the symbols.
//   host            one read-back per pass; build_codes (src/compress/huffman.rs:48-244) with Rust's BinaryHeap,
//                   the block choice and each stream's exact length.
//   k_deflate_emit  one warp per stream: each token's bits at its scanned offset, ORed into a zeroed area, then
//                   copied to the caller's slot; stored streams are copied with their block headers.
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "decode_host.hpp"

namespace pixo {

namespace {

constexpr uint32_t kMaxDist = 32768, kMaxMatch = 258, kLitFlag = 0x80000000u;
constexpr uint32_t kHash = 65536, kHash3 = 32768, kHtBits = 15, kHt = 1u << kHtBits;
// one warp's hash state: head, head3, the level-1 buckets (two per hash) and prev, i32 each (768 KiB)
constexpr size_t kStateWords = kHash + kHash3 + 2 * kHt + kMaxDist;
constexpr int kLzWarpsPerBlock = 8, kLzBlocksPerSm = 2;
constexpr int kEmitWarpsPerBlock = 8;
// streams of 2^31 bytes or more are beyond pixo's i32 positions
constexpr uint64_t kMaxStream = (uint64_t)1 << 31;

// config_for_level, lz77.rs:1415-1480: chain, search depth, nice length, lazy (0 None, 1 Lazy, 2 Lazy2), HT finder
struct LevelCfg { int chain, depth, nice, lazy, ht; };
__constant__ LevelCfg c_cfg[10] = {
    {0, 0, 0, 0, 0},      {4, 4, 32, 0, 1},      {8, 6, 10, 0, 0},        {16, 12, 14, 0, 0},
    {32, 16, 30, 0, 0},   {64, 16, 30, 1, 0},    {128, 35, 65, 1, 0},     {256, 100, 130, 1, 0},
    {1024, 300, 258, 2, 0}, {4096, 600, 258, 2, 0},
};

// deflate.rs:14-34
__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_lextra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dextra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
const uint8_t kLExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
const uint8_t kDExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

// length_code / distance_code, deflate.rs:204-241: the symbol index (0-28, 0-29)
__device__ inline int lcode(uint32_t len)
{
    int c = 0;
    while (c < 28 && len >= c_lbase[c + 1]) c++;
    return c;
}
__device__ inline int dcode(uint32_t d)
{
    int c = 0;
    while (c < 29 && d >= c_dbase[c + 1]) c++;
    return c;
}

// One stream of a pass
struct LzStream {
    const uint8_t *src;
    uint64_t len;
    uint64_t tok;   // its tokens start at tokens + tok
};

// What k_lz77 leaves for the host: token and match counts, the Adler-32, whether is_high_entropy_data fired, and the
// literal/length and distance counts (before the EOB and the dist_freqs[0] = 1 rule)
struct LzRecord {
    uint32_t ntok, nmatch, adler, high_entropy;
    uint32_t lit[286], dist[30];
};

struct Lz {
    const uint8_t *d;
    uint32_t n;
    int32_t *head, *head3, *ht, *prev;
};

__device__ inline uint32_t rd32(const uint8_t *p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }
// hash4 / hash3 / hash4_ht (lz77.rs:239-256,320-326): 0 near the end of the data
__device__ inline uint32_t hash4(const Lz &z, uint32_t p) { return p + 3 >= z.n ? 0 : ((rd32(z.d + p) * 0x1E35A7BDu) >> 16) & (kHash - 1); }
__device__ inline uint32_t hash3(const Lz &z, uint32_t p)
{
    return p + 2 >= z.n ? 0 : (((z.d[p] | z.d[p + 1] << 8 | z.d[p + 2] << 16) * 0x1E35A7BDu) >> 17) & (kHash3 - 1);
}
__device__ inline uint32_t hash4_ht(const Lz &z, uint32_t p) { return p + 3 >= z.n ? 0 : ((rd32(z.d + p) * 0x1E35A7BDu) >> (32 - kHtBits)) & (kHt - 1); }

// match_length, lz77.rs:816-861
__device__ inline uint32_t match_len(const Lz &z, uint32_t a, uint32_t b)
{
    const uint32_t max = min(z.n - b, kMaxMatch);
    uint32_t len = 0;
    while (len < max && z.d[a + len] == z.d[b + len]) len++;
    return len;
}

// update_hash, lz77.rs:864-876
__device__ inline void update_hash(Lz &z, uint32_t p)
{
    if (p + 3 >= z.n) return;
    z.head3[hash3(z, p)] = (int32_t)p;
    const uint32_t h = hash4(z, p);
    z.prev[p % kMaxDist] = z.head[h];
    z.head[h] = (int32_t)p;
}

// find_best_match, lz77.rs:605-749: the length found (0: none) and its distance
__device__ uint32_t find_best(const Lz &z, uint32_t pos, uint32_t chain, uint32_t nice, uint32_t minm, uint32_t &dist)
{
    if (pos + 3 > z.n) return 0;
    const uint8_t *d = z.d;
    uint32_t run = 1;   // detect_same_byte_run, lz77.rs:272-316
    const uint32_t rmax = min(z.n - pos, kMaxMatch);
    while (run < rmax && d[pos + run] == d[pos]) run++;
    const bool is_run = run >= minm && pos >= 1 && d[pos - 1] == d[pos];
    if (is_run && run >= nice) { dist = 1; return run; }
    uint32_t best = minm - 1, bd = 0;
    if (is_run) best = run, bd = 1;
    const int32_t c3 = z.head3[hash3(z, pos)];
    if (c3 >= 0) {
        const uint32_t mp = (uint32_t)c3, dd = pos - mp;
        if (dd != 0 && dd <= kMaxDist && d[pos] == d[mp] && d[pos + 1] == d[mp + 1] && d[pos + 2] == d[mp + 2]) {
            const uint32_t len = match_len(z, mp, pos);
            if (len >= minm && !(len == 3 && dd > 8192) && (len > best || (len == best && dd < bd))) {
                best = len, bd = dd;
                if (best >= nice) { dist = bd; return best; }
            }
        }
    }
    int32_t cp = z.head[hash4(z, pos)];
    const uint32_t maxd = min(pos, kMaxDist);
    const bool has_prefix = pos + 4 <= z.n;
    const uint32_t prefix = has_prefix ? rd32(d + pos) : 0;
    for (uint32_t left = chain; cp >= 0 && left > 0; left--) {
        const uint32_t mp = (uint32_t)cp, dd = pos - mp;
        cp = z.prev[mp % kMaxDist];
        if (dd == 0) continue;
        if (dd > maxd) break;
        if (has_prefix && mp + 4 <= z.n && rd32(d + mp) != prefix) continue;
        const uint32_t len = match_len(z, mp, pos);
        if (len >= minm && !(len == 3 && dd > 8192) && (len > best || (len == best && dd < bd))) {
            best = len, bd = dd;
            if (len >= kMaxMatch || best >= nice) break;
        }
    }
    if (best >= minm) { dist = bd; return best; }
    return 0;
}

// find_best_match_ht, lz77.rs:752-812: inserts pos into its bucket before it searches
__device__ uint32_t find_best_ht(Lz &z, uint32_t pos, uint32_t nice, uint32_t minm, uint32_t &dist)
{
    if (pos + 3 > z.n) return 0;
    int32_t *b = z.ht + 2 * hash4_ht(z, pos);
    const int32_t c[2] = {b[0], b[1]};
    b[1] = c[0];
    b[0] = (int32_t)pos;
    uint32_t best = minm - 1, bd = 0;
    for (int k = 0; k < 2; k++) {
        if (c[k] < 0) continue;
        const uint32_t mp = (uint32_t)c[k], dd = pos - mp;
        if (dd == 0 || dd > kMaxDist || z.d[pos] != z.d[mp] || z.d[pos + 1] != z.d[mp + 1] || z.d[pos + 2] != z.d[mp + 2])
            continue;
        const uint32_t len = match_len(z, mp, pos);
        if (len < minm || (len == 3 && dd > 8192)) continue;
        if (len > best) {
            best = len, bd = dd;
            if (best >= nice) break;
        }
    }
    if (best >= minm) { dist = bd; return best; }
    return 0;
}

struct Sink {
    uint32_t *tok, nt, nmatch;
    uint32_t *lit, *dist;   // the warp's counts in shared memory
    __device__ void literal(uint8_t b) { tok[nt++] = kLitFlag | b; lit[b]++; }
    __device__ void match(uint32_t len, uint32_t d)
    {
        tok[nt++] = (d - 1) << 16 | len;
        lit[257 + lcode(len)]++;
        dist[dcode(d)]++;
        nmatch++;
    }
};

// the hash updates after a match: first and last position of a distance-1 run, every position otherwise
__device__ inline void match_updates(Lz &z, uint32_t pos, uint32_t len, uint32_t dist)
{
    if (dist == 1) {
        update_hash(z, pos);
        update_hash(z, pos + len - 1);
    } else {
        for (uint32_t i = 0; i < len; i++) update_hash(z, pos + i);
    }
}

// Lz77Compressor::compress_into_sink, lz77.rs:403-591 (lane 0)
__device__ void lz77_parse(Lz &z, const LevelCfg c, uint32_t minm, Sink &s)
{
    const uint32_t n = z.n, depth = c.depth, nice = c.nice;
    uint32_t pos = 0, streak = 0, probe = 0, updates = 0, pend_len = 0, pend_dist = 0;
    bool incompressible = false;
    while (pos < n) {
        if (incompressible) {
            if (probe >= 256) {   // INCOMPRESSIBLE_PROBE_INTERVAL, at INCOMPRESSIBLE_CHAIN_LIMIT 1
                probe = 0;
                uint32_t dist, len = find_best(z, pos, min(1u, depth), nice, minm, dist);
                if (len) {
                    incompressible = false, streak = 0;
                    s.match(len, dist);
                    match_updates(z, pos, len, dist);
                    pos += len;
                    continue;
                }
            }
            s.literal(z.d[pos]);
            if (++updates >= 64) update_hash(z, pos), updates = 0;   // INCOMPRESSIBLE_UPDATE_INTERVAL
            pos++, streak++, probe++;
            continue;
        }
        uint32_t chain = c.chain;
        if (streak >= 512) incompressible = true, probe = 0, chain = 1;   // INCOMPRESSIBLE_LITERAL_THRESHOLD
        uint32_t len, dist = 0;
        if (pend_len) len = pend_len, dist = pend_dist, pend_len = 0;
        else if (c.ht) len = find_best_ht(z, pos, nice, minm, dist);
        else len = find_best(z, pos, min(chain, depth), nice, minm, dist);
        if (len) {
            streak = 0, incompressible = false, probe = 0;
            if (c.lazy && len < nice && len < 16 && pos + 1 < n) {   // GOOD_MATCH_LENGTH 16
                update_hash(z, pos);
                const uint32_t next_chain = c.lazy == 2 ? max(chain / 2, 1u) : chain;
                uint32_t nd = 0;
                const uint32_t nl = c.ht ? find_best_ht(z, pos + 1, nice, minm, nd)
                                         : find_best(z, pos + 1, min(next_chain, depth), nice, minm, nd);
                if (nl && (nl >= len + 3 || nl >= nice)) {
                    s.literal(z.d[pos]);
                    pend_len = nl, pend_dist = nd;
                    pos++;
                    continue;
                }
            }
            s.match(len, dist);
            match_updates(z, pos, len, dist);
            pos += len;
        } else {
            if (++streak >= 512) incompressible = true, probe = 0, updates = 0;
            s.literal(z.d[pos]);
            update_hash(z, pos);
            pos++;
        }
    }
}

__global__ void __launch_bounds__(kLzWarpsPerBlock * 32)
k_lz77(const LzStream *__restrict__ streams, const uint32_t *__restrict__ order, uint32_t n, int level,
       uint32_t *__restrict__ tokens, LzRecord *__restrict__ recs, int32_t *__restrict__ state, uint32_t *ticket)
{
    __shared__ uint32_t s_hist[kLzWarpsPerBlock][316];
    __shared__ uint32_t s_seen[kLzWarpsPerBlock][128];   // the census' 256 bits, then is_high_entropy_data's 4096
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int32_t *st = state + (size_t)(blockIdx.x * kLzWarpsPerBlock + w) * kStateWords;
    uint32_t *hist = s_hist[w], *seen = s_seen[w];
    const LevelCfg c = c_cfg[level];
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(ticket, 1u);
        t = __shfl_sync(~0u, t, 0);
        if (t >= n) return;
        const uint32_t si = order[t];
        const LzStream S = streams[si];
        const uint32_t len = (uint32_t)S.len;
        const uint8_t *d = S.src;
        // Adler-32 of 32 consecutive pieces, combined in order (adler32_combine)
        const uint32_t piece = (len + 31) / 32, p0 = min(lane * piece, len), p1 = min(p0 + piece, len);
        uint32_t a = 1, b = 0;
        for (uint32_t i = p0; i < p1;) {
            const uint32_t e = min(i + 5552, p1);
            for (; i < e; i++) a += d[i], b += a;
            a %= 65521, b %= 65521;
        }
        uint32_t adler = 1;
        for (int k = 0; k < 32; k++) {
            const uint32_t ak = __shfl_sync(~0u, a, k), bk = __shfl_sync(~0u, b, k);
            const uint32_t lk = __shfl_sync(~0u, p1 - p0, k);
            const uint64_t M = 65521, a1 = adler & 0xFFFF, a2 = adler >> 16;
            const uint64_t s1 = (a1 + ak + M - 1) % M, s2 = (a2 + bk + (lk % M) * ((a1 + M - 1) % M)) % M;
            adler = (uint32_t)(s2 << 16 | s1);
        }
        // is_high_entropy_data, deflate.rs:1108-1145 (lane 0; only streams of 4 096 bytes or more)
        for (uint32_t i = lane; i < 128; i += 32) seen[i] = 0;
        for (uint32_t i = lane; i < 316; i += 32) hist[i] = 0;
        __syncwarp();
        uint32_t high = 0;
        if (lane == 0 && len >= 4096) {
            const uint32_t sl = min(len, 8192u);
            uint32_t coll = 0;
            for (uint32_t i = 0; i + 4 <= sl; i++) {
                const uint32_t h = ((rd32(d + i) * 0x1E35A7BDu) >> 20) & 4095;
                if (seen[h >> 5] >> (h & 31) & 1) coll++;
                else seen[h >> 5] |= 1u << (h & 31);
            }
            high = (float)coll / (float)(sl - 3) < 0.05f;
        }
        high = __shfl_sync(~0u, high, 0);
        __syncwarp();
        for (uint32_t i = lane; i < 8; i += 32) seen[i] = 0;
        __syncwarp();
        // calculate_min_match_len's census of the first 4 096 bytes, lz77.rs:329-360
        for (uint32_t i = lane; i < min(len, 4096u); i += 32) atomicOr(&seen[d[i] >> 5], 1u << (d[i] & 31));
        __syncwarp();
        uint32_t used = 0;
        for (int k = 0; k < 8; k++) used += __popc(seen[k]);
        uint32_t minm = 3;
        if (c.depth > 4) {
            if (used > 32) minm = 4;
            if (used > 64 && c.depth >= 10) minm = 5;
            if (used > 96 && c.depth >= 20) minm = 6;
        }
        Sink s{tokens + S.tok, 0, 0, hist, hist + 286};
        if (!high && len) {
            // the tables are reset for every stream
            int4 *st4 = reinterpret_cast<int4 *>(st);
            for (size_t i = lane; i < kStateWords / 4; i += 32) st4[i] = make_int4(-1, -1, -1, -1);
            __syncwarp();
            if (lane == 0) {
                Lz z{d, len, st, st + kHash, st + kHash + kHash3, st + kHash + kHash3 + 2 * kHt};
                lz77_parse(z, c, minm, s);
            }
            __syncwarp();
        }
        LzRecord *r = recs + si;
        if (lane == 0) r->ntok = s.nt, r->nmatch = s.nmatch, r->adler = adler, r->high_entropy = high;
        for (uint32_t i = lane; i < 316; i += 32) (i < 286 ? r->lit[i] : r->dist[i - 286]) = hist[i];
        __syncwarp();
    }
}

// How k_deflate_emit writes one stream
struct EmitStream {
    const uint8_t *src;     // stored streams: the input
    const uint32_t *tok;    // coded streams: the tokens
    uint64_t len, ntok;
    uint64_t area;          // coded streams: the first word of its area
    uint64_t zbytes;        // the whole zlib stream
    uint32_t kind;          // 0 stored, 1 fixed, 2 dynamic
    uint32_t hdr_bits;      // the zlib header and the block header, in hdr (words from hdr_word)
    uint64_t hdr_word;
    uint32_t adler;
    uint32_t table;         // (reversed code | length << 16) for 286 literal/length then 30 distance symbols
    uint8_t *dst;
};

__device__ inline void or_bits(uint32_t *w, uint64_t pos, uint32_t v, uint32_t nb)
{
    if (!nb) return;
    const uint64_t x = (uint64_t)v << (pos & 31);
    atomicOr(w + (pos >> 5), (uint32_t)x);
    if ((pos & 31) + nb > 32) atomicOr(w + (pos >> 5) + 1, (uint32_t)(x >> 32));
}

__global__ void __launch_bounds__(kEmitWarpsPerBlock * 32)
k_deflate_emit(const EmitStream *__restrict__ es, uint32_t n, const uint32_t *__restrict__ hdr,
               const uint32_t *__restrict__ tables, uint32_t *__restrict__ area)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = gw; i < n; i += nw) {
        const EmitStream E = es[i];
        if (E.kind == 0) {
            // zlib header, deflate_stored's 65 535-byte blocks (deflate.rs:1664-1688), Adler-32
            const uint64_t nb = E.len ? (E.len + 65534) / 65535 : 0;
            if (lane == 0) E.dst[0] = (uint8_t)hdr[E.hdr_word], E.dst[1] = (uint8_t)(hdr[E.hdr_word] >> 8);
            for (uint64_t b = 0; b < nb; b++) {
                const uint64_t m = min(E.len - b * 65535, (uint64_t)65535);
                uint8_t *o = E.dst + 2 + b * 65540;
                if (lane < 5) {
                    const uint8_t h[5] = {(uint8_t)(b == nb - 1), (uint8_t)m, (uint8_t)(m >> 8), (uint8_t)~m, (uint8_t)(~m >> 8)};
                    o[lane] = h[lane];
                }
                for (uint64_t j = lane; j < m; j += 32) o[5 + j] = E.src[b * 65535 + j];
            }
            if (lane < 4) E.dst[E.zbytes - 4 + lane] = (uint8_t)(E.adler >> (24 - 8 * lane));
            continue;
        }
        uint32_t *w = area + E.area;
        const uint32_t *T = tables + (size_t)E.table * 316;
        for (uint32_t k = lane; k * 32 < E.hdr_bits; k += 32) w[k] = hdr[E.hdr_word + k];
        __syncwarp();
        uint64_t base = E.hdr_bits;
        for (uint64_t t0 = 0; t0 < E.ntok; t0 += 32) {
            uint32_t va = 0, na = 0, vb = 0, nb = 0;
            if (t0 + lane < E.ntok) {
                const uint32_t t = E.tok[t0 + lane];
                if (t & kLitFlag) {
                    const uint32_t e = T[t & 0xFF];
                    va = e & 0xFFFF, na = e >> 16;
                } else {
                    const uint32_t len = t & 0xFFFF, dist = (t >> 16) + 1;
                    const int a = lcode(len), b = dcode(dist);
                    const uint32_t ea = T[257 + a], eb = T[286 + b];
                    va = (ea & 0xFFFF) | (len - c_lbase[a]) << (ea >> 16), na = (ea >> 16) + c_lextra[a];
                    vb = (eb & 0xFFFF) | (dist - c_dbase[b]) << (eb >> 16), nb = (eb >> 16) + c_dextra[b];
                }
            }
            uint32_t incl = na + nb;
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(~0u, incl, o);
                if (lane >= (uint32_t)o) incl += y;
            }
            const uint64_t at = base + incl - (na + nb);
            or_bits(w, at, va, na);
            or_bits(w, at + na, vb, nb);
            base += __shfl_sync(~0u, incl, 31);
        }
        if (lane == 0) {
            or_bits(w, base, T[256] & 0xFFFF, T[256] >> 16);   // end of block
            base = (base + (T[256] >> 16) + 7) / 8 * 8;
            for (int k = 0; k < 4; k++) or_bits(w, base + 8 * k, (E.adler >> (24 - 8 * k)) & 0xFF, 8);
        }
        __syncwarp();
        __threadfence_block();
        const uint8_t *src = reinterpret_cast<const uint8_t *>(w);
        for (uint64_t j = lane; j < E.zbytes; j += 32) E.dst[j] = __ldcg(src + j);
    }
}

// ---- host: build_codes (huffman.rs:48-244) with Rust std's BinaryHeap<Reverse<Node>> -------------------------

struct HNode { uint32_t f; int32_t sym, l, r; };   // sym -1: an internal node (None)

// Node's Ord (huffman.rs:30-37) on (frequency, Option<symbol>), None first; the heap holds Reverse<Node>, so x <= y
// there when node y <= node x
inline int node_cmp(const HNode &a, const HNode &b)
{
    if (a.f != b.f) return a.f < b.f ? -1 : 1;
    return a.sym < b.sym ? -1 : a.sym > b.sym;
}
struct Heap {
    const std::vector<HNode> &N;
    std::vector<int> h;
    bool le(int x, int y) const { return node_cmp(N[y], N[x]) <= 0; }
    bool lt(int x, int y) const { return node_cmp(N[y], N[x]) < 0; }
    size_t sift_up(size_t start, size_t pos)   // BinaryHeap::sift_up
    {
        const int e = h[pos];
        while (pos > start) {
            const size_t parent = (pos - 1) / 2;
            if (le(e, h[parent])) break;
            h[pos] = h[parent], pos = parent;
        }
        h[pos] = e;
        return pos;
    }
    void sift_down_range(size_t pos, size_t end)   // BinaryHeap::sift_down_range
    {
        const int e = h[pos];
        size_t child = 2 * pos + 1;
        while (child + 2 <= end) {
            child += le(h[child], h[child + 1]);
            if (le(h[child], e)) { h[pos] = e; return; }
            h[pos] = h[child], pos = child, child = 2 * pos + 1;
        }
        if (child == end - 1 && lt(e, h[child])) h[pos] = h[child], pos = child;
        h[pos] = e;
    }
    int pop()   // BinaryHeap::pop: sift_down_to_bottom, then sift_up
    {
        int item = h.back();
        h.pop_back();
        if (!h.empty()) {
            std::swap(item, h[0]);
            const size_t end = h.size();
            const int e = h[0];
            size_t pos = 0, child = 1;
            while (child + 2 <= end) {
                child += le(h[child], h[child + 1]);
                h[pos] = h[child], pos = child, child = 2 * pos + 1;
            }
            if (child == end - 1) h[pos] = h[child], pos = child;
            h[pos] = e;
            sift_up(0, pos);
        }
        return item;
    }
    void push(int x)
    {
        h.push_back(x);
        sift_up(0, h.size() - 1);
    }
};

// limit_code_lengths, huffman.rs:128-205
void limit_lengths(uint8_t *len, int n, int maxl)
{
    bool over = false;
    for (int i = 0; i < n; i++) over |= len[i] > maxl;
    if (!over) return;
    for (int i = 0; i < n; i++) len[i] = (uint8_t)std::min<int>(len[i], maxl);
    const uint32_t lim = 1u << maxl;
    uint32_t k = 0;
    for (int i = 0; i < n; i++) if (len[i]) k += 1u << (maxl - len[i]);
    while (k > lim) {
        int bi = -1, bl = maxl;
        for (int i = 0; i < n; i++) if (len[i] > 0 && len[i] < maxl && len[i] < bl) bl = len[i], bi = i;
        if (bi < 0) break;
        k -= 1u << (maxl - len[bi]);
        len[bi]++;
        k += 1u << (maxl - len[bi]);
    }
    while (k < lim) {
        int bi = -1, bl = 0;
        for (int i = 0; i < n; i++) if (len[i] > 1 && len[i] > bl) bl = len[i], bi = i;
        if (bi < 0) break;
        const uint32_t o = 1u << (maxl - len[bi]), nw = 1u << (maxl - (len[bi] - 1));
        if (k - o + nw > lim) break;
        k = k - o + nw, len[bi]--;
    }
}

void depths(const std::vector<HNode> &N, int i, int d, uint8_t *len)
{
    if (N[i].sym >= 0) { len[N[i].sym] = (uint8_t)std::max(d, 1); return; }
    depths(N, N[i].l, d + 1, len), depths(N, N[i].r, d + 1, len);
}

// build_codes' lengths, huffman.rs:48-110
void code_lengths(const uint32_t *freq, int n, int maxl, uint8_t *len)
{
    std::vector<HNode> N;
    memset(len, 0, n);
    for (int i = 0; i < n; i++) if (freq[i]) N.push_back({freq[i], i, -1, -1});
    if (N.empty()) return;
    if (N.size() == 1) { len[N[0].sym] = 1; return; }
    Heap H{N, {}};
    for (size_t i = 0; i < N.size(); i++) H.h.push_back((int)i);
    N.reserve(2 * N.size());
    for (size_t k = H.h.size() / 2; k > 0; k--) H.sift_down_range(k - 1, H.h.size());   // BinaryHeap::rebuild
    while (H.h.size() > 1) {
        const int a = H.pop(), b = H.pop();
        N.push_back({N[a].f + N[b].f, -1, a, b});
        H.push((int)N.size() - 1);
    }
    depths(N, H.h[0], 0, len);
    limit_lengths(len, n, maxl);
}

// generate_canonical_codes (huffman.rs:212-244, u16 arithmetic wrapping as a release build does), bit-reversed as
// prepare_reversed_codes does (deflate.rs:1573-1590): code | length << 16
void canonical(const uint8_t *len, int n, uint32_t *out)
{
    uint32_t bl[16] = {0};
    uint16_t next[16] = {0}, c = 0;
    for (int i = 0; i < n; i++) if (len[i]) bl[len[i]]++;
    for (int b = 1; b <= 15; b++) c = (uint16_t)((uint16_t)(c + (uint16_t)bl[b - 1]) << 1), next[b] = c;
    for (int i = 0; i < n; i++) {
        out[i] = 0;
        if (!len[i]) continue;
        const uint16_t v = next[len[i]]++;
        uint32_t r = 0;
        for (int k = 0; k < len[i]; k++) r |= ((v >> k) & 1u) << (len[i] - 1 - k);
        out[i] = r | (uint32_t)len[i] << 16;
    }
}

// LSB-first bits into words
struct Bits {
    std::vector<uint32_t> &w;
    uint64_t n = 0;
    void put(uint32_t v, uint32_t nb)
    {
        for (uint32_t k = 0; k < nb; k++, n++) {
            if (n / 32 >= w.size()) w.push_back(0);
            w[n / 32] |= ((v >> k) & 1u) << (n % 32);
        }
    }
};

// zlib_header, deflate.rs:1642-1658
uint32_t zlib_header(int level)
{
    uint32_t flg = (uint32_t)(level <= 2 ? 1 : level <= 6 ? 2 : 3) << 6;
    flg |= (31 - ((0x78u << 8 | flg) % 31)) % 31;
    return 0x78 | flg << 8;
}

// One stream's choice and its exact size (compress_packed_zlib, deflate.rs:1008-1047): the header bits (zlib header,
// block header and, for dynamic blocks, the code lengths; encode_dynamic_huffman_packed_with_capacity,
// deflate.rs:1364-1468) go to hdr, the code table to table
struct Plan { uint32_t kind, hdr_bits; uint64_t zbytes; };
Plan plan_stream(const LzRecord &r, uint64_t n, int level, std::vector<uint32_t> &hdr_words, uint32_t *table)
{
    const uint64_t stored_bytes = 2 + n + (n ? (n + 65534) / 65535 : 0) * 5 + 4;
    Bits B{hdr_words};
    B.put(zlib_header(level), 16);
    Plan p{0, 16, stored_bytes};
    if (r.high_entropy || (n && r.nmatch == 0 && n >= 8192)) return p;
    uint32_t lf[286], df[30];
    memcpy(lf, r.lit, sizeof lf), memcpy(df, r.dist, sizeof df);
    lf[256]++;
    uint8_t ll[286], dl[30];
    if (r.ntok <= 128) {   // encode_best_huffman_packed, deflate.rs:121-144: fixed
        for (int i = 0; i < 286; i++) ll[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
        for (int i = 0; i < 30; i++) dl[i] = 5;
        uint32_t fl[288], fd[32];
        uint8_t fll[288], fdl[32];
        memcpy(fll, ll, 286), fll[286] = fll[287] = 8;
        memset(fdl, 5, 32);
        canonical(fll, 288, fl), canonical(fdl, 32, fd);
        memcpy(table, fl, 286 * 4), memcpy(table + 286, fd, 30 * 4);
        B.put(1, 1), B.put(1, 2);
        p.kind = 1;
    } else {
        bool any = false;
        for (int i = 0; i < 30; i++) any |= df[i] != 0;
        if (!any) df[0] = 1;
        code_lengths(lf, 286, 15, ll), code_lengths(df, 30, 15, dl);
        canonical(ll, 286, table), canonical(dl, 30, table + 286);
        int ln = 1, dn = 1;   // last_nonzero, deflate.rs:1470-1476
        for (int i = 285; i >= 0; i--) if (ll[i]) { ln = i + 1; break; }
        for (int i = 29; i >= 0; i--) if (dl[i]) { dn = i + 1; break; }
        const int hlit = std::min(std::max(ln - 257, 0), 29), hdist = std::min(std::max(dn - 1, 0), 29);
        // rle_code_lengths, deflate.rs:1490-1550
        uint8_t seq[316], rs[400], rx[400], rn[400];
        uint32_t cf[19] = {0}, cc[19];
        int ns = 0, nr = 0;
        for (int i = 0; i < 257 + hlit; i++) seq[ns++] = ll[i];
        for (int i = 0; i < 1 + hdist; i++) seq[ns++] = dl[i];
        auto emit = [&](int s, int x, int nb) { rs[nr] = (uint8_t)s, rx[nr] = (uint8_t)x, rn[nr++] = (uint8_t)nb, cf[s]++; };
        for (int i = 0; i < ns;) {
            const int cur = seq[i];
            int run = 1;
            while (i + run < ns && seq[i + run] == cur) run++;
            int rem = run;
            if (cur == 0) {
                while (rem > 0) {
                    if (rem >= 11) { const int k = std::min(rem, 138); emit(18, k - 11, 7), rem -= k; }
                    else if (rem >= 3) { const int k = std::min(rem, 10); emit(17, k - 3, 3), rem -= k; }
                    else emit(0, 0, 0), rem--;
                }
            } else {
                emit(cur, 0, 0);
                rem = run - 1;
                while (rem >= 3) { const int k = std::min(rem, 6); emit(16, k - 3, 2), rem -= k; }
                while (rem > 0) emit(cur, 0, 0), rem--;
            }
            i += run;
        }
        uint8_t cl[19];
        code_lengths(cf, 19, 7, cl);
        canonical(cl, 19, cc);
        static const int kOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
        int hclen = 0;
        for (int i = 18; i >= 0; i--) if (cl[kOrder[i]]) { hclen = std::min(i, 15); break; }
        B.put(1, 1), B.put(2, 2), B.put(hlit, 5), B.put(hdist, 5), B.put(hclen, 4);
        for (int i = 0; i < hclen + 4; i++) B.put(cl[kOrder[i]], 3);
        for (int i = 0; i < nr; i++) {
            B.put(cc[rs[i]] & 0xFFFF, cc[rs[i]] >> 16);
            if (rn[i]) B.put(rx[i], rn[i]);
        }
        p.kind = 2;
    }
    uint64_t bits = B.n - 16 + ll[256];
    for (int i = 0; i < 256; i++) bits += (uint64_t)r.lit[i] * ll[i];
    for (int a = 0; a < 29; a++) bits += (uint64_t)r.lit[257 + a] * (ll[257 + a] + kLExtra[a]);
    for (int b = 0; b < 30; b++) bits += (uint64_t)r.dist[b] * (dl[b] + kDExtra[b]);
    const uint64_t deflated = (bits + 7) / 8;
    // should_use_stored (deflate.rs:1091-1097) counts n / 65535 + 1 block headers, one more than deflate_stored
    // writes when n is a multiple of 65 535; empty_zlib has no such check
    if (n && deflated + 6 >= 2 + n + (n / 65535 + 1) * 5 + 4) {
        hdr_words.resize(1), hdr_words[0] &= 0xFFFF;
        return Plan{0, 16, stored_bytes};
    }
    p.hdr_bits = (uint32_t)B.n;
    p.zbytes = 2 + deflated + 4;
    return p;
}

}  // namespace

int deflate_zlib(pixo_b200_ctx *ctx, const uint8_t *d_streams, size_t stride, const size_t *lens, uint32_t n, int level,
                 uint8_t *d_out, size_t out_cap_each, size_t *out_lens, int32_t *status)
{
    for (uint32_t i = 0; i < n; i++)
        if (lens[i] >= kMaxStream)
            return set_error(ctx, PIXO_B200_ERR_UNSUPPORTED,
                             "stream %u is %zu bytes: streams of 2^31 bytes or more are beyond pixo's i32 positions",
                             i, lens[i]);
    // passes: a stream is charged its tokens (4 B per input byte) and its coded area
    std::vector<uint64_t> charge(n);
    std::vector<const uint64_t *> ptrs(n);
    for (uint32_t i = 0; i < n; i++) charge[i] = 5 * (uint64_t)lens[i] + 64, ptrs[i] = &charge[i];
    for (uint32_t p0 = 0; p0 < n;) {
        const uint32_t p1 = pass_end(ptrs.data(), p0, n, [](uint64_t c) { return c; });
        const uint32_t m = p1 - p0;
        std::vector<LzStream> hs(m);
        std::vector<uint32_t> order(m);
        uint64_t ntok = 0;
        for (uint32_t i = 0; i < m; i++) hs[i] = {d_streams + (size_t)(p0 + i) * stride, lens[p0 + i], ntok}, ntok += lens[p0 + i];
        for (uint32_t i = 0; i < m; i++) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return hs[a].len > hs[b].len; });
        const uint32_t warps = std::min<uint32_t>(m, (uint32_t)ctx->sm_count * kLzWarpsPerBlock * kLzBlocksPerSm);
        const uint32_t blocks = (warps + kLzWarpsPerBlock - 1) / kLzWarpsPerBlock;
        LzStream *d_s;
        uint32_t *d_order, *d_ticket, *d_tok;
        LzRecord *d_rec;
        int32_t *d_state;
        PIXO_TRY(bind(ctx, ctx->d_lz, [&](Layout &L) {
            d_s = L.take<LzStream>(m), d_order = L.take<uint32_t>(m), d_ticket = L.take<uint32_t>(1);
            d_rec = L.take<LzRecord>(m), d_tok = L.take<uint32_t>(std::max<uint64_t>(ntok, 1));
            d_state = L.take<int32_t>((size_t)blocks * kLzWarpsPerBlock * kStateWords);
        }));
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_s, hs.data(), m * sizeof(LzStream), cudaMemcpyHostToDevice, ctx->stream));
        PIXO_CUDA(ctx, cudaMemcpyAsync(d_order, order.data(), m * 4, cudaMemcpyHostToDevice, ctx->stream));
        PIXO_CUDA(ctx, cudaMemsetAsync(d_ticket, 0, 4, ctx->stream));
        PIXO_TRY(launch(ctx, k_lz77, blocks, kLzWarpsPerBlock * 32, 0, d_s, d_order, m, level, d_tok, d_rec, d_state, d_ticket));
        std::vector<LzRecord> rec(m);
        PIXO_CUDA(ctx, cudaMemcpyAsync(rec.data(), d_rec, m * sizeof(LzRecord), cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

        std::vector<EmitStream> es;
        std::vector<uint32_t> hdr, tables;
        uint64_t area_words = 0;
        for (uint32_t i = 0; i < m; i++) {
            const uint32_t f = p0 + i;
            std::vector<uint32_t> h;
            uint32_t table[316];
            const Plan P = plan_stream(rec[i], lens[f], level, h, table);
            out_lens[f] = P.zbytes;
            if (P.zbytes > out_cap_each) {
                status[f] = PIXO_B200_ERR_OUTPUT_TOO_SMALL;
                continue;
            }
            status[f] = 0;
            EmitStream E{};
            E.src = hs[i].src, E.tok = d_tok + hs[i].tok, E.len = lens[f], E.ntok = rec[i].ntok;
            E.zbytes = P.zbytes, E.kind = P.kind, E.hdr_bits = P.hdr_bits, E.hdr_word = hdr.size();
            E.adler = rec[i].adler, E.dst = d_out + (size_t)f * out_cap_each;
            hdr.insert(hdr.end(), h.begin(), h.end());
            if (P.kind) {
                E.table = (uint32_t)(tables.size() / 316), E.area = area_words;
                tables.insert(tables.end(), table, table + 316);
                area_words += (P.zbytes + 3) / 4 + 1;
            }
            es.push_back(E);
        }
        if (!es.empty()) {
            EmitStream *d_es;
            uint32_t *d_hdr, *d_tab, *d_area;
            PIXO_TRY(bind(ctx, ctx->d_zemit, [&](Layout &L) {
                d_es = L.take<EmitStream>(es.size()), d_hdr = L.take<uint32_t>(hdr.size());
                d_tab = L.take<uint32_t>(std::max<size_t>(tables.size(), 1)), d_area = L.take<uint32_t>(std::max<uint64_t>(area_words, 1));
            }));
            PIXO_CUDA(ctx, cudaMemcpyAsync(d_es, es.data(), es.size() * sizeof(EmitStream), cudaMemcpyHostToDevice, ctx->stream));
            PIXO_CUDA(ctx, cudaMemcpyAsync(d_hdr, hdr.data(), hdr.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
            if (!tables.empty())
                PIXO_CUDA(ctx, cudaMemcpyAsync(d_tab, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
            PIXO_CUDA(ctx, cudaMemsetAsync(d_area, 0, std::max<uint64_t>(area_words, 1) * 4, ctx->stream));
            const uint32_t eb = (uint32_t)std::min<size_t>((es.size() + kEmitWarpsPerBlock - 1) / kEmitWarpsPerBlock,
                                                           (size_t)ctx->sm_count * 8);
            PIXO_TRY(launch(ctx, k_deflate_emit, eb, kEmitWarpsPerBlock * 32, 0, d_es, (uint32_t)es.size(), d_hdr, d_tab, d_area));
            // the next pass rebinds the scratch this one's emit reads
            PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
        p0 = p1;
    }
    return 0;
}

}  // namespace pixo
