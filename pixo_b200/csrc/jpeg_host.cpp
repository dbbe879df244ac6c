// jpeg_host.cpp — host half of the JPEG path (see jpeg_host.hpp).
//
// The entropy stage is inherently a serial bit stream (DC prediction chain + variable-length
// codes), but nothing in it depends on *earlier output bits* except byte alignment for 0xFF
// stuffing and restart padding.  So the frame is cut into MCU ranges that worker threads code
// independently into raw (unstuffed, unpadded) bit strings — the DC predecessor of a range is
// simply the previous block's DC in the coefficient array — and one cheap sequential pass over
// the compressed bits splices the strings, applies 0xFF00 stuffing, restart padding and RSTn
// markers.  Output is byte-identical to the reference's single BitWriterMsb
// (src/bits.rs:195-290) driven by encode_scan (src/jpeg/mod.rs:1408-1563).
#include "jpeg_host.hpp"

#include <string.h>

#include <algorithm>
#include <atomic>
#include <queue>
#include <thread>

#include "../../include/pixo_b200.h"

namespace pixo {

namespace {

const uint8_t kStdLum[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                             14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                             18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                             49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kStdChr[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                             24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                             99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                             99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kZig[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                          12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                          35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                          58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Annex-K tables as pixo ships them, src/jpeg/huffman.rs:17-62
const uint8_t kDcLumBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kDcChrBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kAcLumBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125};
const uint8_t kAcChrBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119};
const uint8_t kAcLumVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61,
    0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52,
    0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25,
    0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
    0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
    0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3,
    0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8,
    0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kAcChrVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61,
    0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33,
    0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18,
    0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63,
    0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
    0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
    0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7,
    0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

inline uint32_t clamp255(uint32_t v) { return v < 1 ? 1 : (v > 255 ? 255 : v); }

// canonical code assignment from (bits, vals): src/jpeg/huffman.rs:213-286
bool assign_codes(HuffTables &t, int k, bool strict)
{
    const int table_len = k < 2 ? 12 : 256;
    memset(t.code[k], 0, sizeof t.code[k]);
    memset(t.len[k], 0, sizeof t.len[k]);
    uint16_t code = 0;
    int vi = 0;
    for (int l = 0; l < 16; ++l) {
        for (int c = 0; c < t.bits[k][l]; ++c) {
            if (vi < t.nvals[k]) {
                const int sym = t.vals[k][vi++];
                if (sym < table_len) {
                    t.code[k][sym] = code;
                    t.len[k][sym] = (uint8_t)(l + 1);
                } else if (strict) {
                    return false;
                }
            } else if (strict) {
                return false;
            }
            ++code;
        }
        code = (uint16_t)(code << 1);
    }
    return true;
}

void set_spec(HuffTables &t, int k, const uint8_t bits[16], const uint8_t *vals, int n)
{
    memcpy(t.bits[k], bits, 16);
    memset(t.vals[k], 0, 256);
    memcpy(t.vals[k], vals, (size_t)n);
    t.nvals[k] = n;
}

// build_code_lengths + build_bits_vals, src/jpeg/huffman.rs:288-391.
// Min-heap on (frequency, node index) — same order as BinaryHeap<Reverse<(u64, usize)>>;
// leaf length = depth + 1 (the reference's convention), fail when > 16.
bool spec_from_counts(const uint64_t *counts, int n, uint8_t bits[16], uint8_t *vals, int *nvals)
{
    struct Node { int left, right, sym; };
    std::vector<Node> nodes;
    typedef std::pair<uint64_t, int> Key;
    std::priority_queue<Key, std::vector<Key>, std::greater<Key>> heap;
    for (int s = 0; s < n; ++s) {
        if (!counts[s]) continue;
        heap.push(Key(counts[s], (int)nodes.size()));
        nodes.push_back(Node{-1, -1, s});
    }
    if (heap.empty()) return false;
    uint8_t lengths[256];
    memset(lengths, 0, sizeof lengths);
    if (heap.size() == 1) {
        lengths[nodes[heap.top().second].sym] = 1;
    } else {
        while (heap.size() > 1) {
            const Key a = heap.top(); heap.pop();
            const Key b = heap.top(); heap.pop();
            heap.push(Key(a.first + b.first, (int)nodes.size()));
            nodes.push_back(Node{a.second, b.second, -1});
        }
        std::vector<std::pair<int, int>> stack;
        stack.push_back(std::make_pair(heap.top().second, 0));
        while (!stack.empty()) {
            const std::pair<int, int> cur = stack.back();
            stack.pop_back();
            const Node &nd = nodes[cur.first];
            if (nd.sym >= 0) {
                if (cur.second + 1 > 16) return false;
                lengths[nd.sym] = (uint8_t)(cur.second + 1);
            } else {
                stack.push_back(std::make_pair(nd.left, cur.second + 1));
                stack.push_back(std::make_pair(nd.right, cur.second + 1));
            }
        }
    }
    memset(bits, 0, 16);
    int k = 0;
    for (int l = 1; l <= 16; ++l)
        for (int s = 0; s < n; ++s)
            if (lengths[s] == l) { bits[l - 1]++; vals[k++] = (uint8_t)s; }
    *nvals = k;
    return true;
}

inline int category(int v)
{
    const unsigned a = (unsigned)(v < 0 ? -v : v);
    return a ? 32 - __builtin_clz(a) : 0;
}

// ---- raw bit strings -------------------------------------------------------------------
struct RawBits {
    std::vector<uint8_t> buf;
    size_t pos = 0;       // bytes written
    uint64_t acc = 0;
    int nbits = 0;        // bits pending in acc (< 32 between puts)
    std::vector<uint64_t> cuts;  // bit positions of restart boundaries inside this string

    void reserve_more(size_t need)
    {
        if (pos + need > buf.size()) buf.resize(std::max(buf.size() * 2, pos + need + 4096));
    }
    inline void put(uint32_t v, int n)  // n <= 32
    {
        acc = (acc << n) | v;
        nbits += n;
        if (nbits >= 32) {
            const uint32_t w = (uint32_t)(acc >> (nbits - 32));
            const uint32_t be = __builtin_bswap32(w);
            memcpy(&buf[pos], &be, 4);
            pos += 4;
            nbits -= 32;
        }
    }
    uint64_t bit_length() const { return (uint64_t)pos * 8 + (uint64_t)nbits; }
    void finish()
    {
        reserve_more(16);
        // left-align the remaining bits into whole bytes (zero padded; length is tracked)
        int n = nbits;
        while (n > 0) {
            const int take = n >= 8 ? 8 : n;
            const uint8_t b = (uint8_t)(((acc >> (n - take)) & ((1u << take) - 1)) << (8 - take));
            buf[pos++] = b;
            n -= take;
        }
        // pos now counts the partial byte too; keep the true bit length separately
    }
};

struct CodeLut {
    // per table: code and length; AC entries also pre-shifted for fused code+amplitude puts
    const HuffTables *t;
};

// encode_block, src/jpeg/huffman.rs:423-481 (symbolisation + code lookup), raw bits out.
template <bool ZIGZAG_IN>
inline int encode_block_raw(RawBits &w, const int16_t *blk, int prev_dc, const uint16_t *dccode,
                            const uint8_t *dclen, const uint16_t *accode, const uint8_t *aclen)
{
    const int dc = blk[0];
    const int diff = (int16_t)(dc - prev_dc);
    const int dcat = category(diff);
    {
        const uint32_t amp = (uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << dcat) - 1u);
        w.put(((uint32_t)dccode[dcat] << dcat) | amp, dclen[dcat] + dcat);
    }
    int run = 0;
    for (int i = 1; i < 64; ++i) {
        const int c = ZIGZAG_IN ? blk[i] : blk[kZig[i]];
        if (c == 0) { ++run; continue; }
        while (run >= 16) { w.put(accode[0xF0], aclen[0xF0]); run -= 16; }
        const int cat = category(c);
        const int rs = (run << 4) | cat;
        const uint32_t amp = (uint32_t)(c < 0 ? c - 1 : c) & ((1u << cat) - 1u);
        w.put(((uint32_t)accode[rs] << cat) | amp, aclen[rs] + cat);
        run = 0;
    }
    if (run > 0) w.put(accode[0], aclen[0]);
    return dc;
}

struct ScanJob {
    const int16_t *y, *cb, *cr;
    const FrameGeometry *g;
    const HuffTables *t;
    uint32_t restart;
    bool zigzag_in;
    size_t m0, m1;
    int seed[3] = {0, 0, 0};   // predictors before MCU 0 (a band of a tiled frame)
    RawBits bits;
    uint64_t nbits_total = 0;
};

template <bool ZZ>
void run_job(ScanJob &j)
{
    const FrameGeometry &g = *j.g;
    const HuffTables &t = *j.t;
    const uint32_t ypm = g.y_per_mcu;
    RawBits &w = j.bits;
    w.buf.resize((j.m1 - j.m0) * (ypm + 2) * 24 + 4096);
    int py = 0, pcb = 0, pcr = 0;
    const bool fresh = j.m0 == 0 || (j.restart && j.m0 % j.restart == 0);
    if (j.m0 == 0 && !j.restart) { py = j.seed[0]; pcb = j.seed[1]; pcr = j.seed[2]; }
    if (!fresh) {
        py = j.y[(j.m0 * ypm - 1) * 64];
        if (g.has_chroma) { pcb = j.cb[(j.m0 - 1) * 64]; pcr = j.cr[(j.m0 - 1) * 64]; }
    }
    for (size_t m = j.m0; m < j.m1; ++m) {
        if (j.restart && m != j.m0 && m % j.restart == 0) {
            w.cuts.push_back(w.bit_length());
            py = pcb = pcr = 0;
        }
        w.reserve_more((size_t)(ypm + 2) * 272);
        for (uint32_t k = 0; k < ypm; ++k)
            py = encode_block_raw<ZZ>(w, j.y + (m * ypm + k) * 64, py, t.code[0], t.len[0],
                                      t.code[2], t.len[2]);
        if (g.has_chroma) {
            pcb = encode_block_raw<ZZ>(w, j.cb + m * 64, pcb, t.code[1], t.len[1], t.code[3], t.len[3]);
            pcr = encode_block_raw<ZZ>(w, j.cr + m * 64, pcr, t.code[1], t.len[1], t.code[3], t.len[3]);
        }
    }
    j.nbits_total = w.bit_length();
    w.finish();
}

void job_trampoline(int i, void *arg)
{
    ScanJob &j = (*reinterpret_cast<std::vector<ScanJob> *>(arg))[(size_t)i];
    if (j.zigzag_in) run_job<true>(j); else run_job<false>(j);
}

// Sequential splice: BitWriterMsb semantics (src/bits.rs:216-272) over raw bit strings.
struct StuffWriter {
    uint8_t *out;
    size_t len = 0, cap;
    uint64_t acc = 0;
    int nbits = 0;
    bool overflow = false;

    inline void push(uint8_t b)
    {
        if (len < cap) out[len++] = b; else overflow = true;
    }
    inline void drain_bytes()
    {
        while (nbits >= 8) {
            const uint8_t b = (uint8_t)(acc >> (nbits - 8));
            push(b);
            if (b == 0xFF) push(0x00);
            nbits -= 8;
        }
    }
    inline void put(uint32_t v, int n)  // n <= 32; at most 31 bits pending between calls
    {
        acc = (acc << n) | v;
        nbits += n;
        if (nbits >= 32) {
            const uint32_t w = (uint32_t)(acc >> (nbits - 32));
            const uint32_t x = ~w;  // a 0xFF byte in w is a zero byte in x
            if ((((x - 0x01010101u) & ~x) & 0x80808080u) == 0 && len + 4 <= cap) {
                const uint32_t be = __builtin_bswap32(w);
                memcpy(out + len, &be, 4);
                len += 4;
            } else {
                for (int s = 24; s >= 0; s -= 8) {
                    const uint8_t b = (uint8_t)(w >> s);
                    push(b);
                    if (b == 0xFF) push(0x00);
                }
            }
            nbits -= 32;
        }
    }
    // append bits [b0, b1) of a big-endian raw string
    void append(const uint8_t *p, size_t avail, uint64_t b0, uint64_t b1)
    {
        uint64_t pos = b0;
        // fast path: destination byte aligned and source byte aligned -> scan for 0xFF
        while (pos < b1) {
            if ((nbits & 7) == 0 && (pos & 7) == 0 && b1 - pos >= 8) {
                drain_bytes();
                const size_t nbytes = (size_t)((b1 - pos) >> 3);
                const uint8_t *s = p + (pos >> 3);
                size_t i = 0;
                while (i < nbytes) {
                    const uint8_t *ff = (const uint8_t *)memchr(s + i, 0xFF, nbytes - i);
                    const size_t run = ff ? (size_t)(ff - (s + i)) : nbytes - i;
                    if (len + run + 2 > cap) { overflow = true; return; }
                    memcpy(out + len, s + i, run);
                    len += run;
                    i += run;
                    if (ff) { out[len++] = 0xFF; out[len++] = 0x00; ++i; }
                }
                pos += (uint64_t)nbytes * 8;
                continue;
            }
            const int take = (int)std::min<uint64_t>(32, b1 - pos);
            const size_t byte = (size_t)(pos >> 3);
            uint64_t window = 0;
            if (byte + 8 <= avail) {
                memcpy(&window, p + byte, 8);
                window = __builtin_bswap64(window);
            } else {
                for (int k = 0; k < 8; ++k) window = (window << 8) | (byte + k < avail ? p[byte + k] : 0);
            }
            const int sh = (int)(pos & 7);
            const uint32_t v = (uint32_t)((window << sh) >> (64 - take));
            put(v, take);
            pos += (uint64_t)take;
        }
    }
    void pad_flush()  // BitWriterMsb::flush: pad with 1s, stuff if it became 0xFF
    {
        drain_bytes();
        if (nbits > 0) {
            const int pad = 8 - nbits;
            put((1u << pad) - 1u, pad);
            drain_bytes();
        }
    }
};

}  // namespace

bool coefficients_in_range(const int16_t *blocks, size_t nblocks, uint32_t restart_interval, uint32_t per_mcu,
                           int seed)
{
    int prev = seed;
    for (size_t b = 0; b < nblocks; ++b) {
        const int16_t *blk = blocks + b * 64;
        if (restart_interval && b % per_mcu == 0 && (b / per_mcu) % restart_interval == 0) prev = 0;
        const int diff = (int16_t)(blk[0] - prev);
        if (diff > 2047 || diff < -2047) return false;
        prev = blk[0];
        for (int i = 1; i < 64; ++i)
            if (blk[i] > 1023 || blk[i] < -1023) return false;
    }
    return true;
}

FrameGeometry make_geometry(uint32_t w, uint32_t h, uint32_t color_type, uint32_t subsampling)
{
    FrameGeometry g;
    g.width = w; g.height = h; g.color_type = color_type; g.subsampling = subsampling;
    g.has_chroma = color_type != PIXO_B200_GRAY;
    if (color_type == PIXO_B200_GRAY || subsampling == PIXO_B200_S444) {
        g.mcus_x = (w + 7) / 8; g.mcus_y = (h + 7) / 8; g.y_per_mcu = 1;
    } else {
        g.mcus_x = (w + 15) / 16; g.mcus_y = (h + 15) / 16; g.y_per_mcu = 4;
    }
    g.ny = g.total_mcus() * g.y_per_mcu;
    g.nc = g.has_chroma ? g.total_mcus() : 0;
    return g;
}

void quant_tables(int quality, uint8_t lum_zz[64], uint8_t chr_zz[64], float lum[64], float chr[64])
{
    quality = quality < 1 ? 1 : (quality > 100 ? 100 : quality);
    const uint32_t scale = quality < 50 ? 5000u / (uint32_t)quality : 200u - 2u * (uint32_t)quality;
    for (int i = 0; i < 64; ++i) {
        const uint32_t l = clamp255((kStdLum[i] * scale + 50) / 100);
        const uint32_t c = clamp255((kStdChr[i] * scale + 50) / 100);
        if (lum) lum[i] = (float)l;
        if (chr) chr[i] = (float)c;
    }
    for (int i = 0; i < 64; ++i) {
        if (lum_zz) lum_zz[i] = (uint8_t)clamp255((kStdLum[kZig[i]] * scale + 50) / 100);
        if (chr_zz) chr_zz[i] = (uint8_t)clamp255((kStdChr[kZig[i]] * scale + 50) / 100);
    }
}

void huff_standard(HuffTables &t)
{
    static const uint8_t dcvals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
    set_spec(t, 0, kDcLumBits, dcvals, 12);
    set_spec(t, 1, kDcChrBits, dcvals, 12);
    set_spec(t, 2, kAcLumBits, kAcLumVals, 162);
    set_spec(t, 3, kAcChrBits, kAcChrVals, 162);
    for (int k = 0; k < 4; ++k) assign_codes(t, k, false);
}

bool huff_from_histogram(const uint64_t hist[536], bool has_chroma, HuffTables &t)
{
    static const uint8_t dcvals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
    uint8_t bits[16], vals[256];
    int nv = 0;
    if (!spec_from_counts(hist, 12, bits, vals, &nv)) return false;
    set_spec(t, 0, bits, vals, nv);
    if (!spec_from_counts(hist + 24, 256, bits, vals, &nv)) return false;
    set_spec(t, 2, bits, vals, nv);
    if (has_chroma && spec_from_counts(hist + 12, 12, bits, vals, &nv)) set_spec(t, 1, bits, vals, nv);
    else set_spec(t, 1, kDcChrBits, dcvals, 12);
    if (has_chroma && spec_from_counts(hist + 280, 256, bits, vals, &nv)) set_spec(t, 3, bits, vals, nv);
    else set_spec(t, 3, kAcChrBits, kAcChrVals, 162);
    for (int k = 0; k < 4; ++k)
        if (!assign_codes(t, k, true)) return false;
    return true;
}

void huff_from_dht(const uint8_t dht[1088], HuffTables &t)
{
    for (int k = 0; k < 4; ++k) {
        const uint8_t *b = dht + k * 272;
        int n = 0;
        for (int l = 0; l < 16; ++l) n += b[l];
        set_spec(t, k, b, b + 16, n);
        assign_codes(t, k, false);
    }
}

const uint8_t *dht_standard()
{
    static const struct Block {
        uint8_t dht[1088];
        Block()
        {
            HuffTables t;
            huff_standard(t);
            for (int k = 0; k < 4; ++k) {
                memcpy(dht + k * 272, t.bits[k], 16);
                memcpy(dht + k * 272 + 16, t.vals[k], 256);
            }
        }
    } block;
    return block.dht;
}

// SOI..DRI with the frame header `sof` (0xFFC0 baseline, 0xFFC2 progressive: write_sof_marker,
// src/jpeg/mod.rs:498-560)
static size_t write_frame_headers(uint8_t *out, const FrameGeometry &g, const uint8_t lum_zz[64],
                                  const uint8_t chr_zz[64], const HuffTables &t, uint32_t restart_interval,
                                  unsigned sof)
{
    uint8_t *p = out;
    auto u8 = [&](unsigned v) { *p++ = (uint8_t)v; };
    auto u16 = [&](unsigned v) { *p++ = (uint8_t)(v >> 8); *p++ = (uint8_t)v; };
    u16(0xFFD8);
    u16(0xFFE0); u16(16);
    memcpy(p, "JFIF\0", 5); p += 5;
    u8(1); u8(1); u8(0); u16(1); u16(1); u8(0); u8(0);
    u16(0xFFDB); u16(67); u8(0); memcpy(p, lum_zz, 64); p += 64;
    u16(0xFFDB); u16(67); u8(1); memcpy(p, chr_zz, 64); p += 64;
    const int ncomp = g.has_chroma ? 3 : 1;
    u16(sof); u16(8 + 3 * ncomp); u8(8); u16(g.height & 0xFFFF); u16(g.width & 0xFFFF); u8(ncomp);
    if (ncomp == 1) { u8(1); u8(0x11); u8(0); }
    else {
        u8(1); u8(g.subsampling == PIXO_B200_S420 ? 0x22 : 0x11); u8(0);
        u8(2); u8(0x11); u8(1);
        u8(3); u8(0x11); u8(1);
    }
    static const uint8_t ids[4] = {0x00, 0x01, 0x10, 0x11};
    for (int k = 0; k < 4; ++k) {
        u16(0xFFC4); u16(2 + 1 + 16 + t.nvals[k]); u8(ids[k]);
        memcpy(p, t.bits[k], 16); p += 16;
        memcpy(p, t.vals[k], (size_t)t.nvals[k]); p += t.nvals[k];
    }
    if (restart_interval) { u16(0xFFDD); u16(4); u16(restart_interval & 0xFFFF); }
    return (size_t)(p - out);
}

size_t write_headers(uint8_t *out, const FrameGeometry &g, const uint8_t lum_zz[64],
                     const uint8_t chr_zz[64], const HuffTables &t, uint32_t restart_interval)
{
    uint8_t *p = out + write_frame_headers(out, g, lum_zz, chr_zz, t, restart_interval, 0xFFC0);
    auto u8 = [&](unsigned v) { *p++ = (uint8_t)v; };
    auto u16 = [&](unsigned v) { *p++ = (uint8_t)(v >> 8); *p++ = (uint8_t)v; };
    const int ncomp = g.has_chroma ? 3 : 1;
    u16(0xFFDA); u16(6 + 2 * ncomp); u8(ncomp);
    if (ncomp == 1) { u8(1); u8(0x00); }
    else { u8(1); u8(0x00); u8(2); u8(0x11); u8(3); u8(0x11); }
    u8(0); u8(63); u8(0);
    return (size_t)(p - out);
}

size_t write_headers_progressive(uint8_t *out, const FrameGeometry &g, const uint8_t lum_zz[64],
                                 const uint8_t chr_zz[64], const HuffTables &t, uint32_t restart_interval)
{
    return write_frame_headers(out, g, lum_zz, chr_zz, t, restart_interval, 0xFFC2);
}

size_t write_sos_progressive(uint8_t *out, int scan)
{
    static const uint8_t comp[7] = {0, 1, 2, 0, 0, 1, 2}, ss[7] = {0, 0, 0, 1, 11, 1, 1}, se[7] = {0, 0, 0, 10, 63, 63, 63};
    const uint8_t sos[10] = {0xFF, 0xDA, 0, 8, 1, (uint8_t)(comp[scan] + 1), (uint8_t)(comp[scan] ? 0x11 : 0x00),
                             ss[scan], se[scan], 0};
    memcpy(out, sos, sizeof sos);
    return sizeof sos;
}

void parallel_jobs(int n, int threads, void (*fn)(int, void *), void *arg)
{
    if (threads < 1) threads = 1;
    if (threads > n) threads = n;
    if (threads <= 1) {
        for (int i = 0; i < n; ++i) fn(i, arg);
        return;
    }
    std::atomic<int> next(0);
    auto worker = [&]() {
        for (;;) {
            const int i = next.fetch_add(1);
            if (i >= n) break;
            fn(i, arg);
        }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(worker);
    worker();
    for (auto &th : pool) th.join();
}

size_t entropy_encode_scan(const int16_t *y, const int16_t *cb, const int16_t *cr,
                           const FrameGeometry &g, const HuffTables &t,
                           uint32_t restart_interval, bool zigzag_in, uint8_t *out, size_t cap,
                           int threads)
{
    const size_t total = g.total_mcus();
    if (threads < 1) threads = 1;
    size_t njobs = (size_t)threads * 4;
    const size_t min_mcus = 256;  // do not shred tiny frames
    if (njobs > (total + min_mcus - 1) / min_mcus) njobs = (total + min_mcus - 1) / min_mcus;
    if (njobs < 1) njobs = 1;
    std::vector<ScanJob> jobs(njobs);
    for (size_t i = 0; i < njobs; ++i) {
        ScanJob &j = jobs[i];
        j.y = y; j.cb = cb; j.cr = cr; j.g = &g; j.t = &t;
        j.restart = restart_interval; j.zigzag_in = zigzag_in;
        j.m0 = total * i / njobs;
        j.m1 = total * (i + 1) / njobs;
    }
    parallel_jobs((int)njobs, threads, job_trampoline, &jobs);

    StuffWriter sw;
    sw.out = out; sw.cap = cap;
    unsigned rst = 0;
    auto marker = [&]() {  // handle_restart, src/jpeg/mod.rs:1423-1445
        sw.pad_flush();
        sw.push(0xFF);
        sw.push((uint8_t)(0xD0 + (rst & 7)));
        rst = (rst + 1) & 7;
    };
    for (size_t i = 0; i < njobs; ++i) {
        ScanJob &j = jobs[i];
        if (restart_interval && j.m0 != 0 && j.m0 % restart_interval == 0 && j.m0 < total) marker();
        uint64_t from = 0;
        for (uint64_t cut : j.bits.cuts) {
            sw.append(j.bits.buf.data(), j.bits.pos, from, cut);
            marker();
            from = cut;
        }
        sw.append(j.bits.buf.data(), j.bits.pos, from, j.nbits_total);
        if (sw.overflow) return (size_t)-1;
    }
    sw.pad_flush();
    if (sw.overflow) return (size_t)-1;
    return sw.len;
}

// One band of a tiled frame -> its raw (unstuffed, unpadded) bit string, left-aligned in bytes.
// Returns the bit count, or (uint64_t)-1 when `cap` is too small.
uint64_t band_encode_raw(const int16_t *y, const int16_t *cb, const int16_t *cr, const FrameGeometry &g,
                         const HuffTables &t, const int seed[3], uint8_t *out, size_t cap, uint32_t *tail7)
{
    ScanJob j;
    j.y = y; j.cb = cb; j.cr = cr; j.g = &g; j.t = &t;
    j.restart = 0; j.zigzag_in = false; j.m0 = 0; j.m1 = g.total_mcus();
    for (int k = 0; k < 3; ++k) j.seed[k] = seed ? seed[k] : 0;
    run_job<false>(j);
    const size_t nbytes = (size_t)((j.nbits_total + 7) >> 3);
    if (nbytes > cap) return (uint64_t)-1;
    memcpy(out, j.bits.buf.data(), nbytes);
    if (tail7) {   // the string's last 7 bits
        uint32_t v = 0;
        for (int b = 0; b < 7; ++b) {
            if ((uint64_t)b >= j.nbits_total) break;
            const uint64_t pos = j.nbits_total - 1 - (uint64_t)b;
            v |= (uint32_t)((out[pos >> 3] >> (7 - (pos & 7))) & 1u) << b;
        }
        *tail7 = v;
    }
    return j.nbits_total;
}

// tail_in (phase bits) ++ raw string -> stuffed bytes; the frame's last band pads with 1s.
size_t band_splice(const uint8_t *raw, uint64_t nbits, uint32_t phase, uint32_t tail_in, bool last,
                   uint8_t *out, size_t cap)
{
    StuffWriter sw;
    sw.out = out; sw.cap = cap;
    sw.nbits = (int)(phase & 7u);
    sw.acc = tail_in & ((1u << (phase & 7u)) - 1u);
    sw.append(raw, (size_t)((nbits + 7) >> 3), 0, nbits);
    if (last) sw.pad_flush(); else sw.drain_bytes();
    return sw.overflow ? (size_t)-1 : sw.len;
}

void host_histogram(const int16_t *y, const int16_t *cb, const int16_t *cr,
                    const FrameGeometry &g, uint32_t restart_interval, uint64_t hist[536], const int *seed)
{
    memset(hist, 0, 536 * sizeof(uint64_t));
    auto count = [&](const int16_t *blk, int prev, uint64_t *dc, uint64_t *ac) {
        const int d = blk[0];
        dc[category((int16_t)(d - prev))]++;
        int run = 0;
        for (int i = 1; i < 64; ++i) {
            const int c = blk[kZig[i]];
            if (!c) { ++run; continue; }
            if (run >= 16) { ac[0xF0] += (uint64_t)(run >> 4); run &= 15; }
            ac[(run << 4) | category(c)]++;
            run = 0;
        }
        if (run) ac[0]++;
        return d;
    };
    int py = 0, pcb = 0, pcr = 0;
    if (seed && !restart_interval) { py = seed[0]; pcb = seed[1]; pcr = seed[2]; }
    const size_t total = g.total_mcus();
    for (size_t m = 0; m < total; ++m) {
        if (restart_interval && m && m % restart_interval == 0) py = pcb = pcr = 0;
        for (uint32_t k = 0; k < g.y_per_mcu; ++k)
            py = count(y + (m * g.y_per_mcu + k) * 64, py, hist, hist + 24);
        if (g.has_chroma) {
            pcb = count(cb + m * 64, pcb, hist + 12, hist + 280);
            pcr = count(cr + m * 64, pcr, hist + 12, hist + 280);
        }
    }
}

}  // namespace pixo
