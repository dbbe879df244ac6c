// png_decode.cu — PNG decoding on the device, pixel-identical to pixo::decode::decode_png (src/decode/png.rs,
// inflate.rs, bit_reader.rs), errors included.  The host walks the chunks (png_decode_host.cpp); here, per pass:
//   k_png_crc       the CRC-32 of every IDAT chunk, in pieces over many CTAs, combined by GF(2) shifts
//   k_png_inflate   one warp per zlib stream: lane 0 decodes symbols, the warp writes the bytes, folds in the
//                   Adler-32 and reads the filter byte of every row; the per-file record holds the outcome
//   k_png_unfilter  a wavefront over 32-row groups undoes the five filters, into the caller's frame for 8-bit
//                   Gray / GrayAlpha / RGB / RGBA, in place otherwise
//   k_png_expand    sub-8-bit unpacking, 16 -> 8 bit and palette + tRNS expansion into the caller's frame (launched
//                   only for passes holding such files)
// The host waits once per pass and resolves each file's error in pixo's order.
#include <string.h>

#include "common.cuh"
#include "decode_host.hpp"
#include "png_decode_host.hpp"

namespace pixo {

namespace {

// What k_png_inflate finds; the order of the checks after inflate is pixo's (Adler-32, size, then the filters)
enum PdecCode : uint32_t {
    kOk = 0, kCrc, kEos, kReservedBlock, kLenNlen, kEmptyTable, kBadCode, kRepeatAtStart, kTooManyLengths,
    kBadLitLen, kBadDistCode, kDistTooFar, kAdler, kSize, kFilter, kFault
};

// One file of a pass as the kernels read it
struct PdecFile {
    uint64_t src, src_len;     // the zlib stream (IDAT payloads concatenated): offset into the pass's bytes, length
    uint64_t scratch, cap;     // the inflated bytes: offset into the scratch area, room there (PdecParsed::scratch)
    uint64_t expected, sb;     // calculate_expected_size; scanline bytes
    uint64_t out;              // byte offset of the frame in the caller's buffer
    uint32_t chunk0, nchunks;  // the file's IDAT chunks in the pass's chunk table
    uint32_t width, height, bpp, depth, ctype, channels;
    uint32_t pal;              // indexed: the file's 256-entry RGBA table in the pass's palette area
    uint32_t flags;            // kDirect, kNoPlte
};
constexpr uint32_t kDirect = 1, kNoPlte = 2;

struct PdecChunk {
    uint64_t src;        // payload: offset into the pass's bytes
    uint64_t len;
};

// What k_png_inflate leaves for the host
struct PdecRecord {
    uint32_t code, arg;             // PdecCode; the failing IDAT chunk, literal/length symbol or filter type
    uint32_t stored_adler, adler;
    uint64_t produced;              // bytes the stream produced
};

constexpr uint32_t kCrcPiece = 4096;   // bytes a k_png_crc thread runs the register over
constexpr int kInflateWarps = 4;       // warps per CTA of k_png_inflate
constexpr int kTok = 64, kLits = 1024; // token batch of k_png_inflate: tokens, literal bytes
constexpr uint32_t kRing = 32768;      // bytes past expected_size a file keeps, for back-references
constexpr int kUnfilterWarps = 4;
constexpr int kExpandThreads = 256;
// How long a wavefront wait may see the row above make no progress before it is a fault.  The longest legitimate
// stall is a group's first wait at launch: up to sm_count * 32 groups are in flight, and group k waits for the k
// groups ahead of it to pass 32 pixels each, about 63 steps per group.  At 1 us a step (a load of the row above
// and a shuffle) that is 4 224 * 63 us = 0.27 s on an H100; the limit is 10 s.
constexpr uint64_t kStallNs = 10ull * 1000 * 1000 * 1000;

__device__ __forceinline__ uint64_t globaltimer_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

constexpr uint32_t ADLER_MOD = 65521;

// ---- k_png_crc -------------------------------------------------------------------------------------------

// One thread per piece of kCrcPiece bytes of a chunk: the register over the piece from 0, shifted over the bytes
// after it in the chunk, XORed into the chunk's word.  The host starts that word at the register over "IDAT" shifted
// over the whole payload, inverted and XORed with the stored CRC, so it ends 0 exactly when the CRC matches.
__global__ void __launch_bounds__(256) k_png_crc(const PdecChunk *__restrict__ C, const uint64_t *__restrict__ piece_prefix,
                                                 uint32_t nchunks, uint64_t npieces, const uint8_t *__restrict__ bytes,
                                                 uint32_t *__restrict__ acc)
{
    __shared__ uint32_t tab[256];
    crc32_table(tab);
    __syncthreads();
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= npieces) return;
    const uint32_t c = item_of(piece_prefix, nchunks, g);
    const PdecChunk K = C[c];
    const uint64_t start = (g - __ldg(piece_prefix + c)) * kCrcPiece;
    const uint64_t n = min((uint64_t)kCrcPiece, K.len - start);
    const uint32_t reg = crc32_piece(tab, bytes + K.src + start, n);
    atomicXor(acc + c, crc32_shift(reg, K.len - start - n));
}

// ---- k_png_inflate ---------------------------------------------------------------------------------------

// HuffmanTable as from_lengths builds it (src/decode/inflate.rs:59-127): the 9-bit lookup in which a later symbol
// overwrites an earlier one (symbol | length << 12, 0: no code of at most 9 bits), and for decode_slow the canonical
// codes per length, unbounded as pixo keeps them in u32, with the symbols of each length in symbol order
struct Huff {
    uint16_t lookup[512];
    uint32_t first[16];
    uint16_t count[16], off[16];
    uint16_t sorted[288];
    uint32_t maxlen;
};

struct Token {
    uint32_t kind_len;   // kind << 24 | length
    uint32_t dist;       // match: distance; literal run: first byte in lits
    uint64_t src;        // stored block: first byte in the DEFLATE data
};
constexpr uint32_t kTokLit = 0, kTokMatch = 1, kTokStored = 2;

struct InflateSmem {
    Huff lit, dist;      // the code length code's table goes in `dist` while the lengths are read
    Token tok[kTok];
    uint8_t lits[kLits];
    uint8_t lens[320];
    uint32_t ntok, state;   // state: 0 more to come, 1 the stream ended, 2 an error ended it
};

__device__ const uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59,
                                            67, 83, 99, 115, 131, 163, 195, 227, 258};
__device__ const uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4,
                                            5, 5, 5, 5, 0};
__device__ const uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513,
                                             769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__device__ const uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10,
                                             11, 11, 12, 12, 13, 13};
__device__ const uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ void build_huff(Huff &t, const uint8_t *len, uint32_t n)
{
    uint32_t maxlen = 0, bl[16] = {};
    for (uint32_t s = 0; s < n; ++s) {
        maxlen = max(maxlen, (uint32_t)len[s]);
        if (len[s]) ++bl[len[s]];
    }
    t.maxlen = maxlen;
    if (!maxlen) return;
    uint32_t code = 0, next[16], o = 0;
    for (int b = 1; b <= 15; ++b) {
        code = (code + bl[b - 1]) << 1;
        next[b] = code;
        t.first[b] = code;
        t.count[b] = (uint16_t)bl[b];
        t.off[b] = (uint16_t)o;
        o += bl[b];
    }
    for (int i = 0; i < 512; ++i) t.lookup[i] = 0;
    uint32_t rank[16] = {};
    for (uint32_t s = 0; s < n; ++s) {
        const uint32_t L = len[s];
        if (!L) continue;
        t.sorted[t.off[L] + rank[L]++] = (uint16_t)s;
        const uint32_t c = next[L]++;
        if (L > 9) continue;
        const uint32_t rev = __brev(c) >> (32 - L);
        for (uint32_t i = 0; i < (1u << (9 - L)); ++i) t.lookup[rev | (i << L)] = (uint16_t)(s | (L << 12));
    }
}

// BitReader (src/decode/bit_reader.rs:10-135) over the DEFLATE data data[2 .. len-4]: whole bytes are loaded into
// a 64-bit buffer, so the bits left are cnt plus those of the bytes not loaded
struct Bits {
    const uint8_t *d;
    uint64_t n, next;
    uint64_t buf;
    uint32_t cnt;
    __device__ void refill()
    {
        while (cnt <= 56 && next < n) {
            buf |= (uint64_t)__ldg(d + next++) << cnt;
            cnt += 8;
        }
    }
    __device__ bool read(uint32_t k, uint32_t &v)
    {
        if (cnt < k) refill();
        if (cnt < k) return false;
        v = (uint32_t)(buf & ((1ull << k) - 1));
        buf >>= k;
        cnt -= k;
        return true;
    }
};

// HuffmanTable::decode and decode_slow (inflate.rs:130-186)
__device__ uint32_t huff_decode(const Huff &t, Bits &r, uint32_t &sym)
{
    if (!t.maxlen) return kEmptyTable;
    if (r.cnt < 9) r.refill();
    const uint32_t avail = min(r.cnt, 9u);
    if (avail > 0) {
        const uint32_t e = t.lookup[(uint32_t)(r.buf & ((1u << avail) - 1))], L = e >> 12;
        if (L > 0 && L <= avail) {
            r.buf >>= L;
            r.cnt -= L;
            sym = e & 0xFFF;
            return kOk;
        }
    }
    uint32_t code = 0;
    for (uint32_t L = 1; L <= t.maxlen; ++L) {
        uint32_t bit;
        if (!r.read(1, bit)) return kEos;
        code = (code << 1) | bit;
        if (code - t.first[L] < t.count[L]) {
            sym = t.sorted[t.off[L] + code - t.first[L]];
            return kOk;
        }
    }
    return kBadCode;
}

// inflate_dynamic's header (inflate.rs:386-455): the tables of the block into S.lit and S.dist
__device__ uint32_t read_dynamic(InflateSmem &S, Bits &r)
{
    uint32_t hlit, hdist, hclen, v;
    if (!r.read(5, hlit) || !r.read(5, hdist) || !r.read(4, hclen)) return kEos;
    hlit += 257;
    hdist += 1;
    hclen += 4;
    uint8_t cl[19] = {};
    for (uint32_t i = 0; i < hclen; ++i) {
        if (!r.read(3, v)) return kEos;
        cl[c_cl_order[i]] = (uint8_t)v;
    }
    build_huff(S.dist, cl, 19);
    const uint32_t total = hlit + hdist;
    for (uint32_t i = 0; i < total; ++i) S.lens[i] = 0;
    for (uint32_t i = 0; i < total;) {
        uint32_t sym;
        const uint32_t e = huff_decode(S.dist, r, sym);
        if (e) return e;
        if (sym < 16) {
            S.lens[i++] = (uint8_t)sym;
            continue;
        }
        uint32_t rep, val = 0;
        if (sym == 16) {
            if (i == 0) return kRepeatAtStart;
            if (!r.read(2, rep)) return kEos;
            rep += 3;
            val = S.lens[i - 1];
        } else if (sym == 17) {
            if (!r.read(3, rep)) return kEos;
            rep += 3;
        } else {
            if (!r.read(7, rep)) return kEos;
            rep += 11;
        }
        for (uint32_t k = 0; k < rep; ++k) {
            if (i >= total) return kTooManyLengths;
            S.lens[i++] = (uint8_t)val;
        }
    }
    build_huff(S.lit, S.lens, hlit);
    build_huff(S.dist, S.lens + hlit, hdist);
    return kOk;
}

// Lane 0's share: decode symbols into the token batch until it is full or the stream ends
struct Decoder {
    Bits r;
    uint64_t produced;
    uint32_t in_block, final_block, tables;   // tables: 1 the fixed ones are built
    uint32_t err, arg;
};

__device__ void decode_batch(InflateSmem &S, Decoder &D)
{
    uint32_t nt = 0, nl = 0;
    int open_lit = -1;   // the literal run the next literal extends
    for (;;) {
        if (nt >= kTok - 1 || nl >= kLits) break;
        if (!D.in_block) {
            if (D.final_block) { S.state = 1; break; }
            uint32_t bfinal, btype;
            if (!D.r.read(1, bfinal) || !D.r.read(2, btype)) { D.err = kEos; break; }
            D.final_block = bfinal;
            if (btype == 0) {   // inflate_stored (inflate.rs:355-376)
                const uint32_t drop = D.r.cnt & 7;
                D.r.buf >>= drop;
                D.r.cnt -= drop;
                uint32_t len, nlen;
                if (!D.r.read(16, len) || !D.r.read(16, nlen)) { D.err = kEos; break; }
                if (len != (~nlen & 0xFFFF)) { D.err = kLenNlen; break; }
                const uint64_t at = D.r.next - D.r.cnt / 8;   // the byte the buffer's bits start at
                if (at + len > D.r.n) { D.err = kEos; break; }
                D.r.next = at + len;
                D.r.buf = 0;
                D.r.cnt = 0;
                if (len) {
                    S.tok[nt++] = Token{kTokStored << 24 | len, 0, at};
                    open_lit = -1;
                    D.produced += len;
                }
                continue;
            }
            if (btype == 3) { D.err = kReservedBlock; break; }
            if (btype == 1) {
                if (D.tables != 1) {
                    for (int s = 0; s < 288; ++s) S.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
                    build_huff(S.lit, S.lens, 288);
                    for (int s = 0; s < 32; ++s) S.lens[s] = 5;
                    build_huff(S.dist, S.lens, 32);
                    D.tables = 1;
                }
            } else {
                D.tables = 0;
                const uint32_t e = read_dynamic(S, D.r);
                if (e) { D.err = e; break; }
            }
            D.in_block = 1;
        }
        uint32_t sym;
        uint32_t e = huff_decode(S.lit, D.r, sym);
        if (e) { D.err = e; break; }
        if (sym < 256) {
            if (open_lit < 0) {
                open_lit = nt;
                S.tok[nt++] = Token{kTokLit << 24, nl, 0};
            }
            S.lits[nl++] = (uint8_t)sym;
            S.tok[open_lit].kind_len++;
            D.produced++;
            continue;
        }
        if (sym == 256) {
            D.in_block = 0;
            continue;
        }
        if (sym > 285) { D.err = kBadLitLen; D.arg = sym; break; }
        uint32_t extra, dsym;
        if (!D.r.read(c_len_extra[sym - 257], extra)) { D.err = kEos; break; }
        const uint32_t len = c_len_base[sym - 257] + extra;
        e = huff_decode(S.dist, D.r, dsym);
        if (e) { D.err = e; break; }
        if (dsym >= 30) { D.err = kBadDistCode; break; }
        if (!D.r.read(c_dist_extra[dsym], extra)) { D.err = kEos; break; }
        const uint32_t dist = c_dist_base[dsym] + extra;
        if (dist > D.produced) { D.err = kDistTooFar; break; }
        S.tok[nt++] = Token{kTokMatch << 24 | len, dist, 0};
        open_lit = -1;
        D.produced += len;
    }
    if (D.err) S.state = 2;
    S.ntok = nt;
}

// One warp per zlib stream, in `order` (longest first), handed out by a ticket.  Lane 0 decodes a batch of tokens;
// the warp writes them, 32 bytes a step (a match of distance d < 32 in steps of the largest multiple of d), folds
// each byte into its lane's Adler-32 sums and reads the filter byte of every row it writes.  Bytes before
// expected_size go to the file's scratch, later ones to the warp's ring, which keeps the last 32 KiB of them for
// back-references.  Every loop is bounded by the stream's bits: a symbol takes at least one.
__global__ void __launch_bounds__(kInflateWarps * 32) k_png_inflate(const PdecFile *__restrict__ F,
                                                                    const uint32_t *__restrict__ order, uint32_t n,
                                                                    const uint32_t *__restrict__ crc_acc,
                                                                    const uint8_t *__restrict__ bytes, uint8_t *scratch,
                                                                    uint8_t *rings, uint32_t *ticket,
                                                                    PdecRecord *__restrict__ rec)
{
    __shared__ InflateSmem smem[kInflateWarps];
    const uint32_t lane = threadIdx.x & 31, w = threadIdx.x / 32;
    InflateSmem &S = smem[w];
    uint8_t *ring = rings + ((uint64_t)blockIdx.x * kInflateWarps + w) * kRing;
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= n) return;
        const uint32_t f = order[t];
        const PdecFile J = F[f];
        PdecRecord R{kOk, 0, 0, 0, 0};
        // the first IDAT chunk whose CRC failed (k_png_crc)
        for (uint32_t c0 = 0; c0 < J.nchunks && R.code == kOk; c0 += 32) {
            const bool bad = c0 + lane < J.nchunks && __ldg(crc_acc + J.chunk0 + c0 + lane) != 0;
            const uint32_t b = __ballot_sync(0xffffffffu, bad);
            if (b) R = PdecRecord{kCrc, c0 + __ffs(b) - 1, 0, 0, 0};
        }
        if (R.code != kOk) {
            if (lane == 0) rec[f] = R;
            continue;
        }
        const uint8_t *zs = bytes + J.src;
        uint8_t *out = scratch + J.scratch;
        Decoder D;
        if (lane == 0) {
            D.r = Bits{zs + 2, J.src_len - 6, 0, 0, 0};
            D.produced = 0;
            D.in_block = D.final_block = D.tables = D.err = D.arg = 0;
            S.state = 0;
        }
        uint64_t pos = 0, s1 = 0, s2 = 0, nrs = 0, row = 0;   // nrs: where the next row's filter byte is
        uint32_t pm = 0, bad_row_val = 0xFFFFFFFFu;
        bool fault = false;
        const uint64_t rowlen = J.sb + 1;
        for (;;) {
            if (lane == 0) decode_batch(S, D);
            __syncwarp();
            const uint32_t nt = S.ntok, state = S.state;
            for (uint32_t k = 0; k < nt; ++k) {
                const Token T = S.tok[k];
                const uint32_t kind = T.kind_len >> 24, L = T.kind_len & 0xFFFFFF;
                const uint32_t step = kind != kTokMatch || T.dist >= 32 ? 32 : T.dist * (32 / T.dist);
                for (uint32_t o = 0; o < L; o += step) {
                    const uint32_t cnt = min(step, L - o);
                    const uint64_t p = pos + o + lane;
                    uint32_t v = 0;
                    if (lane < cnt) {
                        if (kind == kTokLit) {
                            v = S.lits[T.dist + o + lane];
                        } else if (kind == kTokStored) {
                            v = __ldg(zs + 2 + T.src + o + lane);
                        } else {
                            const uint64_t q = pos + o + lane % T.dist - T.dist;
                            v = q < J.expected ? out[q] : ring[q & (kRing - 1)];
                        }
                    }
                    __syncwarp();
                    if (lane < cnt) {
                        if (p < J.expected) {
                            if (p < J.cap) out[p] = (uint8_t)v;
                            else fault = true;
                        } else {
                            ring[p & (kRing - 1)] = (uint8_t)v;
                        }
                        s1 += v;
                        s2 += (uint64_t)(pm + lane) * v;
                    }
                    // the filter byte of every row starting in this step
                    const uint64_t base = pos + o;
                    while (nrs < base + cnt && nrs < J.expected) {
                        const uint32_t fb = __shfl_sync(0xffffffffu, v, (uint32_t)(nrs - base));
                        if (fb > 4 && bad_row_val == 0xFFFFFFFFu) bad_row_val = fb;
                        nrs = bad_row_val == 0xFFFFFFFFu ? nrs + rowlen : J.expected;
                        ++row;
                    }
                    pm += cnt;
                    if (pm >= ADLER_MOD) pm -= ADLER_MOD;
                    __syncwarp();
                }
                pos += L;
            }
            __syncwarp();
            if (state) break;
        }
        // Adler-32 over every byte produced: a = 1 + S1, b = N (1 + S1) - S2 with S2 = sum of position * byte
        for (int d = 16; d; d >>= 1) {
            s1 += __shfl_xor_sync(0xffffffffu, s1, d);
            s2 += __shfl_xor_sync(0xffffffffu, s2, d);
        }
        fault = __any_sync(0xffffffffu, fault);
        if (lane == 0) {
            if (D.err) {
                R = PdecRecord{D.err, D.arg, 0, 0, D.produced};
            } else {
                const uint32_t a = (uint32_t)((1 + s1) % ADLER_MOD);
                const uint32_t b = (uint32_t)(((pos % ADLER_MOD) * a + ADLER_MOD - s2 % ADLER_MOD) % ADLER_MOD);
                const uint8_t *ad = zs + J.src_len - 4;
                const uint32_t stored = (uint32_t)ad[0] << 24 | (uint32_t)ad[1] << 16 | (uint32_t)ad[2] << 8 | ad[3];
                const uint32_t adler = b << 16 | a;
                if (fault) R = PdecRecord{kFault, 0, 0, 0, pos};
                else if (stored != adler) R = PdecRecord{kAdler, 0, stored, adler, pos};
                else if (pos != J.expected) R = PdecRecord{kSize, 0, stored, adler, pos};
                else if (bad_row_val != 0xFFFFFFFFu) R = PdecRecord{kFilter, bad_row_val, stored, adler, pos};
                else R = PdecRecord{kOk, 0, stored, adler, pos};
            }
            rec[f] = R;
        }
        __syncwarp();
    }
}

// ---- k_png_unfilter --------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t paeth(uint32_t a, uint32_t b, uint32_t c)
{
    const int p = (int)a + (int)b - (int)c;
    const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
    return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

// unfilter_row (png.rs:370-410) on one pixel of bpp bytes, packed little-endian in 64 bits: a its left neighbour,
// b the pixel above, c the one above-left (0 outside the row / frame)
__device__ __forceinline__ uint64_t unfilter_px(uint32_t ft, uint64_t raw, uint64_t a, uint64_t b, uint64_t c,
                                                uint32_t bpp)
{
    uint64_t o = 0;
#pragma unroll
    for (uint32_t j = 0; j < 8; ++j) {
        if (j >= bpp) break;
        const uint32_t x = (raw >> 8 * j) & 255, aj = (a >> 8 * j) & 255, bj = (b >> 8 * j) & 255,
                       cj = (c >> 8 * j) & 255;
        const uint32_t pred = ft == 1 ? aj : ft == 2 ? bj : ft == 3 ? (aj + bj) >> 1 : ft == 4 ? paeth(aj, bj, cj) : 0;
        o |= (uint64_t)((x + pred) & 255) << 8 * j;
    }
    return o;
}

struct UnfilterParams {
    const PdecFile *files;
    const PdecRecord *rec;
    const uint64_t *group_prefix;   // [n + 1]: the files' 32-row groups, in ticket order
    uint32_t n;
    uint64_t groups;
    uint8_t *scratch, *out;
    uint32_t *progress;             // [groups]: pixels of the group's last row written
    uint32_t *ticket;               // [0] next ticket, [1] status (bit 0: a wait timed out)
};

// A warp owns 32 rows of one file, one lane per row; lane k handles pixel s - k at step s, so lane k-1 has
// finished the pixel above one step before lane k needs it and passes it down with a shuffle (the one above-left
// stays in a register).  Groups are handed out through a ticket counter in order; lane 0 of a group waits for the
// previous group's last row, which publishes its progress every 32 pixels.  A group only waits on one a running warp
// claimed earlier, so the wavefront cannot deadlock; every wait is bounded and a timeout sets a status bit.
__global__ void __launch_bounds__(kUnfilterWarps * 32) k_png_unfilter(UnfilterParams P)
{
    const uint32_t lane = threadIdx.x & 31;
    volatile uint32_t *status = P.ticket + 1;
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(P.ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= P.groups) return;
        const uint32_t f = item_of(P.group_prefix, P.n, t);
        const PdecFile J = P.files[f];
        if (P.rec[f].code != kOk || (J.flags & kNoPlte)) continue;
        const uint32_t g = (uint32_t)(t - P.group_prefix[f]), groups = (J.height + 31) / 32;
        const uint64_t y = (uint64_t)g * 32 + lane, rowlen = J.sb + 1;
        const bool row_ok = y < J.height;
        const uint32_t bpp = J.bpp, U = (uint32_t)(J.sb / bpp);
        const bool direct = J.flags & kDirect;
        const uint8_t *src = P.scratch + J.scratch + y * rowlen;
        uint8_t *dst = direct ? P.out + J.out + y * J.sb : P.scratch + J.scratch + y * rowlen + 1;
        const uint8_t *above = g == 0 ? nullptr
                             : direct ? P.out + J.out + (y - 1) * J.sb : P.scratch + J.scratch + (y - 1) * rowlen + 1;
        const uint32_t ft = row_ok ? src[0] : 0;
        const bool publish = lane == 31 && g + 1 < groups;
        uint32_t seen = 0;
        uint64_t last = 0, up0 = 0;
        for (uint32_t s = 0; s < U + 31; ++s) {
            const int x = (int)s - (int)lane;
            uint64_t up = __shfl_up_sync(0xffffffffu, last, 1);
            const bool active = row_ok && x >= 0 && x < (int)U;
            if (lane == 0) {
                up = 0;
                if (above && active) {
                    if (seen <= (uint32_t)x) {
                        const volatile uint32_t *pw = P.progress + (t - 1);
                        uint32_t spins = 0, last_seen = *pw;
                        uint64_t since = globaltimer_ns();
                        while ((seen = *pw) <= (uint32_t)x) {
                            if (seen != last_seen) {   // the row above moved: the wait starts again
                                last_seen = seen;
                                since = globaltimer_ns();
                            }
                            if (*status || ((++spins & 63) == 0 && globaltimer_ns() - since > kStallNs)) {
                                atomicOr(P.ticket + 1, 1u);
                                seen = U;
                                break;
                            }
                            if (spins > 64) __nanosleep(128);
                        }
                        __threadfence();
                    }
                    for (uint32_t j = 0; j < bpp; ++j) up |= (uint64_t)__ldcg(above + (uint64_t)x * bpp + j) << 8 * j;
                }
            }
            if (x == 0) up0 = 0;   // nothing above-left of a row's first pixel
            if (active) {
                uint64_t raw = 0;
                for (uint32_t j = 0; j < bpp; ++j) raw |= (uint64_t)src[1 + (uint64_t)x * bpp + j] << 8 * j;
                const uint64_t v = unfilter_px(ft, raw, x ? last : 0, up, up0, bpp);
                for (uint32_t j = 0; j < bpp; ++j) dst[(uint64_t)x * bpp + j] = (uint8_t)(v >> 8 * j);
                last = v;
                if (publish && ((x & 31) == 31 || x == (int)U - 1)) {
                    __threadfence();
                    *(volatile uint32_t *)(P.progress + t) = (uint32_t)x + 1;
                }
            } else {
                last = 0;
            }
            up0 = up;
        }
    }
}

// ---- k_png_expand ----------------------------------------------------------------------------------------

// convert_to_pixels (png.rs:430-626) for the files that need more than their unfiltered rows: one thread per output
// pixel, kExpandThreads pixels of one file per CTA, the palette in shared memory
__global__ void __launch_bounds__(kExpandThreads) k_png_expand(const PdecFile *__restrict__ F,
                                                               const PdecRecord *__restrict__ rec,
                                                               const uint64_t *__restrict__ cta_prefix, uint32_t n,
                                                               const uint32_t *__restrict__ pal,
                                                               const uint8_t *__restrict__ scratch, uint8_t *out)
{
    __shared__ uint32_t P[256];
    const uint32_t f = item_of(cta_prefix, n, blockIdx.x);
    const PdecFile &J = F[f];
    if (rec[f].code != kOk || (J.flags & (kDirect | kNoPlte))) return;
    if (J.ctype == 3) P[threadIdx.x] = __ldg(pal + (uint64_t)J.pal * 256 + threadIdx.x);
    __syncthreads();
    const uint64_t i = (blockIdx.x - cta_prefix[f]) * kExpandThreads + threadIdx.x, W = J.width;
    if (i >= W * J.height) return;
    const uint64_t y = i / W, x = i % W;
    const uint8_t *row = scratch + J.scratch + y * (J.sb + 1) + 1;
    uint8_t *o = out + J.out + i * J.channels;
    const uint32_t bd = J.depth;
    if (J.depth == 16) {   // the high byte of every sample
        for (uint32_t c = 0; c < J.channels; ++c) o[c] = row[(x * J.channels + c) * 2];
        return;
    }
    uint32_t v = bd == 8 ? row[x] : (row[x * bd / 8] >> (8 - bd - (x * bd) % 8)) & ((1u << bd) - 1);
    if (J.ctype == 0) {   // scale_to_8bit: bit replication
        o[0] = (uint8_t)(bd == 1 ? (v ? 255 : 0) : bd == 2 ? v * 0x55 : v * 0x11);
        return;
    }
    const uint32_t e = P[v];
    o[0] = (uint8_t)(e >> 24);
    o[1] = (uint8_t)(e >> 16);
    o[2] = (uint8_t)(e >> 8);
    if (J.channels == 4) o[3] = (uint8_t)e;
}

// ---- the passes ------------------------------------------------------------------------------------------

struct PdecPass {
    PdecFile *files = nullptr;
    PdecChunk *chunks = nullptr;
    uint64_t *piece_prefix = nullptr, *group_prefix = nullptr, *cta_prefix = nullptr;
    uint32_t *crc_acc = nullptr, *order = nullptr, *pal = nullptr;
    uint8_t *bytes = nullptr;
    size_t up = 0;   // bytes of the uploaded part, from files to the end of bytes
    PdecRecord *rec = nullptr;
    uint32_t *progress = nullptr, *ctl = nullptr;   // ctl: inflate ticket, unfilter ticket and status
    uint8_t *rings = nullptr, *scratch = nullptr;
};

struct PassSizes {
    uint32_t n = 0, nchunks = 0, npal = 0, rings = 0;
    uint64_t bytes = 0, scratch = 0, groups = 0;
};

void describe_pass(Layout &L, const PassSizes &s, PdecPass &P)
{
    P.files = L.take<PdecFile>(s.n);
    P.chunks = L.take<PdecChunk>(s.nchunks);
    P.piece_prefix = L.take<uint64_t>(s.nchunks + 1);
    P.group_prefix = L.take<uint64_t>(s.n + 1);
    P.cta_prefix = L.take<uint64_t>(s.n + 1);
    P.crc_acc = L.take<uint32_t>(s.nchunks);
    P.order = L.take<uint32_t>(s.n);
    P.pal = L.take<uint32_t>((uint64_t)s.npal * 256);
    P.bytes = L.take<uint8_t>(s.bytes);
    P.up = L.end();
    P.rec = L.take<PdecRecord>(s.n);
    P.progress = L.take<uint32_t>(s.groups);
    P.ctl = L.take<uint32_t>(4);
    P.rings = L.take<uint8_t>((uint64_t)s.rings * kRing);
    P.scratch = L.take<uint8_t>(s.scratch);
}

// A file's device scratch in a pass
uint64_t file_scratch(const PdecParsed &p)
{
    return p.idat_total + p.scratch() + p.idat_len.size() * 28 + (p.height / 32 + 1) * 12 + 1024 + sizeof(PdecFile) +
           sizeof(PdecRecord) + 64;
}

// The file's status from its record: clear, pixo's error, or PIXO_B200_ERR_CUDA for a fault
void resolve(const PdecParsed &p, const PdecRecord &r, DecodeStatus &res)
{
    switch (r.code) {
    case kOk:
        if (p.ctype == 3 && !p.has_plte) decode_fail(res, kInvalidDecode, "missing PLTE chunk");
        else res = DecodeStatus();
        return;
    case kCrc: decode_fail(res, kInvalidDecode, "CRC mismatch in IDAT chunk"); return;
    case kEos: decode_fail(res, kInvalidDecode, "unexpected end of stream"); return;
    case kReservedBlock: decode_fail(res, kInvalidDecode, "reserved block type"); return;
    case kLenNlen: decode_fail(res, kInvalidDecode, "stored block LEN/NLEN mismatch"); return;
    case kEmptyTable: decode_fail(res, kInvalidDecode, "empty Huffman table"); return;
    case kBadCode: decode_fail(res, kInvalidDecode, "invalid Huffman code"); return;
    case kRepeatAtStart: decode_fail(res, kInvalidDecode, "repeat code at start"); return;
    case kTooManyLengths: decode_fail(res, kInvalidDecode, "too many code lengths"); return;
    case kBadLitLen: decode_fail(res, kInvalidDecode, "invalid literal/length code: %u", r.arg); return;
    case kBadDistCode: decode_fail(res, kInvalidDecode, "invalid distance code"); return;
    case kDistTooFar: decode_fail(res, kInvalidDecode, "distance too far back"); return;
    case kAdler:
        decode_fail(res, kInvalidDecode, "Adler32 mismatch: expected %08X, got %08X", r.stored_adler, r.adler);
        return;
    case kSize:
        decode_fail(res, kInvalidDecode, "decompressed size mismatch: expected %llu, got %llu",
                    (unsigned long long)p.expected, (unsigned long long)r.produced);
        return;
    case kFilter: decode_fail(res, kInvalidDecode, "invalid filter type: %u", r.arg); return;
    default: decode_fail(res, PIXO_B200_ERR_CUDA, "k_png_inflate: a file produced more than its scratch bound"); return;
    }
}

}  // namespace

int launch_decode(pixo_b200_ctx *ctx, const PdecParsed *const *files, const uint8_t *const *data, uint32_t n,
                  const uint64_t *out_off, uint8_t *d_out, DecodeStatus *res)
{
    for (uint32_t p0 = 0, p1; p0 < n; p0 = p1) {
        p1 = pass_end(files, p0, n, file_scratch);
        const uint32_t m = p1 - p0;
        PassSizes s;
        s.n = m;
        s.rings = (uint32_t)std::min<uint64_t>(m, (uint64_t)ctx->sm_count * 16);
        s.rings = (s.rings + kInflateWarps - 1) / kInflateWarps * kInflateWarps;
        for (uint32_t i = p0; i < p1; ++i) {
            const PdecParsed &f = *files[i];
            s.nchunks += (uint32_t)f.idat_len.size();
            s.npal += f.ctype == 3;
            s.bytes += f.idat_total;
            s.scratch += (f.scratch() + 15) / 16 * 16;
            s.groups += (f.height + 31) / 32;
        }
        PdecPass H;
        const std::vector<uint8_t> host = host_image(s, H);
        uint64_t by = 0, scr = 0, pieces = 0, groups = 0, ctas = 0;
        uint32_t c = 0, pal = 0;
        bool expand = false;
        for (uint32_t i = 0; i < m; ++i) {
            const PdecParsed &f = *files[p0 + i];
            PdecFile &J = H.files[i];
            memset(&J, 0, sizeof J);
            J.src = by;
            J.src_len = f.idat_total;
            J.scratch = scr;
            J.cap = f.scratch();
            J.expected = f.expected;
            J.sb = f.sb;
            J.out = out_off[p0 + i];
            J.chunk0 = c;
            J.nchunks = (uint32_t)f.idat_len.size();
            J.width = f.width;
            J.height = f.height;
            J.bpp = f.bpp;
            J.depth = f.depth;
            J.ctype = f.ctype;
            J.channels = f.out_channels;
            J.flags = (f.direct() ? kDirect : 0) | (f.ctype == 3 && !f.has_plte ? kNoPlte : 0);
            // the chunks: payloads back to back, each word starting as k_png_crc expects
            const uint8_t kIdat[4] = {'I', 'D', 'A', 'T'};
            const uint32_t s0 = crc32_update(0xFFFFFFFFu, kIdat, 4);
            for (size_t k = 0; k < f.idat_len.size(); ++k, ++c) {
                const uint32_t L = f.idat_len[k];
                memcpy(H.bytes + by, data[p0 + i] + f.idat_off[k], L);
                H.chunks[c] = PdecChunk{by, L};
                H.crc_acc[c] = crc32_shift(s0, L) ^ 0xFFFFFFFFu ^ f.idat_crc[k];
                H.piece_prefix[c] = pieces;
                pieces += (L + kCrcPiece - 1) / kCrcPiece;
                by += L;
            }
            if (f.ctype == 3) {   // index -> RGBA: past PLTE 0,0,0,255; past tRNS alpha 255
                J.pal = pal;
                uint32_t *T = H.pal + (uint64_t)pal++ * 256;
                const size_t np = f.plte.size() / 3;
                for (uint32_t k = 0; k < 256; ++k)
                    T[k] = k < np ? (uint32_t)f.plte[3 * k] << 24 | (uint32_t)f.plte[3 * k + 1] << 16 |
                                        (uint32_t)f.plte[3 * k + 2] << 8 | (k < f.trns.size() ? f.trns[k] : 255u)
                                  : 255u;
            }
            H.group_prefix[i] = groups;
            groups += (f.height + 31) / 32;
            H.cta_prefix[i] = ctas;
            if (!f.direct()) {
                ctas += ((uint64_t)f.width * f.height + kExpandThreads - 1) / kExpandThreads;
                expand = true;
            }
            scr += (f.scratch() + 15) / 16 * 16;
        }
        H.piece_prefix[c] = pieces;
        H.group_prefix[m] = groups;
        H.cta_prefix[m] = ctas;
        PdecPass D;
        PIXO_TRY(upload_pass(ctx, ctx->d_pdec, s, H, host, D));
        PIXO_CUDA(ctx, cudaMemsetAsync(D.ctl, 0, 16, ctx->stream));
        PIXO_CUDA(ctx, cudaMemsetAsync(D.progress, 0, groups * 4, ctx->stream));
        if (pieces)
            PIXO_TRY(launch(ctx, k_png_crc, dim3((unsigned)((pieces + 255) / 256)), dim3(256), 0, D.chunks,
                            D.piece_prefix, s.nchunks, pieces, D.bytes, D.crc_acc));
        PIXO_TRY(launch(ctx, k_png_inflate, dim3(s.rings / kInflateWarps), dim3(kInflateWarps * 32), 0, D.files,
                        D.order, m, D.crc_acc, D.bytes, D.scratch, D.rings, D.ctl, D.rec));
        const uint64_t uw = std::min<uint64_t>(groups, (uint64_t)ctx->sm_count * 32);
        UnfilterParams U{D.files, D.rec, D.group_prefix, m, groups, D.scratch, d_out, D.progress, D.ctl + 1};
        PIXO_TRY(launch(ctx, k_png_unfilter, dim3((unsigned)((uw + kUnfilterWarps - 1) / kUnfilterWarps)),
                        dim3(kUnfilterWarps * 32), 0, U));
        if (expand)
            PIXO_TRY(launch(ctx, k_png_expand, dim3((unsigned)ctas), dim3(kExpandThreads), 0, D.files, D.rec,
                            D.cta_prefix, m, D.pal, D.scratch, d_out));
        std::vector<PdecRecord> rec(m);
        uint32_t ctl[4];
        PIXO_CUDA(ctx, cudaMemcpyAsync(rec.data(), D.rec, m * sizeof(PdecRecord), cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaMemcpyAsync(ctl, D.ctl, 16, cudaMemcpyDeviceToHost, ctx->stream));
        PIXO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (ctl[2] & 1u)
            return set_error(ctx, PIXO_B200_ERR_CUDA, "k_png_unfilter: a row group's wait for the rows above timed out");
        for (uint32_t i = 0; i < m; ++i) {
            DecodeStatus &r = res[p0 + i];
            resolve(*files[p0 + i], rec[i], r);
            if (r.code == PIXO_B200_ERR_CUDA) return set_error(ctx, r.code, "%s", r.msg.c_str());
        }
    }
    return 0;
}

}  // namespace pixo
