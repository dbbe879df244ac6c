// jpeg_decode.cu — baseline JPEG decoding on the device, pixel-identical to pixo::decode::decode_jpeg
// (src/decode/jpeg.rs, bit_reader.rs, idct.rs).  The host parses the headers (jpeg_decode_host.cpp); here:
//   k_jdec_scan   one thread per file runs pixo's bit reader and MCU loop over the file's entropy bytes and writes
//                 the quantised coefficients (zig-zag order) at their block positions, plus the blocks it stored
//   k_jdec_idct   dequantise + pixo's integer IDCT, 8 lanes per block, into u8 component planes; a block at or past
//                 its file's stored count is 0, as pixo leaves the blocks it never stored
//   k_jdec_color  crop (gray) or ycbcr_to_rgb into each file's packed frame
// Arithmetic follows pixo's release build: integer overflow wraps, shift counts are masked, casts truncate.
#include <string.h>

#include "common.cuh"
#include "decode_host.hpp"
#include "jpeg_decode_host.hpp"

namespace pixo {

namespace {

// MsbBitReader (bit_reader.rs:141-235) over one file's entropy bytes; every read is bounded by their length
struct Reader {
    const uint8_t *data;
    uint64_t len, pos;
    uint32_t buf, nbits;   // nbits is pixo's u8 bits_in_buf: kept modulo 256

    // next_byte (:160-194): FF 00 is a stuffed FF; RSTn is skipped and clears the bit buffer at the moment the
    // byte is fetched; any other marker ends the data (the position backs up to the FF)
    __device__ bool next_byte(uint32_t &out)
    {
        for (;;) {
            if (pos >= len) return false;
            const uint32_t b = __ldg(data + pos++);
            if (b == 0xFF) {
                if (pos >= len) return false;
                const uint32_t nx = __ldg(data + pos);
                if (nx == 0x00) {
                    ++pos;
                } else if (nx >= 0xD0 && nx <= 0xD7) {
                    ++pos;
                    buf = 0;
                    nbits = 0;
                    continue;
                } else {
                    --pos;
                    return false;
                }
            }
            out = b;
            return true;
        }
    }
    // ensure + peek_bits (:198-215)
    __device__ bool peek(uint32_t n, uint32_t &out)
    {
        while (nbits < n) {
            uint32_t b;
            if (!next_byte(b)) return false;
            buf = (buf << 8) | b;
            nbits = (nbits + 8) & 0xFF;
        }
        out = (buf >> ((nbits - n) & 31)) & ((1u << (n & 31)) - 1u);
        return true;
    }
    // consume (:219-227)
    __device__ void consume(uint32_t n)
    {
        nbits = (nbits - n) & 0xFF;
        buf &= (nbits >= 32 ? 0u : (1u << nbits)) - 1u;
    }
    __device__ bool read(uint32_t n, uint32_t &out)
    {
        if (!peek(n, out)) return false;
        consume(n);
        return true;
    }
};

// HuffmanTable::decode / decode_slow (src/decode/jpeg.rs:150-179); t in shared memory, its values in global
__device__ bool huff_decode(const JdecHuff *__restrict__ t, const uint8_t *__restrict__ vals, Reader &r, uint32_t &sym)
{
    uint32_t p;
    if (r.peek(8, p)) {
        const uint32_t e = t->lookup[p], len = e >> 8;
        if (len > 0 && len <= 8) {
            r.consume(len);
            sym = e & 0xFF;
            return true;
        }
    }
    int32_t code = 0;
    for (int len = 1; len <= 16; ++len) {
        uint32_t bit;
        if (!r.read(1, bit)) return false;
        code = (int32_t)(((uint32_t)code << 1) | bit);
        if (code <= t->max_code[len]) {
            const int64_t idx = (int64_t)code + t->val_offset[len];
            if (idx < 0 || idx >= (int64_t)t->nvalues) return false;
            sym = __ldg(vals + t->values + idx);
            return true;
        }
    }
    return false;
}

// read_amplitude (src/decode/jpeg.rs:674-686), in wrapping i32
__device__ bool read_amplitude(Reader &r, uint32_t size, int32_t &out)
{
    uint32_t bits;
    if (!r.read(size, bits)) return false;
    const uint32_t thr = 1u << ((size - 1) & 31);
    out = (int32_t)bits < (int32_t)thr ? (int32_t)(bits - (2u * thr - 1u)) : (int32_t)bits;
    return true;
}

// The MCU loop of decode_scan (src/decode/jpeg.rs:486-612), one file per warp: the warp stages the file's tables in
// shared memory, then lane 0 decodes.  A warp of its own keeps the sequential chains of different files from sharing
// one instruction stream, so they run side by side on all SMs; blocks go in `order` (longest scan first, so the
// longest chain starts earliest).  Any read failure ends the file's loop; the block being decoded is not counted.
// coef is zero where nothing is written.
constexpr int kScanTables = 6;   // a DC and an AC table per component
static_assert(sizeof(JdecHuff) % 4 == 0, "tables are staged in words");
__global__ void __launch_bounds__(32) k_jdec_scan(const JdecFile *__restrict__ F, const JdecHuff *__restrict__ T,
                                                  const uint8_t *__restrict__ vals, const uint8_t *__restrict__ bytes,
                                                  const uint32_t *__restrict__ order, int16_t *__restrict__ coef,
                                                  uint64_t *__restrict__ stored)
{
    __shared__ JdecHuff tabs[kScanTables];
    const uint32_t f = order[blockIdx.x];
    const JdecFile &J = F[f];
    // the host lays a file's tables out consecutively: component c's DC table at dc[0] + 2c, its AC table after it
    const uint32_t first = J.dc[0], words = 2 * J.ncomp * (uint32_t)(sizeof(JdecHuff) / 4);
    const uint32_t *src = reinterpret_cast<const uint32_t *>(T + first);
    for (uint32_t k = threadIdx.x; k < words; k += 32) reinterpret_cast<uint32_t *>(tabs)[k] = __ldg(src + k);
    __syncwarp();
    if (threadIdx.x != 0) return;
    Reader r{bytes + J.src, J.src_len, 0, 0, 0};
    const uint32_t nc = J.ncomp, restart = J.restart, mw = J.mcu_w, mh = J.mcu_h;
    int32_t pred[3] = {0, 0, 0};
    uint64_t count = 0;
    uint32_t mcu_count = 0;
    for (uint32_t my = 0; my < mh; ++my)
        for (uint32_t mx = 0; mx < mw; ++mx) {
            if (restart > 0 && mcu_count > 0 && mcu_count % restart == 0) pred[0] = pred[1] = pred[2] = 0;
            for (uint32_t c = 0; c < nc; ++c) {
                const uint32_t h = J.h[c], v = J.v[c];
                const JdecHuff *dc = tabs + (J.dc[c] - first), *ac = tabs + (J.ac[c] - first);
                const uint64_t bw = (uint64_t)mw * h;
                for (uint32_t by = 0; by < v; ++by)
                    for (uint32_t bx = 0; bx < h; ++bx) {
                        int16_t *blk = coef + (J.coef[c] + ((uint64_t)my * v + by) * bw + (uint64_t)mx * h + bx) * 64;
                        uint32_t cat;
                        int32_t diff = 0;
                        if (!huff_decode(dc, vals, r, cat)) goto done;
                        if (cat > 0 && !read_amplitude(r, cat, diff)) goto done;
                        pred[c] = (int32_t)((uint32_t)pred[c] + (uint32_t)diff);
                        blk[0] = (int16_t)pred[c];
                        for (uint32_t k = 1; k < 64;) {
                            uint32_t s;
                            if (!huff_decode(ac, vals, r, s)) goto done;
                            if (s == 0) break;
                            if (s == 0xF0) {
                                k += 16;
                                continue;
                            }
                            k += s >> 4;
                            if (k >= 64) break;
                            if (s & 15) {
                                int32_t a;
                                if (!read_amplitude(r, s & 15, a)) goto done;
                                blk[k] = (int16_t)a;
                            }
                            ++k;
                        }
                        ++count;
                    }
            }
            ++mcu_count;
        }
done:
    stored[f] = count;
}

__device__ __forceinline__ int32_t fix_mul(int32_t a, int32_t b) { return (int32_t)(((int64_t)a * b) >> 13); }
__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
__device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }

// one 1-D pass of idct_2d_integer (src/decode/idct.rs:49-113, 118-192) before its descale: o[k] is output k
__device__ __forceinline__ void idct_1d(const int32_t d[8], int32_t o[8])
{
    const int32_t t0 = (int32_t)((uint32_t)d[0] << 13), t1 = (int32_t)((uint32_t)d[2] << 13);
    const int32_t t2 = (int32_t)((uint32_t)d[4] << 13), t3 = (int32_t)((uint32_t)d[6] << 13);
    const int32_t tmp10 = wadd(t0, t2), tmp11 = wsub(t0, t2);
    const int32_t z1 = fix_mul(wadd(t1, t3), 4433);
    const int32_t tmp12 = wsub(z1, fix_mul(t3, 15137)), tmp13 = wadd(z1, fix_mul(t1, 6270));
    const int32_t e0 = wadd(tmp10, tmp13), e3 = wsub(tmp10, tmp13), e1 = wadd(tmp11, tmp12), e2 = wsub(tmp11, tmp12);
    const int32_t z5 = fix_mul(wadd(d[1], d[5]), 9633);
    const int32_t y1 = fix_mul(wadd(d[1], d[7]), -7373), y2 = fix_mul(wadd(d[3], d[5]), -20995);
    const int32_t y3 = wadd(fix_mul(wadd(d[5], d[7]), -16069), z5), y4 = wadd(fix_mul(wadd(d[1], d[3]), -3196), z5);
    const int32_t o10 = wadd(wadd(fix_mul(d[1], 2446), y1), y3), o11 = wadd(wadd(fix_mul(d[3], 16819), y2), y4);
    const int32_t o12 = wadd(wadd(fix_mul(d[5], 25172), y2), y3), o13 = wadd(wadd(fix_mul(d[7], 12299), y1), y4);
    o[0] = wadd(e0, o13); o[7] = wsub(e0, o13);
    o[1] = wadd(e1, o12); o[6] = wsub(e1, o12);
    o[2] = wadd(e2, o11); o[5] = wsub(e2, o11);
    o[3] = wadd(e3, o10); o[4] = wsub(e3, o10);
}

__constant__ uint8_t c_zz_nat[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

constexpr int kIdctThreads = 256;

// dequantize (idct.rs:214-230) + idct_2d_integer (:45-204) over every block of a pass.  Lane l of a block's 8 loads
// zig-zag positions 8l..8l+7, does column l of pass 1 and row l of pass 2; the block goes between the steps through
// shared memory.
__global__ void __launch_bounds__(kIdctThreads) k_jdec_idct(const JdecFile *__restrict__ F,
                                                            const uint64_t *__restrict__ blk_prefix, uint32_t n,
                                                            uint64_t total, const int16_t *__restrict__ coef,
                                                            const uint64_t *__restrict__ stored,
                                                            uint8_t *__restrict__ planes)
{
    __shared__ int32_t ws[kIdctThreads / 8][64];
    const uint64_t g = ((uint64_t)blockIdx.x * kIdctThreads + threadIdx.x) / 8;
    const uint32_t lane = threadIdx.x & 7;
    const unsigned group = 0xFFu << (threadIdx.x & 24);   // the block's 8 lanes: they return together
    if (g >= total) return;
    const uint32_t f = item_of(blk_prefix, n, g);
    const JdecFile &J = F[f];
    uint64_t b = g - __ldg(blk_prefix + f);   // block within the file, component planes in turn
    uint32_t c = 0;
    uint64_t bw = (uint64_t)J.mcu_w * J.h[0], nb = bw * J.mcu_h * J.v[0];
    while (b >= nb && c + 1 < J.ncomp) {
        b -= nb;
        ++c;
        bw = (uint64_t)J.mcu_w * J.h[c];
        nb = bw * J.mcu_h * J.v[c];
    }
    const uint32_t h = J.h[c], v = J.v[c];
    const uint64_t px = b % bw, py = b / bw;
    // the block's place in decode order: its MCU, the component's first block there, its row and column in the MCU
    const uint64_t di = ((py / v) * J.mcu_w + px / h) * J.bpm + J.first[c] + (py % v) * h + px % h;
    uint2 *dst = reinterpret_cast<uint2 *>(planes + J.plane[c] + (py * 8 + lane) * (bw * 8) + px * 8);
    if (di >= __ldg(stored + f)) {   // never stored: pixo's plane keeps its 0
        *dst = make_uint2(0, 0);
        return;
    }
    int32_t *w = ws[threadIdx.x / 8];
    const int4 raw = __ldg(reinterpret_cast<const int4 *>(coef + (J.coef[c] + b) * 64) + lane);
    const uint4 qraw = __ldg(reinterpret_cast<const uint4 *>(J.quant[c]) + lane);
    const int16_t *k8 = reinterpret_cast<const int16_t *>(&raw);
    const uint16_t *q8 = reinterpret_cast<const uint16_t *>(&qraw);
#pragma unroll
    for (int j = 0; j < 8; ++j) w[c_zz_nat[lane * 8 + j]] = (int32_t)k8[j] * (int32_t)q8[j];
    __syncwarp(group);
    int32_t d[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = w[lane + 8 * k];
    idct_1d(d, o);
    __syncwarp(group);
#pragma unroll
    for (int k = 0; k < 8; ++k) w[lane + 8 * k] = wadd(o[k], 1 << 10) >> 11;
    __syncwarp(group);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = w[lane * 8 + k];
    idct_1d(d, o);
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int32_t p = wadd(wadd(o[k], 1 << 17) >> 18, 128);
        const uint32_t u = (uint32_t)min(max(p, 0), 255);
        if (k < 4) lo |= u << (8 * k);
        else hi |= u << (8 * (k - 4));
    }
    *dst = make_uint2(lo, hi);
}

// Crop (gray, src/decode/jpeg.rs:615-631) or ycbcr_to_rgb (:689-735) of every pixel of a pass into the files'
// packed frames.  Plane indices are pixo's flat ones, so a read past a plane gives 0 (Y) or 128 (Cb, Cr) as there.
__global__ void k_jdec_color(const JdecFile *__restrict__ F, const uint64_t *__restrict__ px_prefix, uint32_t n,
                             uint64_t total, const uint8_t *__restrict__ planes, uint8_t *__restrict__ out)
{
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= total) return;
    const uint32_t f = item_of(px_prefix, n, g);
    const JdecFile &J = F[f];
    const uint64_t i = g - __ldg(px_prefix + f), W = J.width, y = i / W, x = i % W;
    const uint8_t *p0 = planes + J.plane[0];
    if (J.ncomp == 1) {   // the plane can be smaller than the frame: a second SOF0 keeps the first one's maxima
        const uint64_t yi = y * ((uint64_t)J.mcu_w * J.h[0] * 8) + x;
        out[J.out + i] = yi < J.plane_len[0] ? p0[yi] : 0;
        return;
    }
    const uint64_t yw = (uint64_t)J.mcu_w * J.max_h * 8;
    const uint32_t hb = J.max_h / J.h[1], vb = J.max_v / J.v[1], hr = J.max_h / J.h[2], vr = J.max_v / J.v[2];
    const uint64_t yi = y * yw + x;
    const uint64_t bi = (y / vb) * ((uint64_t)J.mcu_w * J.h[1] * 8) + x / hb;
    const uint64_t ri = (y / vr) * ((uint64_t)J.mcu_w * J.h[2] * 8) + x / hr;
    const int32_t Y = yi < J.plane_len[0] ? p0[yi] : 0;
    const int32_t cb = (bi < J.plane_len[1] ? planes[J.plane[1] + bi] : 128) - 128;
    const int32_t cr = (ri < J.plane_len[2] ? planes[J.plane[2] + ri] : 128) - 128;
    const int32_t r = Y + ((cr * 359) >> 8), gg = Y - ((cb * 88 + cr * 183) >> 8), bb = Y + ((cb * 454) >> 8);
    uint8_t *o = out + J.out + 3 * i;
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[1] = (uint8_t)min(max(gg, 0), 255);
    o[2] = (uint8_t)min(max(bb, 0), 255);
}

// A pass's scratch: the records, tables, values and entropy bytes as uploaded (one region, `up` bytes), then the
// stored counts, coefficient planes and u8 planes
struct JdecPass {
    JdecFile *files = nullptr;
    JdecHuff *tabs = nullptr;
    uint32_t *order = nullptr;
    uint64_t *blk_prefix = nullptr, *px_prefix = nullptr;
    uint8_t *vals = nullptr, *bytes = nullptr;
    uint64_t *stored = nullptr;
    int16_t *coef = nullptr;
    uint8_t *planes = nullptr;
    size_t up = 0;   // bytes of the uploaded part, from files to the end of bytes
};

struct PassSizes {
    uint32_t n = 0, ntab = 0;
    uint64_t vals = 0, bytes = 0, blocks = 0;
};

void describe_pass(Layout &L, const PassSizes &s, JdecPass &P)
{
    P.files = L.take<JdecFile>(s.n);
    P.tabs = L.take<JdecHuff>(s.ntab);
    P.order = L.take<uint32_t>(s.n);
    P.blk_prefix = L.take<uint64_t>(s.n + 1);
    P.px_prefix = L.take<uint64_t>(s.n + 1);
    P.vals = L.take<uint8_t>(s.vals);
    P.bytes = L.take<uint8_t>(s.bytes);
    P.up = L.end();
    P.stored = L.take<uint64_t>(s.n);
    P.coef = L.take<int16_t>(s.blocks * 64);
    P.planes = L.take<uint8_t>(s.blocks * 64);
}

// A file's device scratch in a pass.  Scratch is what ends a JPEG pass: every file is charged at least
// kJdecFileTables, so a pass holds fewer than kDecodePassFiles files.
constexpr uint64_t kJdecFileTables = 8 * 2048;   // a file's tables, values, order and prefix entries, rounded up
static_assert(kDecodePassBytes / (kJdecFileTables + sizeof(JdecFile)) < kDecodePassFiles, "passes end by scratch");

uint64_t file_scratch(const JdecParsed &p)
{
    return p.blocks() * 192 + p.entropy_len + sizeof(JdecFile) + kJdecFileTables;
}

}  // namespace

int launch_decode(pixo_b200_ctx *ctx, const JdecParsed *const *files, const uint8_t *const *data, uint32_t n,
                  const uint64_t *out_off, uint8_t *d_out, DecodeStatus *)
{
    for (uint32_t p0 = 0, p1; p0 < n; p0 = p1) {
        p1 = pass_end(files, p0, n, file_scratch);
        const uint32_t m = p1 - p0;
        PassSizes s;
        s.n = m;
        for (uint32_t i = p0; i < p1; ++i) {
            const JdecParsed &f = *files[i];
            for (uint32_t c = 0; c < f.ncomp; ++c) s.vals += f.vals[f.dc[c]].size() + f.vals[4 + f.ac[c]].size();
            s.ntab += 2 * f.ncomp;
            s.bytes += f.entropy_len;
            s.blocks += f.blocks();
        }
        JdecPass H;
        const std::vector<uint8_t> host = host_image(s, H);
        uint32_t t = 0;
        uint64_t v = 0, by = 0, blk = 0, plane = 0, px = 0;
        for (uint32_t i = 0; i < m; ++i) {
            const JdecParsed &f = *files[p0 + i];
            JdecFile &J = H.files[i];
            memset(&J, 0, sizeof J);
            J.src = by;
            J.src_len = f.entropy_len;
            memcpy(H.bytes + by, data[p0 + i] + f.entropy, f.entropy_len);
            by += f.entropy_len;
            J.out = out_off[p0 + i];
            J.width = f.width;
            J.height = f.height;
            J.mcu_w = f.mcu_w();
            J.mcu_h = f.mcu_h();
            J.ncomp = f.ncomp;
            J.restart = f.restart;
            J.max_h = f.max_h;
            J.max_v = f.max_v;
            H.blk_prefix[i] = blk;
            H.px_prefix[i] = px;
            for (uint32_t c = 0; c < f.ncomp; ++c) {
                J.h[c] = f.h[c];
                J.v[c] = f.v[c];
                J.first[c] = J.bpm;
                J.bpm += f.h[c] * f.v[c];
                J.coef[c] = blk;
                J.plane[c] = plane;
                J.plane_len[c] = f.plane_w(c) * f.plane_h(c);
                blk += J.plane_len[c] / 64;
                plane += J.plane_len[c];
                memcpy(J.quant[c], f.quant[f.q[c]], sizeof J.quant[c]);
                const int src[2] = {f.dc[c], 4 + f.ac[c]};
                uint32_t *dst[2] = {&J.dc[c], &J.ac[c]};
                for (int k = 0; k < 2; ++k) {
                    JdecHuff &T = H.tabs[t];
                    T = f.tab[src[k]];
                    T.values = (uint32_t)v;
                    memcpy(H.vals + v, f.vals[src[k]].data(), f.vals[src[k]].size());
                    v += f.vals[src[k]].size();
                    *dst[k] = t++;
                }
            }
            px += f.width * (uint64_t)f.height;
        }
        H.blk_prefix[m] = blk;
        H.px_prefix[m] = px;
        JdecPass D;
        PIXO_TRY(upload_pass(ctx, ctx->d_jdec, s, H, host, D));
        if (s.blocks) PIXO_CUDA(ctx, cudaMemsetAsync(D.coef, 0, s.blocks * 128, ctx->stream));
        PIXO_TRY(launch(ctx, k_jdec_scan, dim3(m), dim3(32), 0, D.files, D.tabs, D.vals, D.bytes, D.order, D.coef,
                        D.stored));
        if (s.blocks)
            PIXO_TRY(launch(ctx, k_jdec_idct, dim3((unsigned)((s.blocks * 8 + kIdctThreads - 1) / kIdctThreads)),
                            dim3(kIdctThreads), 0, D.files, D.blk_prefix, m, s.blocks, D.coef, D.stored, D.planes));
        if (px)
            PIXO_TRY(launch(ctx, k_jdec_color, dim3((unsigned)((px + 255) / 256)), dim3(256), 0, D.files, D.px_prefix,
                            m, px, D.planes, d_out));
    }
    return 0;
}

}  // namespace pixo
