/*
 * jpeg_progressive.c — CPU restatement of pixo's progressive encoder as its encode_into runs it with
 * options.progressive (src/jpeg/mod.rs:395-447, encode_progressive :872-927, encode_dc_scan /
 * encode_ac_first_scan :1248-1365; src/jpeg/progressive.rs simple_progressive_script :98-110,
 * encode_ac_first :141-210, flush_eob_run :313-345, get_code_from_table :363-380 with its (0, 4)
 * fallback; BitWriterMsb src/bits.rs:195-278).  Writes whole files.
 *
 * TEST INFRASTRUCTURE ONLY (see pixo_oracle.h).  Headers and tables come from pixo_oracle.c: the
 * baseline file po_jpeg_encode_from_coefficients writes for the plain-rounded coefficients carries
 * exactly the SOI..DRI pixo writes for the progressive file (same DQT, same DHT: pixo builds the optimised
 * tables from the plain-rounded statistics in both modes), with SOF0 where pixo writes SOF2.  The
 * coefficients come from pixo_oracle.c (plain) or jpeg_trellis.c (trellis_quant).  Built by
 * oracle/jpeg_progressive.py.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "pixo_oracle.h"

void po_jpeg_coefficients_trellis(const uint8_t *data, uint32_t w, uint32_t h, int color_type, int subsampling,
                                  const float lum_q[64], const float chr_q[64], int16_t *y, int16_t *cb,
                                  int16_t *cr);

typedef struct {
    uint8_t *buf;
    size_t cap, n;
    uint32_t cur, pos;   /* pos: free bits in cur (8 = empty) */
    int overflow;
} bw_t;

static void bw_byte(bw_t *w)
{
    if (w->n + 2 > w->cap) { w->overflow = 1; }
    else {
        w->buf[w->n++] = (uint8_t)w->cur;
        if (w->cur == 0xFF) w->buf[w->n++] = 0;
    }
    w->cur = 0;
    w->pos = 8;
}

static void bw_write(bw_t *w, uint32_t value, uint32_t n)
{
    while (n > 0) {
        const uint32_t t = n < w->pos ? n : w->pos;
        const uint32_t bits = (value >> (n - t)) & ((1u << t) - 1u);
        w->pos -= t;
        w->cur |= bits << w->pos;
        n -= t;
        if (w->pos == 0) bw_byte(w);
    }
}

static void bw_finish(bw_t *w)
{
    if (w->pos < 8) {
        w->cur |= (1u << w->pos) - 1u;
        bw_byte(w);
    }
}

/* get_code_from_table over one DHT table (16 counts, then the values) */
typedef struct { uint16_t code[256]; uint8_t len[256]; } codes_t;

static void codes_from(const uint8_t bits[16], const uint8_t *vals, codes_t *c)
{
    for (int s = 0; s < 256; ++s) { c->code[s] = 0; c->len[s] = 4; }
    uint8_t seen[256] = {0};
    uint32_t code = 0;
    int idx = 0;
    for (int l = 0; l < 16; ++l) {
        for (int k = 0; k < bits[l]; ++k, ++idx, ++code)
            if (!seen[vals[idx]]) {
                seen[vals[idx]] = 1;
                c->code[vals[idx]] = (uint16_t)code;
                c->len[vals[idx]] = (uint8_t)(l + 1);
            }
        code <<= 1;
    }
}

static int cat_of(int v)
{
    unsigned a = (unsigned)(v < 0 ? -v : v);
    int n = 0;
    while (a) { ++n; a >>= 1; }
    return n;
}

static void put_sym(bw_t *w, const codes_t *t, int sym) { bw_write(w, t->code[sym], t->len[sym]); }

static void put_value(bw_t *w, int v, int cat)
{
    if (cat) bw_write(w, (uint32_t)(v < 0 ? v - 1 : v) & ((1u << cat) - 1u), (uint32_t)cat);
}

static void flush_eob(bw_t *w, const codes_t *ac, uint32_t *run)
{
    if (!*run) return;
    int nbits = 0;
    while ((*run >> (nbits + 1)) != 0) ++nbits;
    put_sym(w, ac, nbits << 4);
    if (nbits) bw_write(w, *run - (1u << nbits), (uint32_t)nbits);
    *run = 0;
}

static const int SCRIPT[7][3] = {{0, 0, 0}, {1, 0, 0}, {2, 0, 0}, {0, 1, 10}, {0, 11, 63}, {1, 1, 63}, {2, 1, 63}};

/* The 7 entropy-coded segments of simple_progressive_script over natural-order arrays (blocks in array
 * order), with the tables of dht (4 x (16 counts + 256 values): dc_lum, dc_chrom, ac_lum, ac_chrom).
 * Segment s goes to out + off, its length to lens[s].  Returns the total, or -1 when cap is too small. */
long po_progressive_scans(const int16_t *y, size_t ny, const int16_t *cb, const int16_t *cr, size_t nc,
                          const uint8_t *dht, uint8_t *out, size_t cap, size_t lens[7])
{
    codes_t *t = malloc(4 * sizeof(codes_t));
    for (int k = 0; k < 4; ++k) codes_from(dht + k * 272, dht + k * 272 + 16, &t[k]);
    size_t total = 0;
    int bad = 0;
    for (int s = 0; s < 7; ++s) {
        const int comp = SCRIPT[s][0], ss = SCRIPT[s][1], se = SCRIPT[s][2];
        const int16_t *blocks = comp == 0 ? y : (comp == 1 ? cb : cr);
        const size_t nb = comp == 0 ? ny : nc;
        const codes_t *dc = &t[comp ? 1 : 0], *ac = &t[comp ? 3 : 2];
        bw_t w = {out + total, cap - total, 0, 0, 8, 0};
        if (ss == 0) {
            int prev = 0;
            for (size_t b = 0; b < nb; ++b) {
                const int d = blocks[b * 64];
                const int diff = (int)(int16_t)(d - prev);
                const int cat = cat_of(diff);
                put_sym(&w, dc, cat);
                put_value(&w, diff, cat);
                prev = d;
            }
        } else {
            uint32_t run = 0;
            for (size_t b = 0; b < nb; ++b) {
                const int16_t *blk = blocks + b * 64;
                int last = ss - 1;
                for (int k = ss; k <= se; ++k)
                    if (blk[PO_ZIGZAG[k]]) last = k;
                if (last < ss) {
                    if (++run == 0x7FFF) flush_eob(&w, ac, &run);
                    continue;
                }
                flush_eob(&w, ac, &run);
                int zr = 0;
                for (int k = ss; k <= last; ++k) {
                    const int c = blk[PO_ZIGZAG[k]];
                    if (!c) { ++zr; continue; }
                    while (zr >= 16) { put_sym(&w, ac, 0xF0); zr -= 16; }
                    const int cat = cat_of(c);
                    put_sym(&w, ac, (zr << 4) | cat);
                    put_value(&w, c, cat);
                    zr = 0;
                }
                if (last < se) run = 1;
            }
            flush_eob(&w, ac, &run);
        }
        bw_finish(&w);
        bad |= w.overflow;
        lens[s] = w.n;
        total += w.n;
    }
    free(t);
    return bad ? -1 : (long)total;
}

/* Parses the DHT segments of a baseline file into dht[4 * 272]; returns the offset of its SOS marker. */
static size_t read_headers(const uint8_t *f, size_t n, uint8_t *dht)
{
    size_t i = 2;
    memset(dht, 0, 4 * 272);
    while (i + 4 <= n) {
        const int m = f[i + 1];
        const size_t len = ((size_t)f[i + 2] << 8) | f[i + 3];
        if (m == 0xDA) return i;
        if (m == 0xC4) {
            size_t j = i + 4;
            while (j < i + 2 + len) {
                const int tc = f[j] >> 4, th = f[j] & 15, k = tc * 2 + th;
                int cnt = 0;
                for (int l = 0; l < 16; ++l) cnt += f[j + 1 + l];
                memcpy(dht + k * 272, f + j + 1, 16);
                memcpy(dht + k * 272 + 16, f + j + 17, (size_t)cnt);
                j += 17 + (size_t)cnt;
            }
        }
        i += 2 + len;
    }
    return 0;
}

/* encode_into with progressive = true.  Returns bytes written or po_jpeg_encode's negative errors. */
long po_jpeg_encode_progressive(const uint8_t *data, size_t data_len, uint32_t w, uint32_t h, int color_type,
                                int quality, int subsampling, uint32_t restart_interval, int optimize_huffman,
                                int trellis_quant, uint8_t *out, size_t cap)
{
    if (quality < 1 || quality > 100) return -1;
    if (w == 0 || h == 0) return -2;
    if (w > 65535 || h > 65535) return -3;
    if (color_type != PO_RGB && color_type != PO_GRAY) return -4;
    if (data_len != (size_t)w * h * (color_type == PO_GRAY ? 1 : 3)) return -5;
    size_t ny, nc;
    po_jpeg_block_counts(w, h, color_type, subsampling, &ny, &nc);
    uint8_t lz[64], cz[64];
    float lq[64], cq[64];
    po_quant_tables(quality, lz, cz, lq, cq);
    const size_t nca = nc ? nc : 1;
    int16_t *y = calloc(ny * 64, 2), *cb = calloc(nca * 64, 2), *cr = calloc(nca * 64, 2);
    po_jpeg_coefficients(data, w, h, color_type, subsampling, lq, cq, y, cb, cr, 0, 0);
    /* the baseline file of the plain coefficients: pixo's headers and tables */
    const size_t bcap = ny * 64 * 8 + nc * 64 * 16 + 65536;
    uint8_t *base = malloc(bcap);
    long rc = po_jpeg_encode_from_coefficients(y, cb, cr, w, h, color_type, quality, subsampling, restart_interval,
                                               optimize_huffman, base, bcap);
    uint8_t dht[4 * 272];
    size_t hdr = rc > 0 ? read_headers(base, (size_t)rc, dht) : 0;
    if (rc > 0 && hdr + 2 > cap) rc = -6;
    if (rc > 0) {
        memcpy(out, base, hdr);
        for (size_t i = 2; i < hdr;) {   /* SOF0 -> SOF2 */
            if (out[i + 1] == 0xC0) out[i + 1] = 0xC2;
            i += 2 + (((size_t)out[i + 2] << 8) | out[i + 3]);
        }
        if (trellis_quant) po_jpeg_coefficients_trellis(data, w, h, color_type, subsampling, lq, cq, y, cb, cr);
        /* segments first (at the end of out), then moved behind their SOS headers */
        size_t lens[7];
        const size_t room = cap - hdr - 2 - 70;
        long body = cap > hdr + 72 ? po_progressive_scans(y, ny, cb, cr, nc, dht, out + hdr + 70, room, lens) : -1;
        if (body < 0) {
            rc = -6;
        } else {
            uint8_t *seg = malloc((size_t)body + 1);
            memcpy(seg, out + hdr + 70, (size_t)body);
            size_t p = hdr, o = 0;
            for (int s = 0; s < 7; ++s) {
                const uint8_t sos[10] = {0xFF, 0xDA, 0, 8, 1, (uint8_t)(SCRIPT[s][0] + 1),
                                         (uint8_t)(SCRIPT[s][0] ? 0x11 : 0x00), (uint8_t)SCRIPT[s][1],
                                         (uint8_t)SCRIPT[s][2], 0};
                memcpy(out + p, sos, 10);
                p += 10;
                memcpy(out + p, seg + o, lens[s]);
                p += lens[s];
                o += lens[s];
            }
            out[p++] = 0xFF;
            out[p++] = 0xD9;
            free(seg);
            rc = (long)p;
        }
    }
    free(base); free(y); free(cb); free(cr);
    return rc;
}
