/* jpeg_decode.c - CPU restatement of pixo::decode::decode_jpeg (src/decode/jpeg.rs, bit_reader.rs,
 * idct.rs) for the tests.  Written from the contract, not from the source: every function cites the
 * lines it restates.
 *
 * pixo ships a release build (Cargo.toml: no overflow checks), so integer overflow wraps, shift counts are
 * masked to the type's width and `as` casts truncate.  All of that is written here with unsigned arithmetic,
 * so nothing is undefined in C.
 *
 * jd_decode(data, len, pixels, coefs, info, msg):
 *   info[0] status: 0 Ok, 1 Error::InvalidDecode, 2 Error::UnsupportedDecode, 3 a file pixo panics on (an SOS
 *           with no components before any SOF0: ycbcr_to_rgb indexes components[1])
 *   info[1..3] width, height, colour type (0 Gray, 2 Rgb)
 *   info[4] component count, info[5] blocks of the scan (decode order), info[6] blocks stored
 *   info[7] pixel bytes
 *   msg: pixo's message (without the "Decode error: " prefix), 256 bytes
 * pixels (info[7] bytes) and coefs (info[5] blocks of 64 int16, zig-zag order, in decode order: MCU by MCU,
 * component by component, the component's blocks of the MCU row by row) may be NULL: the call then only parses
 * the headers, which decide every error. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    uint16_t lookup[256];
    uint8_t *values;
    uint32_t nvalues;
    int32_t max_code[17];
    int32_t val_offset[17];
} Huff;

typedef struct {
    uint8_t id, h, v, q, dc, ac;
} Comp;

typedef struct {
    const uint8_t *data;
    size_t len, pos;
    uint32_t width, height;
    Comp comp[3];
    uint32_t ncomp;
    uint16_t quant[4][64];
    Huff dc[4], ac[4];
    uint16_t restart_interval;
    uint8_t max_h, max_v;
    char *msg;
} Dec;

enum { OK = 0, INVALID = 1, UNSUPPORTED = 2, PANIC = 3 };

static int fail(Dec *d, int kind, const char *m)
{
    snprintf(d->msg, 256, "%s", m);
    return kind;
}

/* HuffmanTable::build, jpeg.rs:77-147 */
static void huff_build(Huff *t, const uint8_t bits[16], const uint8_t *values, uint32_t nvalues)
{
    free(t->values);
    memset(t, 0, sizeof *t);
    t->values = (uint8_t *)malloc(nvalues ? nvalues : 1);
    memcpy(t->values, values, nvalues);
    t->nvalues = nvalues;
    uint8_t *huffsize = (uint8_t *)malloc(nvalues ? nvalues : 1);
    uint16_t *huffcode = (uint16_t *)malloc(2 * (nvalues ? nvalues : 1));
    uint32_t n = 0;
    for (int i = 0; i < 16; ++i)
        for (int c = 0; c < bits[i]; ++c) huffsize[n++] = (uint8_t)(i + 1);
    uint32_t code = 0;
    uint8_t si = n ? huffsize[0] : 0;
    for (uint32_t k = 0; k < n; ++k) {
        while (huffsize[k] > si) {
            code <<= 1;
            si++;
        }
        huffcode[k] = (uint16_t)code;
        code++;
    }
    uint32_t val_idx = 0;
    for (int i = 1; i <= 16; ++i) {
        if (bits[i - 1] > 0) {
            t->val_offset[i] = (int32_t)(val_idx - (val_idx < n ? huffcode[val_idx] : 0));
            val_idx += bits[i - 1];
            t->max_code[i] = huffcode[val_idx - 1];
        } else {
            t->max_code[i] = -1;
        }
    }
    t->max_code[0] = -1;
    uint32_t code_idx = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int c = 0; c < bits[len - 1]; ++c) {
            if (len <= 8) {
                const uint32_t fill = 8 - len, base = (uint32_t)huffcode[code_idx] << fill;
                for (uint32_t i = 0; i < (1u << fill); ++i)
                    if ((base | i) < 256) t->lookup[base | i] = (uint16_t)(values[code_idx] | (len << 8));
            }
            code_idx++;
        }
    }
    free(huffsize);
    free(huffcode);
}

static void huff_default(Huff *t)
{
    memset(t, 0, sizeof *t);
    for (int i = 0; i < 17; ++i) t->max_code[i] = -1;
}

/* ---- MsbBitReader, bit_reader.rs:141-235 ---- */
typedef struct {
    const uint8_t *data;
    size_t len, pos;
    uint32_t buf;
    uint8_t nbits;
} Reader;

/* next_byte, :160-194: FF 00 is a stuffed FF; RSTn is skipped and clears the bit buffer; any other marker
 * backs up to the FF and fails */
static int next_byte(Reader *r, uint8_t *out)
{
    for (;;) {
        if (r->pos >= r->len) return -1;
        const uint8_t b = r->data[r->pos++];
        if (b == 0xFF) {
            if (r->pos >= r->len) return -1;
            const uint8_t nx = r->data[r->pos];
            if (nx == 0x00) {
                r->pos++;
            } else if (nx >= 0xD0 && nx <= 0xD7) {
                r->pos++;
                r->buf = 0;
                r->nbits = 0;
                continue;
            } else {
                r->pos--;
                return -1;
            }
        }
        *out = b;
        return 0;
    }
}

/* ensure / peek_bits, :198-215 (bits_in_buf is a u8 and wraps) */
static int peek_bits(Reader *r, uint8_t n, uint32_t *out)
{
    while (r->nbits < n) {
        uint8_t b;
        if (next_byte(r, &b)) return -1;
        r->buf = (r->buf << 8) | b;
        r->nbits = (uint8_t)(r->nbits + 8);
    }
    const uint32_t s = (uint8_t)(r->nbits - n) & 31u;
    *out = (r->buf >> s) & ((1u << (n & 31u)) - 1u);
    return 0;
}

/* consume, :219-227 */
static void consume(Reader *r, uint8_t n)
{
    r->nbits = (uint8_t)(r->nbits - n);
    r->buf &= (r->nbits >= 32 ? 0u : (1u << r->nbits)) - 1u;
}

static int read_bits(Reader *r, uint8_t n, uint32_t *out)
{
    if (peek_bits(r, n, out)) return -1;
    consume(r, n);
    return 0;
}

/* HuffmanTable::decode / decode_slow, jpeg.rs:150-179 */
static int huff_decode(const Huff *t, Reader *r, uint8_t *sym)
{
    uint32_t peek;
    if (peek_bits(r, 8, &peek) == 0) {
        const uint16_t e = t->lookup[peek];
        const uint8_t len = (uint8_t)(e >> 8);
        if (len > 0 && len <= 8) {
            consume(r, len);
            *sym = (uint8_t)e;
            return 0;
        }
    }
    int32_t code = 0;
    for (int len = 1; len <= 16; ++len) {
        uint32_t bit;
        if (read_bits(r, 1, &bit)) return -1;
        code = (int32_t)(((uint32_t)code << 1) | bit);
        if (code <= t->max_code[len]) {
            const int64_t idx = (int64_t)code + t->val_offset[len];
            if (idx < 0 || idx >= (int64_t)t->nvalues) return -1;
            *sym = t->values[idx];
            return 0;
        }
    }
    return -1;
}

/* read_amplitude, jpeg.rs:674-686, in i32 with wrapping */
static int read_amplitude(Reader *r, uint8_t size, int32_t *out)
{
    if (size == 0) {
        *out = 0;
        return 0;
    }
    uint32_t bits;
    if (read_bits(r, size, &bits)) return -1;
    const uint32_t thr = 1u << ((uint32_t)(uint8_t)(size - 1) & 31u);
    *out = (int32_t)bits < (int32_t)thr ? (int32_t)(bits - (2u * thr - 1u)) : (int32_t)bits;
    return 0;
}

/* find_entropy_end, jpeg.rs:653-671 */
size_t jd_find_entropy_end(const uint8_t *d, size_t n)
{
    if (n < 2) return n;
    size_t i = 0;
    while (i < n - 1) {
        if (d[i] == 0xFF && d[i + 1] != 0x00 && d[i + 1] != 0xFF) {
            if (d[i + 1] >= 0xD0 && d[i + 1] <= 0xD7) {
                i += 2;
                continue;
            }
            return i;
        }
        i++;
    }
    return n;
}

/* ---- idct.rs ---- */
static const int UNZIGZAG[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

static int32_t fix_mul(int32_t a, int32_t b) { return (int32_t)(uint32_t)(uint64_t)(((int64_t)a * b) >> 13); }
#define ADD(a, b) ((int32_t)((uint32_t)(a) + (uint32_t)(b)))
#define SUB(a, b) ((int32_t)((uint32_t)(a) - (uint32_t)(b)))
#define SHL13(a) ((int32_t)((uint32_t)(a) << 13))

/* one 1-D pass of idct_2d_integer (:49-113 and :118-192 are the same butterfly): out[0..7] before descale */
static void idct_1d(const int32_t d[8], int32_t o[8])
{
    const int32_t t0 = SHL13(d[0]), t1 = SHL13(d[2]), t2 = SHL13(d[4]), t3 = SHL13(d[6]);
    const int32_t tmp10 = ADD(t0, t2), tmp11 = SUB(t0, t2);
    const int32_t z1 = fix_mul(ADD(t1, t3), 4433);
    const int32_t tmp12 = SUB(z1, fix_mul(t3, 15137)), tmp13 = ADD(z1, fix_mul(t1, 6270));
    const int32_t e0 = ADD(tmp10, tmp13), e3 = SUB(tmp10, tmp13), e1 = ADD(tmp11, tmp12), e2 = SUB(tmp11, tmp12);
    const int32_t z5 = fix_mul(ADD(d[1], d[5]), 9633);
    int32_t o10 = fix_mul(d[1], 2446), o11 = fix_mul(d[3], 16819), o12 = fix_mul(d[5], 25172), o13 = fix_mul(d[7], 12299);
    const int32_t y1 = fix_mul(ADD(d[1], d[7]), -7373), y2 = fix_mul(ADD(d[3], d[5]), -20995);
    const int32_t y3 = ADD(fix_mul(ADD(d[5], d[7]), -16069), z5), y4 = ADD(fix_mul(ADD(d[1], d[3]), -3196), z5);
    o10 = ADD(ADD(o10, y1), y3);
    o11 = ADD(ADD(o11, y2), y4);
    o12 = ADD(ADD(o12, y2), y3);
    o13 = ADD(ADD(o13, y1), y4);
    o[0] = ADD(e0, o13); o[7] = SUB(e0, o13);
    o[1] = ADD(e1, o12); o[6] = SUB(e1, o12);
    o[2] = ADD(e2, o11); o[5] = SUB(e2, o11);
    o[3] = ADD(e3, o10); o[4] = SUB(e3, o10);
}

/* dequantize (:214-230) + idct_2d_integer (:45-204) */
void jd_idct_block(const int16_t coef[64], const uint16_t q[64], uint8_t out[64])
{
    int32_t nat[64], ws[64], c[8], o[8];
    for (int i = 0; i < 64; ++i) nat[UNZIGZAG[i]] = (int32_t)coef[i] * (int32_t)q[i];
    for (int col = 0; col < 8; ++col) {
        for (int k = 0; k < 8; ++k) c[k] = nat[col + 8 * k];
        idct_1d(c, o);
        for (int k = 0; k < 8; ++k) ws[col + 8 * k] = ADD(o[k], 1 << 10) >> 11;
    }
    for (int row = 0; row < 8; ++row) {
        idct_1d(ws + 8 * row, o);
        for (int k = 0; k < 8; ++k) {
            int32_t v = ADD(ADD(o[k], 1 << 17) >> 18, 128);
            out[8 * row + k] = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
        }
    }
}

/* ---- markers and segments, jpeg.rs:214-484 ---- */
/* read_marker, :253-292: *seg points into the data */
static int read_marker(Dec *d, uint8_t *marker, const uint8_t **seg, size_t *seglen)
{
    while (d->pos < d->len && d->data[d->pos] != 0xFF) d->pos++;
    while (d->pos < d->len && d->data[d->pos] == 0xFF) d->pos++;
    if (d->pos >= d->len) return fail(d, INVALID, "unexpected end of file");
    const uint8_t m = d->data[d->pos++];
    *marker = m;
    *seg = NULL;
    *seglen = 0;
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7)) return OK;
    if (d->pos + 2 > d->len) return fail(d, INVALID, "truncated marker");
    const size_t length = ((size_t)d->data[d->pos] << 8) | d->data[d->pos + 1];
    d->pos += 2;
    if (length < 2 || d->pos + length - 2 > d->len) return fail(d, INVALID, "invalid marker length");
    *seg = d->data + d->pos;
    *seglen = length - 2;
    d->pos += length - 2;
    return OK;
}

static int parse_sof0(Dec *d, const uint8_t *s, size_t n)   /* :294-357 */
{
    char m[256];
    if (n < 8) return fail(d, INVALID, "invalid SOF0 length");
    if (s[0] != 8) {
        snprintf(m, sizeof m, "%u-bit precision not supported", s[0]);
        return fail(d, UNSUPPORTED, m);
    }
    d->height = ((uint32_t)s[1] << 8) | s[2];
    d->width = ((uint32_t)s[3] << 8) | s[4];
    const uint32_t nc = s[5];
    if (nc != 1 && nc != 3) {
        snprintf(m, sizeof m, "%u components not supported", nc);
        return fail(d, UNSUPPORTED, m);
    }
    if (n < 6 + nc * 3) return fail(d, INVALID, "truncated SOF0 components");
    d->ncomp = 0;
    for (uint32_t i = 0; i < nc; ++i) {
        const uint8_t *c = s + 6 + i * 3;
        const uint8_t h = c[1] >> 4, v = c[1] & 15;
        if (h == 0 || v == 0) {
            snprintf(m, sizeof m, "invalid sampling factors %ux%u for component %u", h, v, c[0]);
            return fail(d, INVALID, m);
        }
        if (c[2] > 3) {
            snprintf(m, sizeof m, "invalid quantization table ID %u for component %u", c[2], c[0]);
            return fail(d, INVALID, m);
        }
        if (h > d->max_h) d->max_h = h;
        if (v > d->max_v) d->max_v = v;
        d->comp[i] = (Comp){c[0], h, v, c[2], 0, 0};
        d->ncomp = i + 1;
    }
    return OK;
}

static int parse_dht(Dec *d, const uint8_t *s, size_t n)   /* :359-396 */
{
    size_t off = 0;
    while (off < n) {
        const uint8_t info = s[off];
        const uint32_t cls = info >> 4, id = info & 15;
        if (id > 3) return fail(d, INVALID, "invalid Huffman table ID");
        off++;
        if (off + 16 > n) return fail(d, INVALID, "truncated DHT");
        const uint8_t *bits = s + off;
        off += 16;
        uint32_t nv = 0;
        for (int i = 0; i < 16; ++i) nv += bits[i];
        if (off + nv > n) return fail(d, INVALID, "truncated DHT values");
        huff_build(cls == 0 ? &d->dc[id] : &d->ac[id], bits, s + off, nv);
        off += nv;
    }
    return OK;
}

static int parse_dqt(Dec *d, const uint8_t *s, size_t n)   /* :398-434 */
{
    size_t off = 0;
    while (off < n) {
        const uint8_t info = s[off];
        const uint32_t prec = info >> 4, id = info & 15;
        if (id > 3) return fail(d, INVALID, "invalid quantization table ID");
        off++;
        if (prec == 0) {
            if (off + 64 > n) return fail(d, INVALID, "truncated DQT");
            for (int i = 0; i < 64; ++i) d->quant[id][i] = s[off + i];
            off += 64;
        } else {
            if (off + 128 > n) return fail(d, INVALID, "truncated DQT");
            for (int i = 0; i < 64; ++i) d->quant[id][i] = (uint16_t)((s[off + 2 * i] << 8) | s[off + 2 * i + 1]);
            off += 128;
        }
    }
    return OK;
}

static int parse_sos(Dec *d, const uint8_t *s, size_t n)   /* :446-484 */
{
    char m[256];
    if (n == 0) return fail(d, INVALID, "empty SOS segment");
    if (s[0] != d->ncomp) return fail(d, INVALID, "SOS component count mismatch");
    for (uint32_t i = 0; i < d->ncomp; ++i) {
        const size_t off = 1 + i * 2;
        if (off + 1 >= n) return fail(d, INVALID, "truncated SOS segment");
        const uint8_t id = s[off], dc = s[off + 1] >> 4, ac = s[off + 1] & 15;
        if (dc > 3) {
            snprintf(m, sizeof m, "invalid DC Huffman table ID %u for component %u", dc, id);
            return fail(d, INVALID, m);
        }
        if (ac > 3) {
            snprintf(m, sizeof m, "invalid AC Huffman table ID %u for component %u", ac, id);
            return fail(d, INVALID, m);
        }
        d->comp[i].dc = dc;
        d->comp[i].ac = ac;
    }
    return OK;
}

/* decode_scan, jpeg.rs:486-612: the MCU loop.  coefs: decode order; returns the blocks stored */
static uint64_t decode_scan(Dec *d, int16_t *coefs)
{
    const uint64_t mw = (d->width + d->max_h * 8u - 1) / (d->max_h * 8u);
    const uint64_t mh = (d->height + d->max_v * 8u - 1) / (d->max_v * 8u);
    const size_t n = jd_find_entropy_end(d->data + d->pos, d->len - d->pos);
    Reader r = {d->data + d->pos, n, 0, 0, 0};
    int32_t pred[3] = {0, 0, 0};
    uint32_t mcu_count = 0;
    uint64_t stored = 0;
    for (uint64_t my = 0; my < mh; ++my)
        for (uint64_t mx = 0; mx < mw; ++mx) {
            if (d->restart_interval > 0 && mcu_count > 0 && mcu_count % d->restart_interval == 0)
                pred[0] = pred[1] = pred[2] = 0;
            for (uint32_t ci = 0; ci < d->ncomp; ++ci) {
                const Comp *c = &d->comp[ci];
                for (int b = 0; b < c->h * c->v; ++b) {
                    int16_t k64[64];
                    memset(k64, 0, sizeof k64);
                    uint8_t cat;
                    int32_t diff = 0;
                    if (huff_decode(&d->dc[c->dc], &r, &cat)) return stored;
                    if (cat > 0 && read_amplitude(&r, cat, &diff)) return stored;
                    pred[ci] = ADD(pred[ci], diff);
                    k64[0] = (int16_t)pred[ci];
                    uint32_t k = 1;
                    while (k < 64) {
                        uint8_t sym;
                        if (huff_decode(&d->ac[c->ac], &r, &sym)) return stored;
                        if (sym == 0) break;
                        if (sym == 0xF0) {
                            k += 16;
                            continue;
                        }
                        k += sym >> 4;
                        if (k >= 64) break;
                        if (sym & 15) {
                            int32_t a;
                            if (read_amplitude(&r, sym & 15, &a)) return stored;
                            k64[k] = (int16_t)a;
                        }
                        k++;
                    }
                    if (coefs) memcpy(coefs + 64 * stored, k64, sizeof k64);
                    stored++;
                }
            }
            mcu_count++;
        }
    return stored;
}

static void free_tables(Dec *d)
{
    for (int i = 0; i < 4; ++i) {
        free(d->dc[i].values);
        free(d->ac[i].values);
    }
}

/* decode, jpeg.rs:214-251 */
static int parse(Dec *d)
{
    if (d->len < 2 || d->data[0] != 0xFF || d->data[1] != 0xD8) return fail(d, INVALID, "not a JPEG file");
    d->pos = 2;
    for (;;) {
        uint8_t m;
        const uint8_t *s;
        size_t n;
        int rc = read_marker(d, &m, &s, &n);
        if (rc) return rc;
        switch (m) {
        case 0xC0: rc = parse_sof0(d, s, n); break;
        case 0xC2: return fail(d, UNSUPPORTED, "progressive JPEG not supported");
        case 0xC4: rc = parse_dht(d, s, n); break;
        case 0xDB: rc = parse_dqt(d, s, n); break;
        case 0xDD:   /* parse_dri, :436-444 */
            if (n != 2) return fail(d, INVALID, "invalid DRI length");
            d->restart_interval = (uint16_t)((s[0] << 8) | s[1]);
            break;
        case 0xDA:
            rc = parse_sos(d, s, n);
            if (rc) return rc;
            if (d->ncomp == 0) return fail(d, PANIC, "SOS with no frame components");   /* pixo panics */
            return OK;
        case 0xD9: return fail(d, INVALID, "no image data found");
        default: break;
        }
        if (rc) return rc;
    }
}

void jd_decode(const uint8_t *data, size_t len, uint8_t *pixels, int16_t *coefs, uint64_t info[8], char *msg)
{
    Dec d;
    memset(&d, 0, sizeof d);
    d.data = data;
    d.len = len;
    d.max_h = d.max_v = 1;
    d.msg = msg;
    msg[0] = 0;
    for (int i = 0; i < 4; ++i) {
        huff_default(&d.dc[i]);
        huff_default(&d.ac[i]);
    }
    memset(info, 0, 8 * sizeof(uint64_t));
    const int st = parse(&d);
    info[0] = (uint64_t)st;
    if (st != OK) {
        free_tables(&d);
        return;
    }
    const uint64_t mw = (d.width + d.max_h * 8u - 1) / (d.max_h * 8u);
    const uint64_t mh = (d.height + d.max_v * 8u - 1) / (d.max_v * 8u);
    uint64_t bpm = 0, pw[3], plen[3];
    for (uint32_t c = 0; c < d.ncomp; ++c) {
        bpm += (uint64_t)d.comp[c].h * d.comp[c].v;
        pw[c] = mw * d.comp[c].h * 8;
        plen[c] = pw[c] * mh * d.comp[c].v * 8;
    }
    info[1] = d.width;
    info[2] = d.height;
    info[3] = d.ncomp == 1 ? 0 : 2;
    info[4] = d.ncomp;
    info[5] = mw * mh * bpm;
    info[7] = (uint64_t)d.width * d.height * (d.ncomp == 1 ? 1 : 3);
    if (!pixels && !coefs) {
        free_tables(&d);
        return;
    }
    int16_t *k = (int16_t *)malloc(64 * 2 * (info[5] ? info[5] : 1));
    const uint64_t stored = decode_scan(&d, k);
    info[6] = stored;
    if (coefs) memcpy(coefs, k, 128 * stored);
    if (pixels) {
        /* the component planes: every stored block through dequantize + IDCT, the rest 0 (:587-606) */
        uint8_t *pl[3] = {0, 0, 0};
        for (uint32_t c = 0; c < d.ncomp; ++c) pl[c] = (uint8_t *)calloc(plen[c] ? plen[c] : 1, 1);
        uint64_t i = 0;
        for (uint64_t my = 0; my < mh && i < stored; ++my)
            for (uint64_t mx = 0; mx < mw && i < stored; ++mx)
                for (uint32_t c = 0; c < d.ncomp && i < stored; ++c)
                    for (uint32_t by = 0; by < d.comp[c].v && i < stored; ++by)
                        for (uint32_t bx = 0; bx < d.comp[c].h && i < stored; ++bx, ++i) {
                            uint8_t px[64];
                            jd_idct_block(k + 64 * i, d.quant[d.comp[c].q], px);
                            const uint64_t x0 = (mx * d.comp[c].h + bx) * 8, y0 = (my * d.comp[c].v + by) * 8;
                            for (int r = 0; r < 8; ++r) memcpy(pl[c] + (y0 + r) * pw[c] + x0, px + 8 * r, 8);
                        }
        const uint64_t W = d.width, H = d.height;
        if (d.ncomp == 1) {   /* crop, :615-631: get(idx).unwrap_or(0), for a plane sized by an earlier SOF0's maxima */
            for (uint64_t y = 0; y < H; ++y)
                for (uint64_t x = 0; x < W; ++x) {
                    const uint64_t i = y * pw[0] + x;
                    pixels[y * W + x] = i < plen[0] ? pl[0][i] : 0;
                }
        } else {              /* ycbcr_to_rgb, :689-735 */
            const uint64_t yw = mw * d.max_h * 8;
            const uint32_t hb = d.max_h / d.comp[1].h, vb = d.max_v / d.comp[1].v;
            const uint32_t hr = d.max_h / d.comp[2].h, vr = d.max_v / d.comp[2].v;
            uint8_t *o = pixels;
            for (uint64_t y = 0; y < H; ++y)
                for (uint64_t x = 0; x < W; ++x) {
                    const uint64_t yi = y * yw + x, bi = (y / vb) * pw[1] + x / hb, ri = (y / vr) * pw[2] + x / hr;
                    const int32_t Y = yi < plen[0] ? pl[0][yi] : 0;
                    const int32_t cb = (bi < plen[1] ? pl[1][bi] : 128) - 128;
                    const int32_t cr = (ri < plen[2] ? pl[2][ri] : 128) - 128;
                    const int32_t rr = Y + ((cr * 359) >> 8), gg = Y - ((cb * 88 + cr * 183) >> 8),
                                  bb = Y + ((cb * 454) >> 8);
                    *o++ = (uint8_t)(rr < 0 ? 0 : rr > 255 ? 255 : rr);
                    *o++ = (uint8_t)(gg < 0 ? 0 : gg > 255 ? 255 : gg);
                    *o++ = (uint8_t)(bb < 0 ? 0 : bb > 255 ? 255 : bb);
                }
        }
        for (uint32_t c = 0; c < d.ncomp; ++c) free(pl[c]);
    }
    free(k);
    free_tables(&d);
}
