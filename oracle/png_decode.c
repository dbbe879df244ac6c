/* png_decode.c — CPU restatement of pixo's PNG decoder, pixo::decode::decode_png (src/decode/png.rs:101-626),
 * its inflate (src/decode/inflate.rs:46-513) and its LSB bit reader (src/decode/bit_reader.rs:10-135).  Test
 * infrastructure only: it follows pixo's structure step by step (a byte-at-a-time bit buffer, the 9-bit lookup
 * filled in symbol order, decode_slow comparing canonical codes symbol by symbol), so that the kernels, which do
 * the same work another way, are checked against pixo's own steps.
 *
 * pd_decode(data, len, pixels, info, msg): info[0] kind (0 Ok, 1 InvalidDecode, 2 UnsupportedDecode,
 *   3 InvalidDimensions, 4 ImageTooLarge), [1] width, [2] height, [3] pixo_b200 colour type, [4] frame bytes;
 *   msg: pixo's Display text.  pixels may be NULL (geometry and error only).
 * pd_inflate_zlib(data, len, expected, out, cap, info, msg): inflate_zlib_with_size; info[0] kind, [1] bytes
 *   produced (copied to out up to cap).
 */
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

enum { OK = 0, INVALID = 1, UNSUPPORTED = 2, DIMENSIONS = 3, TOO_LARGE = 4 };

typedef struct {
    int kind;
    char *msg;
} Err;

static int err(Err *e, int kind, const char *fmt, ...)
{
    char tmp[200];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(tmp, sizeof tmp, fmt, ap);
    va_end(ap);
    e->kind = kind;
    if (kind == INVALID) snprintf(e->msg, 256, "Decode error: %s", tmp);
    else if (kind == UNSUPPORTED) snprintf(e->msg, 256, "Unsupported: %s", tmp);
    else snprintf(e->msg, 256, "%s", tmp);
    return kind;
}

/* ---- output vector ---- */
typedef struct {
    uint8_t *p;
    size_t n, cap;
} Vec;

static void push(Vec *v, uint8_t b)
{
    if (v->n == v->cap) {
        v->cap = v->cap ? v->cap * 2 : 4096;
        v->p = realloc(v->p, v->cap);
    }
    v->p[v->n++] = b;
}

/* ---- BitReader ---- */
typedef struct {
    const uint8_t *data;
    size_t len, pos;
    uint64_t buf;
    unsigned bits;
} BR;

static int ensure(BR *r, unsigned n, Err *e)
{
    while (r->bits < n) {
        if (r->pos >= r->len) return err(e, INVALID, "unexpected end of stream");
        r->buf |= (uint64_t)r->data[r->pos++] << r->bits;
        r->bits += 8;
    }
    return OK;
}

static int read_bits(BR *r, unsigned n, uint32_t *v, Err *e)
{
    if (ensure(r, n, e)) return e->kind;
    *v = (uint32_t)(r->buf & ((1ull << n) - 1));
    r->buf >>= n;
    r->bits -= n;
    return OK;
}

static unsigned try_peek(BR *r, unsigned n, uint32_t *v)
{
    while (r->bits < n && r->pos < r->len) {
        r->buf |= (uint64_t)r->data[r->pos++] << r->bits;
        r->bits += 8;
    }
    unsigned a = r->bits < n ? r->bits : n;
    *v = (uint32_t)(r->buf & ((1ull << a) - 1));
    return a;
}

/* ---- HuffmanTable ---- */
typedef struct {
    uint16_t lookup[512];
    uint8_t lengths[320];
    uint32_t codes[320];   /* code_for_symbol of every symbol, computed once */
    unsigned n, max_len;
} Huff;

static void from_lengths(Huff *t, const uint8_t *lengths, unsigned n)
{
    memset(t, 0, sizeof *t);
    memcpy(t->lengths, lengths, n);
    t->n = n;
    for (unsigned i = 0; i < n; i++)
        if (lengths[i] > t->max_len) t->max_len = lengths[i];
    if (!t->max_len) return;
    unsigned bl[16] = {0}, next[16] = {0}, code = 0;
    for (unsigned i = 0; i < n; i++)
        if (lengths[i]) bl[lengths[i]]++;
    for (unsigned b = 1; b <= 15; b++) {
        code = (code + bl[b - 1]) << 1;
        next[b] = code;
    }
    uint32_t *codes = t->codes;
    for (unsigned s = 0; s < n; s++) codes[s] = lengths[s] ? next[lengths[s]]++ : 0xFFFFFFFFu;
    for (unsigned s = 0; s < n; s++) {
        unsigned len = lengths[s];
        if (!len || len > 9) continue;
        uint16_t c = (uint16_t)codes[s], rev = 0;
        for (unsigned k = 0; k < len; k++) {
            rev = (uint16_t)((rev << 1) | (c & 1));
            c >>= 1;
        }
        for (unsigned i = 0; i < (1u << (9 - len)); i++) t->lookup[rev | (i << len)] = (uint16_t)(s | (len << 12));
    }
}

static int decode_slow(const Huff *t, BR *r, uint32_t *sym, Err *e)
{
    uint32_t code = 0;
    for (unsigned len = 1; len <= t->max_len; len++) {
        uint32_t bit;
        if (read_bits(r, 1, &bit, e)) return e->kind;
        code = (code << 1) | bit;
        for (unsigned s = 0; s < t->n; s++)
            if (t->lengths[s] == len && t->codes[s] == code) {
                *sym = s;
                return OK;
            }
    }
    return err(e, INVALID, "invalid Huffman code");
}

static int huff_decode(const Huff *t, BR *r, uint32_t *sym, Err *e)
{
    if (!t->max_len) return err(e, INVALID, "empty Huffman table");
    uint32_t peek;
    unsigned avail = try_peek(r, 9, &peek);
    if (avail >= 9) {
        uint16_t en = t->lookup[peek];
        unsigned len = en >> 12;
        if (len > 0 && len <= 9) {
            r->buf >>= len;
            r->bits -= len;
            *sym = en & 0xFFF;
            return OK;
        }
        return decode_slow(t, r, sym, e);
    }
    if (avail > 0) {
        uint16_t en = t->lookup[peek];
        unsigned len = en >> 12;
        if (len > 0 && len <= avail) {
            r->buf >>= len;
            r->bits -= len;
            *sym = en & 0xFFF;
            return OK;
        }
    }
    return decode_slow(t, r, sym, e);
}

/* ---- inflate ---- */
static const uint16_t LEN_BASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83,
                                      99, 115, 131, 163, 195, 227, 258};
static const uint8_t LEN_EXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t DIST_BASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                       1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t DIST_EXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
                                       12, 12, 13, 13};
static const uint8_t CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

static int inflate_block(BR *r, Vec *out, const Huff *lit, const Huff *dist, Err *e)
{
    for (;;) {
        uint32_t sym;
        if (huff_decode(lit, r, &sym, e)) return e->kind;
        if (sym < 256) {
            push(out, (uint8_t)sym);
        } else if (sym == 256) {
            return OK;
        } else if (sym <= 285) {
            uint32_t extra, ds;
            unsigned li = sym - 257;
            if (read_bits(r, LEN_EXTRA[li], &extra, e)) return e->kind;
            size_t length = LEN_BASE[li] + extra;
            if (huff_decode(dist, r, &ds, e)) return e->kind;
            if (ds >= 30) return err(e, INVALID, "invalid distance code");
            if (read_bits(r, DIST_EXTRA[ds], &extra, e)) return e->kind;
            size_t distance = DIST_BASE[ds] + extra;
            if (distance > out->n) return err(e, INVALID, "distance too far back");
            size_t start = out->n - distance;
            for (size_t i = 0; i < length; i++) push(out, out->p[start + i % distance]);
        } else {
            return err(e, INVALID, "invalid literal/length code: %u", sym);
        }
    }
}

static int inflate_raw(const uint8_t *data, size_t len, Vec *out, Err *e)
{
    BR r = {data, len, 0, 0, 0};
    static Huff lit, dist, cl;   /* large: kept off the stack (single-threaded test oracle) */
    for (;;) {
        uint32_t bfinal, btype;
        if (read_bits(&r, 1, &bfinal, e) || read_bits(&r, 2, &btype, e)) return e->kind;
        if (btype == 0) {
            unsigned discard = r.bits % 8;
            r.buf >>= discard;
            r.bits -= discard;
            uint32_t l, nl;
            if (read_bits(&r, 16, &l, e) || read_bits(&r, 16, &nl, e)) return e->kind;
            if ((uint16_t)l != (uint16_t)~nl) return err(e, INVALID, "stored block LEN/NLEN mismatch");
            unsigned from_buf = r.bits / 8 < l ? r.bits / 8 : l;
            uint8_t tmp[65535];
            for (unsigned i = 0; i < from_buf; i++) {
                tmp[i] = (uint8_t)r.buf;
                r.buf >>= 8;
                r.bits -= 8;
            }
            size_t rest = l - from_buf;
            if (r.pos + rest > r.len) return err(e, INVALID, "unexpected end of stream");
            memcpy(tmp + from_buf, r.data + r.pos, rest);
            r.pos += rest;
            for (unsigned i = 0; i < l; i++) push(out, tmp[i]);
        } else if (btype == 1) {
            uint8_t L[288], D[32];
            for (int i = 0; i < 288; i++) L[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
            for (int i = 0; i < 32; i++) D[i] = 5;
            from_lengths(&lit, L, 288);
            from_lengths(&dist, D, 32);
            if (inflate_block(&r, out, &lit, &dist, e)) return e->kind;
        } else if (btype == 2) {
            uint32_t hlit, hdist, hclen, v;
            if (read_bits(&r, 5, &hlit, e) || read_bits(&r, 5, &hdist, e) || read_bits(&r, 4, &hclen, e))
                return e->kind;
            hlit += 257;
            hdist += 1;
            hclen += 4;
            uint8_t cll[19] = {0};
            for (unsigned i = 0; i < hclen; i++) {
                if (read_bits(&r, 3, &v, e)) return e->kind;
                cll[CL_ORDER[i]] = (uint8_t)v;
            }
            from_lengths(&cl, cll, 19);
            uint8_t lengths[320] = {0};
            unsigned n = hlit + hdist, i = 0;
            while (i < n) {
                uint32_t sym;
                if (huff_decode(&cl, &r, &sym, e)) return e->kind;
                if (sym <= 15) {
                    lengths[i++] = (uint8_t)sym;
                } else if (sym == 16) {
                    if (i == 0) return err(e, INVALID, "repeat code at start");
                    uint32_t rep;
                    if (read_bits(&r, 2, &rep, e)) return e->kind;
                    uint8_t prev = lengths[i - 1];
                    for (unsigned k = 0; k < rep + 3; k++) {
                        if (i >= n) return err(e, INVALID, "too many code lengths");
                        lengths[i++] = prev;
                    }
                } else if (sym == 17 || sym == 18) {
                    uint32_t rep;
                    if (read_bits(&r, sym == 17 ? 3 : 7, &rep, e)) return e->kind;
                    rep += sym == 17 ? 3 : 11;
                    for (unsigned k = 0; k < rep; k++) {
                        if (i >= n) return err(e, INVALID, "too many code lengths");
                        lengths[i++] = 0;
                    }
                } else {
                    return err(e, INVALID, "invalid code length code");
                }
            }
            from_lengths(&lit, lengths, hlit);
            from_lengths(&dist, lengths + hlit, hdist);
            if (inflate_block(&r, out, &lit, &dist, e)) return e->kind;
        } else {
            return err(e, INVALID, "reserved block type");
        }
        if (bfinal) return OK;
    }
}

static uint32_t adler32(const uint8_t *p, size_t n)
{
    uint32_t a = 1, b = 0;
    for (size_t i = 0; i < n; i++) {
        a = (a + p[i]) % 65521;
        b = (b + a) % 65521;
    }
    return b << 16 | a;
}

static int inflate_zlib(const uint8_t *data, size_t len, uint64_t expected, Vec *out, Err *e)
{
    if (len < 6) return err(e, INVALID, "zlib stream too short");
    if ((data[0] & 0x0F) != 8) return err(e, INVALID, "invalid zlib compression method");
    if ((((unsigned)data[0] << 8) | data[1]) % 31 != 0) return err(e, INVALID, "invalid zlib header checksum");
    if (data[1] & 0x20) return err(e, UNSUPPORTED, "preset dictionary not supported");
    if (inflate_raw(data + 2, len - 6, out, e)) return e->kind;
    const uint8_t *s = data + len - 4;
    uint32_t stored = (uint32_t)s[0] << 24 | (uint32_t)s[1] << 16 | (uint32_t)s[2] << 8 | s[3];
    uint32_t computed = adler32(out->p, out->n);
    if (stored != computed) return err(e, INVALID, "Adler32 mismatch: expected %08X, got %08X", stored, computed);
    if (out->n != expected)
        return err(e, INVALID, "decompressed size mismatch: expected %llu, got %llu", (unsigned long long)expected,
                   (unsigned long long)out->n);
    return OK;
}

/* ---- decode_png ---- */
static uint32_t crc_table[256];

static uint32_t crc32(const uint8_t *a, size_t na, const uint8_t *b, size_t nb)
{
    if (!crc_table[1])
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int k = 0; k < 8; k++) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            crc_table[i] = c;
        }
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < na; i++) c = crc_table[(c ^ a[i]) & 0xFF] ^ (c >> 8);
    for (size_t i = 0; i < nb; i++) c = crc_table[(c ^ b[i]) & 0xFF] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

static uint32_t be32(const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

/* String::from_utf8_lossy of 4 bytes */
static void lossy(const uint8_t *s, char *out)
{
    size_t i = 0, o = 0;
    while (i < 4) {
        uint8_t b = s[i];
        if (b < 0x80) { out[o++] = (char)b; i++; continue; }
        unsigned need = 0;
        uint8_t lo = 0x80, hi = 0xBF;
        if (b >= 0xC2 && b <= 0xDF) need = 1;
        else if (b >= 0xE0 && b <= 0xEF) { need = 2; if (b == 0xE0) lo = 0xA0; if (b == 0xED) hi = 0x9F; }
        else if (b >= 0xF0 && b <= 0xF4) { need = 3; if (b == 0xF0) lo = 0x90; if (b == 0xF4) hi = 0x8F; }
        unsigned k = 1;
        int good = need > 0;
        while (good && k <= need) {
            if (i + k >= 4) { good = 0; break; }
            uint8_t c = s[i + k];
            uint8_t l = k == 1 ? lo : 0x80, h = k == 1 ? hi : 0xBF;
            if (c < l || c > h) { good = 0; break; }
            k++;
        }
        if (good) { memcpy(out + o, s + i, need + 1); o += need + 1; i += need + 1; }
        else { memcpy(out + o, "\xEF\xBF\xBD", 3); o += 3; i += need ? k : 1; }
    }
    out[o] = 0;
}

static const char *ct_name(uint8_t c)
{
    return c == 0 ? "Grayscale" : c == 2 ? "Rgb" : c == 3 ? "Indexed" : c == 4 ? "GrayscaleAlpha" : "Rgba";
}

static int paeth(int a, int b, int c)
{
    int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return pa <= pb && pa <= pc ? a : pb <= pc ? b : c;
}

static int decode(const uint8_t *data, size_t len, uint8_t *pixels, uint64_t *info, Err *e)
{
    static const uint8_t SIG[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    if (len < 8 || memcmp(data, SIG, 8)) return err(e, INVALID, "not a PNG file");
    size_t pos = 8;
    int have_ihdr = 0, seen_iend = 0;
    uint32_t w = 0, h = 0;
    uint8_t depth = 0, ct = 0, comp = 0, filt = 0, inter = 0;
    const uint8_t *plte = NULL, *trns = NULL;
    size_t plte_len = 0, trns_len = 0;
    Vec idat = {0}, out = {0};
    int rc = OK;
    while (pos + 12 <= len) {
        size_t length = be32(data + pos);
        const uint8_t *type = data + pos + 4;
        size_t ds = pos + 8, de = ds + length;
        if (de + 4 > len) { rc = err(e, INVALID, "truncated PNG chunk"); goto done; }
        if (be32(data + de) != crc32(type, 4, data + ds, length)) {
            char name[16];
            lossy(type, name);
            rc = err(e, INVALID, "CRC mismatch in %s chunk", name);
            goto done;
        }
        if (!memcmp(type, "IHDR", 4)) {
            if (length != 13) { rc = err(e, INVALID, "invalid IHDR length"); goto done; }
            const uint8_t *d = data + ds;
            if (d[9] != 0 && d[9] != 2 && d[9] != 3 && d[9] != 4 && d[9] != 6) {
                rc = err(e, INVALID, "invalid PNG color type: %u", d[9]);
                goto done;
            }
            have_ihdr = 1;
            w = be32(d); h = be32(d + 4); depth = d[8]; ct = d[9]; comp = d[10]; filt = d[11]; inter = d[12];
        } else if (!memcmp(type, "PLTE", 4)) {
            if (length % 3) { rc = err(e, INVALID, "invalid PLTE length"); goto done; }
            plte = data + ds; plte_len = length / 3;
        } else if (!memcmp(type, "tRNS", 4)) {
            trns = data + ds; trns_len = length;
        } else if (!memcmp(type, "IDAT", 4)) {
            for (size_t i = 0; i < length; i++) push(&idat, data[ds + i]);
        } else if (!memcmp(type, "IEND", 4)) {
            seen_iend = 1;
            break;
        }
        pos = de + 4;
    }
    if (!seen_iend) { rc = err(e, INVALID, "missing IEND chunk"); goto done; }
    if (!have_ihdr) { rc = err(e, INVALID, "missing IHDR chunk"); goto done; }
    if (!w || !h) { rc = err(e, DIMENSIONS, "Invalid image dimensions: %ux%u", w, h); goto done; }
    if (w > (1u << 24) || h > (1u << 24)) {
        rc = err(e, TOO_LARGE, "Image %ux%u exceeds maximum dimension %u", w, h, 1u << 24);
        goto done;
    }
    if (comp) { rc = err(e, INVALID, "unsupported compression method"); goto done; }
    if (filt) { rc = err(e, INVALID, "unsupported filter method"); goto done; }
    if (inter) { rc = err(e, UNSUPPORTED, "Adam7 interlaced images not supported"); goto done; }
    int valid = ct == 0 ? (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)
              : ct == 3 ? (depth == 1 || depth == 2 || depth == 4 || depth == 8) : (depth == 8 || depth == 16);
    if (!valid) { rc = err(e, INVALID, "invalid bit depth %u for color type %s", depth, ct_name(ct)); goto done; }
    if (!idat.n) { rc = err(e, INVALID, "no IDAT data"); goto done; }
    size_t W = w, H = h, bd = depth, sb, bpp;
    switch (ct) {
    case 0: sb = (W * bd + 7) / 8; bpp = (bd + 7) / 8; break;
    case 2: bpp = 3 * bd / 8; sb = W * bpp; break;
    case 3: sb = (W * bd + 7) / 8; bpp = 1; break;
    case 4: bpp = 2 * bd / 8; sb = W * bpp; break;
    default: bpp = 4 * bd / 8; sb = W * bpp; break;
    }
    uint64_t expected = (uint64_t)H * (1 + sb);
    if (inflate_zlib(idat.p, idat.n, expected, &out, e)) { rc = e->kind; goto done; }
    /* reconstruct_image: unfilter every row, in place */
    for (size_t y = 0; y < H; y++) {
        uint8_t *row = out.p + y * (1 + sb) + 1, *prev = y ? out.p + (y - 1) * (1 + sb) + 1 : NULL;
        uint8_t f = row[-1];
        if (f > 4) { rc = err(e, INVALID, "invalid filter type: %u", f); goto done; }
        for (size_t i = 0; i < sb; i++) {
            int a = i >= bpp ? row[i - bpp] : 0, b = prev ? prev[i] : 0, c = prev && i >= bpp ? prev[i - bpp] : 0;
            int p = f == 0 ? 0 : f == 1 ? (i >= bpp ? a : 0) : f == 2 ? b : f == 3 ? (a + b) / 2 : paeth(a, b, c);
            row[i] = (uint8_t)(row[i] + p);
        }
    }
    int alpha = 0;
    for (size_t i = 0; i < trns_len; i++) alpha |= trns[i] != 0xFF;
    unsigned ch, oct;
    switch (ct) {
    case 0: ch = 1; oct = 0; break;
    case 4: ch = 2; oct = 1; break;
    case 2: ch = 3; oct = 2; break;
    case 6: ch = 4; oct = 3; break;
    default:
        if (!plte) { rc = err(e, INVALID, "missing PLTE chunk"); goto done; }
        ch = alpha ? 4 : 3; oct = alpha ? 3 : 2; break;
    }
    info[1] = w; info[2] = h; info[3] = oct; info[4] = (uint64_t)W * H * ch;
    if (pixels) {
        uint8_t *o = pixels;
        for (size_t y = 0; y < H; y++) {
            const uint8_t *row = out.p + y * (1 + sb) + 1;
            for (size_t x = 0; x < W; x++) {
                if (bd == 16) {
                    for (unsigned c = 0; c < ch; c++) *o++ = row[(x * ch + c) * 2];
                    continue;
                }
                unsigned v = bd == 8 ? row[x] : (row[x * bd / 8] >> (8 - bd - (x * bd) % 8)) & ((1u << bd) - 1);
                if (ct == 3) {
                    if (v < plte_len) {
                        *o++ = plte[3 * v]; *o++ = plte[3 * v + 1]; *o++ = plte[3 * v + 2];
                        if (alpha) *o++ = v < trns_len ? trns[v] : 255;
                    } else {
                        *o++ = 0; *o++ = 0; *o++ = 0;
                        if (alpha) *o++ = 255;
                    }
                } else if (ct == 0) {
                    *o++ = (uint8_t)(bd == 1 ? (v ? 255 : 0) : bd == 2 ? v * 0x55 : bd == 4 ? v * 0x11 : v);
                } else {
                    for (unsigned c = 0; c < ch; c++) *o++ = row[x * ch + c];
                }
            }
        }
    }
done:
    free(idat.p);
    free(out.p);
    return rc;
}

void pd_decode(const uint8_t *data, size_t len, uint8_t *pixels, uint64_t *info, char *msg)
{
    Err e = {OK, msg};
    msg[0] = 0;
    memset(info, 0, 8 * sizeof *info);
    info[0] = (uint64_t)decode(data, len, pixels, info, &e);
}

void pd_inflate_zlib(const uint8_t *data, size_t len, uint64_t expected, uint8_t *out, size_t cap, uint64_t *info,
                     char *msg)
{
    Err e = {OK, msg};
    Vec v = {0};
    msg[0] = 0;
    info[0] = (uint64_t)inflate_zlib(data, len, expected, &v, &e);
    info[1] = v.n;
    if (out) memcpy(out, v.p, v.n < cap ? v.n : cap);
    free(v.p);
}

uint32_t pd_crc32(const uint8_t *data, size_t len) { return crc32(data, len, NULL, 0); }
