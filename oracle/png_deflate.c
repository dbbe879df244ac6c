/* Plain-C restatement of pixo's deflate_zlib_packed at levels 1-9 (test infrastructure only; the library never
 * links it).  Every function cites the file:line of pixo @ 437bf63 it follows.
 *
 *   pd_lz77            Lz77Compressor::compress_into_sink        src/compress/lz77.rs:403-591
 *   pd_code_lengths    huffman::build_codes (lengths only)       src/compress/huffman.rs:48-205
 *   pd_high_entropy    is_high_entropy_data                      src/compress/deflate.rs:1108-1145
 *   pd_deflate_zlib    deflate_zlib_packed -> compress_packed_zlib src/compress/deflate.rs:1008-1047,1074-1079
 *
 * Built by oracle/png_deflate.py into oracle/libpng_deflate.so. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MAX_DISTANCE 32768
#define MAX_MATCH 258
#define MIN_MATCH 3
#define GOOD_MATCH 16
#define HASH_SIZE 65536
#define HASH3_SIZE 32768
#define HT_BITS 15
#define HT_SIZE (1 << HT_BITS)
#define LIT_FLAG 0x80000000u

/* config_for_level, lz77.rs:1415-1480 */
typedef struct { int chain, depth, nice, lazy, ht; } Cfg;   /* lazy: 0 None, 1 Lazy, 2 Lazy2 */
static const Cfg CFG[10] = {
    {0, 0, 0, 0, 0},      {4, 4, 32, 0, 1},      {8, 6, 10, 0, 0},        {16, 12, 14, 0, 0},
    {32, 16, 30, 0, 0},   {64, 16, 30, 1, 0},    {128, 35, 65, 1, 0},     {256, 100, 130, 1, 0},
    {1024, 300, 258, 2, 0}, {4096, 600, 258, 2, 0},
};

typedef struct {
    const uint8_t *d;
    size_t n;
    int32_t *head, *head3, *ht, *prev;
} Lz;

/* hash4 / hash3 / hash4_ht, lz77.rs:239-256,320-326 */
static uint32_t rd32(const uint8_t *p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }
static size_t hash4(const Lz *z, size_t p) { return p + 3 >= z->n ? 0 : ((rd32(z->d + p) * 0x1E35A7BDu) >> 16) & (HASH_SIZE - 1); }
static size_t hash3(const Lz *z, size_t p)
{
    if (p + 2 >= z->n) return 0;
    uint32_t v = z->d[p] | z->d[p + 1] << 8 | z->d[p + 2] << 16;
    return ((v * 0x1E35A7BDu) >> 17) & (HASH3_SIZE - 1);
}
static size_t hash4_ht(const Lz *z, size_t p) { return p + 3 >= z->n ? 0 : ((rd32(z->d + p) * 0x1E35A7BDu) >> (32 - HT_BITS)) & (HT_SIZE - 1); }

/* detect_same_byte_run, lz77.rs:272-316 (the 8-byte steps give the same count as a byte loop) */
static size_t same_run(const Lz *z, size_t p)
{
    if (p >= z->n) return 0;
    if (p + 1 >= z->n) return 1;
    size_t max = z->n - p < MAX_MATCH ? z->n - p : MAX_MATCH, len = 1;
    while (len < max && z->d[p + len] == z->d[p]) len++;
    return len;
}

/* match_length, lz77.rs:816-861 */
static size_t match_len(const Lz *z, size_t a, size_t b)
{
    size_t max = z->n - b < MAX_MATCH ? z->n - b : MAX_MATCH, len = 0;
    while (len < max && z->d[a + len] == z->d[b + len]) len++;
    return len;
}

/* update_hash, lz77.rs:864-876 */
static void update_hash(Lz *z, size_t p)
{
    if (p + 3 >= z->n) return;
    z->head3[hash3(z, p)] = (int32_t)p;
    size_t h = hash4(z, p);
    z->prev[p % MAX_DISTANCE] = z->head[h];
    z->head[h] = (int32_t)p;
}

/* find_best_match, lz77.rs:605-749; returns the length (0: none), *dist the distance */
static size_t find_best(const Lz *z, size_t pos, size_t chain, size_t nice, size_t minm, size_t *dist)
{
    if (pos + MIN_MATCH > z->n) return 0;
    const uint8_t *d = z->d;
    size_t run = same_run(z, pos);
    int is_run = run >= minm && pos >= 1 && d[pos - 1] == d[pos];
    if (is_run && (run >= nice || run >= MAX_MATCH)) {
        *dist = 1;
        return run < MAX_MATCH ? run : MAX_MATCH;
    }
    size_t best = minm > 0 ? minm - 1 : 0, bd = 0;
    if (is_run) best = run, bd = 1;
    int32_t c3 = z->head3[hash3(z, pos)];
    if (c3 >= 0) {
        size_t mp = (size_t)c3, dd = pos - mp;
        if (dd != 0 && dd <= MAX_DISTANCE && mp + 3 <= z->n && !memcmp(d + pos, d + mp, 3)) {
            size_t len = match_len(z, mp, pos);
            if (len >= minm && !(len == 3 && dd > 8192) && (len > best || (len == best && dd < bd))) {
                best = len, bd = dd;
                if (best >= nice) { *dist = bd; return best; }
            }
        }
    }
    int32_t cp = z->head[hash4(z, pos)];
    size_t maxd = pos < MAX_DISTANCE ? pos : MAX_DISTANCE, left = chain;
    int has_prefix = pos + 4 <= z->n;
    uint32_t prefix = has_prefix ? rd32(d + pos) : 0;
    while (cp >= 0 && left > 0) {
        size_t mp = (size_t)cp, dd = pos - mp;
        if (dd == 0) { cp = z->prev[mp % MAX_DISTANCE]; left--; continue; }
        if (dd > maxd) break;
        if (has_prefix && mp + 4 <= z->n && rd32(d + mp) != prefix) { cp = z->prev[mp % MAX_DISTANCE]; left--; continue; }
        size_t len = match_len(z, mp, pos);
        if (len >= minm && !(len == 3 && dd > 8192) && (len > best || (len == best && dd < bd))) {
            best = len, bd = dd;
            if (len >= MAX_MATCH || best >= nice) break;
        }
        cp = z->prev[mp % MAX_DISTANCE];
        left--;
    }
    if (best >= minm) { *dist = bd; return best; }
    return 0;
}

/* find_best_match_ht, lz77.rs:752-812: inserts pos into its bucket before it searches */
static size_t find_best_ht(Lz *z, size_t pos, size_t nice, size_t minm, size_t *dist)
{
    if (pos + MIN_MATCH > z->n) return 0;
    int32_t *b = z->ht + 2 * hash4_ht(z, pos);
    int32_t c[2] = {b[0], b[1]};
    b[1] = c[0];
    b[0] = (int32_t)pos;
    size_t best = minm > 0 ? minm - 1 : 0, bd = 0;
    for (int k = 0; k < 2; k++) {
        if (c[k] < 0) continue;
        size_t mp = (size_t)c[k], dd = pos - mp;
        if (dd == 0 || dd > MAX_DISTANCE || mp + 3 > z->n || memcmp(z->d + pos, z->d + mp, 3)) continue;
        size_t len = match_len(z, mp, pos);
        if (len < minm || (len == 3 && dd > 8192)) continue;
        if (len > best) {
            best = len, bd = dd;
            if (best >= nice) break;
        }
    }
    if (best >= minm) { *dist = bd; return best; }
    return 0;
}

/* calculate_min_match_len / choose_min_match_len, lz77.rs:329-360 */
static size_t min_match_len(const uint8_t *d, size_t n, size_t depth)
{
    int used[256] = {0}, k = 0;
    for (size_t i = 0; i < (n < 4096 ? n : 4096); i++)
        if (!used[d[i]]) used[d[i]] = 1, k++;
    if (depth <= 4) return MIN_MATCH;
    size_t m = MIN_MATCH;
    if (k > 32) m = 4;
    if (k > 64 && depth >= 10) m = 5;
    if (k > 96 && depth >= 20) m = 6;
    return m;
}

static void push_match(uint32_t *t, size_t *nt, size_t len, size_t dist) { t[(*nt)++] = (uint32_t)(dist - 1) << 16 | (uint32_t)len; }

/* Lz77Compressor::compress_into_sink, lz77.rs:403-591.  tokens: room for n; returns the token count. */
size_t pd_lz77(const uint8_t *d, size_t n, int level, uint32_t *tok)
{
    if (n == 0) return 0;
    const Cfg c = CFG[level < 1 ? 1 : level > 9 ? 9 : level];
    Lz z = {d, n, malloc(HASH_SIZE * 4), malloc(HASH3_SIZE * 4), malloc(HT_SIZE * 8), malloc(MAX_DISTANCE * 4)};
    memset(z.head, 0xFF, HASH_SIZE * 4), memset(z.head3, 0xFF, HASH3_SIZE * 4);
    memset(z.ht, 0xFF, HT_SIZE * 8), memset(z.prev, 0xFF, MAX_DISTANCE * 4);
    const size_t minm = min_match_len(d, n, (size_t)c.depth), depth = (size_t)c.depth, nice = (size_t)c.nice;
    size_t pos = 0, nt = 0, streak = 0, probe = 0, updates = 0, pend_len = 0, pend_dist = 0;
    int incompressible = 0;
    while (pos < n) {
        if (incompressible) {
            if (probe >= 256) {   /* INCOMPRESSIBLE_PROBE_INTERVAL, chain INCOMPRESSIBLE_CHAIN_LIMIT 1 */
                probe = 0;
                size_t dist, len = find_best(&z, pos, 1 < depth ? 1 : depth, nice, minm, &dist);
                if (len) {
                    incompressible = 0, streak = 0;
                    push_match(tok, &nt, len, dist);
                    if (dist == 1) {
                        update_hash(&z, pos);
                        update_hash(&z, pos + len - 1);
                    } else {
                        for (size_t i = 0; i < len; i++) update_hash(&z, pos + i);
                    }
                    pos += len;
                    continue;
                }
            }
            tok[nt++] = LIT_FLAG | d[pos];
            if (++updates >= 64) update_hash(&z, pos), updates = 0;   /* INCOMPRESSIBLE_UPDATE_INTERVAL */
            pos++, streak++, probe++;
            continue;
        }
        size_t chain = (size_t)c.chain;
        if (streak >= 512) incompressible = 1, probe = 0, chain = 1;   /* INCOMPRESSIBLE_LITERAL_THRESHOLD */
        size_t len = 0, dist = 0;
        if (pend_len) len = pend_len, dist = pend_dist, pend_len = 0;
        else if (c.ht) len = find_best_ht(&z, pos, nice, minm, &dist);
        else len = find_best(&z, pos, chain < depth ? chain : depth, nice, minm, &dist);
        if (len) {
            streak = 0, incompressible = 0, probe = 0;
            if (c.lazy && len < nice && len < GOOD_MATCH && pos + 1 < n) {
                update_hash(&z, pos);
                size_t next_chain = c.lazy == 2 ? (chain / 2 > 1 ? chain / 2 : 1) : chain, nd = 0;
                size_t nl = c.ht ? find_best_ht(&z, pos + 1, nice, minm, &nd)
                                 : find_best(&z, pos + 1, next_chain < depth ? next_chain : depth, nice, minm, &nd);
                if (nl && (nl >= len + 3 || nl >= nice)) {
                    tok[nt++] = LIT_FLAG | d[pos];
                    pend_len = nl, pend_dist = nd;
                    pos++;
                    continue;
                }
            }
            push_match(tok, &nt, len, dist);
            if (dist == 1) {
                update_hash(&z, pos);
                update_hash(&z, pos + len - 1);
            } else {
                for (size_t i = 0; i < len; i++) update_hash(&z, pos + i);
            }
            pos += len;
        } else {
            if (++streak >= 512) incompressible = 1, probe = 0, updates = 0;
            tok[nt++] = LIT_FLAG | d[pos];
            update_hash(&z, pos);
            pos++;
        }
    }
    free(z.head), free(z.head3), free(z.ht), free(z.prev);
    return nt;
}

/* ---- Huffman: build_codes with Rust std's BinaryHeap<Reverse<Node>> ---------------------------------------- */

typedef struct { uint32_t f; int32_t sym; int32_t l, r; } Node;   /* sym -1: None (internal) */

/* Node's Ord, huffman.rs:30-37: (frequency, Option<symbol>), None < Some */
static int node_cmp(const Node *a, const Node *b)
{
    if (a->f != b->f) return a->f < b->f ? -1 : 1;
    return a->sym < b->sym ? -1 : a->sym > b->sym;
}
/* the heap holds Reverse<Node>: x <= y as heap elements iff node y <= node x */
static int hle(const Node *N, int x, int y) { return node_cmp(&N[y], &N[x]) <= 0; }
static int hlt(const Node *N, int x, int y) { return node_cmp(&N[y], &N[x]) < 0; }
static int hge(const Node *N, int x, int y) { return hle(N, y, x); }

/* BinaryHeap::sift_up */
static size_t sift_up(const Node *N, int *h, size_t start, size_t pos)
{
    int e = h[pos];
    while (pos > start) {
        size_t parent = (pos - 1) / 2;
        if (hle(N, e, h[parent])) break;
        h[pos] = h[parent];
        pos = parent;
    }
    h[pos] = e;
    return pos;
}
/* BinaryHeap::sift_down_range */
static void sift_down_range(const Node *N, int *h, size_t pos, size_t end)
{
    int e = h[pos];
    size_t child = 2 * pos + 1;
    while (child + 2 <= end) {   /* child <= end.saturating_sub(2) */
        child += hle(N, h[child], h[child + 1]);
        if (hge(N, e, h[child])) { h[pos] = e; return; }
        h[pos] = h[child];
        pos = child;
        child = 2 * pos + 1;
    }
    if (child == end - 1 && hlt(N, e, h[child])) h[pos] = h[child], pos = child;
    h[pos] = e;
}
/* BinaryHeap::sift_down_to_bottom */
static void sift_down_to_bottom(const Node *N, int *h, size_t end)
{
    size_t pos = 0, child = 1;
    int e = h[0];
    while (child + 2 <= end) {
        child += hle(N, h[child], h[child + 1]);
        h[pos] = h[child];
        pos = child;
        child = 2 * pos + 1;
    }
    if (child == end - 1) h[pos] = h[child], pos = child;
    h[pos] = e;
    sift_up(N, h, 0, pos);
}
static int heap_pop(const Node *N, int *h, size_t *len)
{
    int item = h[--*len];
    if (*len) {
        int top = h[0];
        h[0] = item;
        sift_down_to_bottom(N, h, *len);
        item = top;
    }
    return item;
}

static void depths(const Node *N, int i, int d, uint8_t *len)
{
    if (N[i].sym >= 0) { len[N[i].sym] = (uint8_t)(d > 1 ? d : 1); return; }
    depths(N, N[i].l, d + 1, len), depths(N, N[i].r, d + 1, len);
}

/* limit_code_lengths, huffman.rs:128-205 */
static void limit_lengths(uint8_t *len, int n, int maxl)
{
    int over = 0;
    for (int i = 0; i < n; i++) over |= len[i] > maxl;
    if (!over) return;
    for (int i = 0; i < n; i++) if (len[i] > maxl) len[i] = (uint8_t)maxl;
    uint32_t lim = 1u << maxl, k = 0;
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
        uint32_t o = 1u << (maxl - len[bi]), nw = 1u << (maxl - (len[bi] - 1));
        if (k - o + nw <= lim) k = k - o + nw, len[bi]--;
        else break;
    }
}

/* build_codes' lengths, huffman.rs:48-110 (n <= 286) */
void pd_code_lengths(const uint32_t *freq, int n, int maxl, uint8_t *len)
{
    Node N[2 * 286];
    int h[286], nn = 0;
    memset(len, 0, (size_t)n);
    for (int i = 0; i < n; i++)
        if (freq[i]) N[nn] = (Node){freq[i], i, -1, -1}, h[nn] = nn, nn++;
    if (nn == 0) return;
    if (nn == 1) { len[N[0].sym] = 1; return; }
    size_t hl = (size_t)nn;
    for (size_t k = hl / 2; k > 0; k--) sift_down_range(N, h, k - 1, hl);   /* BinaryHeap::rebuild */
    int next = nn;
    while (hl > 1) {
        int a = heap_pop(N, h, &hl), b = heap_pop(N, h, &hl);
        N[next] = (Node){N[a].f + N[b].f, -1, a, b};
        h[hl] = next++;
        sift_up(N, h, 0, hl++);   /* BinaryHeap::push */
    }
    depths(N, h[0], 0, len);
    limit_lengths(len, n, maxl);
}

/* generate_canonical_codes, huffman.rs:212-244 (u16 arithmetic wraps as in a release build); codes bit-reversed
 * as prepare_reversed_codes does, deflate.rs:1573-1590 */
static void canonical_rev(const uint8_t *len, int n, uint32_t *code)
{
    uint32_t bl[16] = {0};
    uint16_t next[16] = {0}, c = 0;
    for (int i = 0; i < n; i++) if (len[i]) bl[len[i]]++;
    for (int b = 1; b <= 15; b++) c = (uint16_t)((uint16_t)(c + (uint16_t)bl[b - 1]) << 1), next[b] = c;
    for (int i = 0; i < n; i++) {
        code[i] = 0;
        if (!len[i]) continue;
        uint16_t v = next[len[i]]++;
        uint32_t r = 0;
        for (int k = 0; k < len[i]; k++) r |= ((v >> k) & 1u) << (len[i] - 1 - k);
        code[i] = r;
    }
}

/* ---- block writers ----------------------------------------------------------------------------------------- */

typedef struct { uint8_t *o; size_t cap, n; uint64_t acc; int bits; } Bw;   /* BitWriter64, bits.rs:121-181 */
static void put(Bw *w, uint32_t v, int nb)
{
    w->acc |= (uint64_t)(v & (nb == 32 ? 0xFFFFFFFFu : (1u << nb) - 1)) << w->bits;
    w->bits += nb;
    while (w->bits >= 8) {
        if (w->n < w->cap) w->o[w->n] = (uint8_t)w->acc;
        w->n++, w->acc >>= 8, w->bits -= 8;
    }
}
static void flush(Bw *w)
{
    if (w->bits) put(w, 0, 8 - w->bits);
}

static const uint16_t LBASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static const uint8_t LEXTRA[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t DBASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t DEXTRA[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

/* length_code / distance_code, deflate.rs:204-241 */
static int lcode(unsigned len) { int c = 0; while (c < 28 && !(len >= LBASE[c] && len < LBASE[c + 1])) c++; return c; }
static int dcode(unsigned d) { int c = 0; while (c < 29 && !(d >= DBASE[c] && d < DBASE[c + 1])) c++; return c; }

static void tokens(Bw *w, const uint32_t *t, size_t nt, const uint32_t *lc, const uint8_t *ll, const uint32_t *dc, const uint8_t *dl)
{
    for (size_t i = 0; i < nt; i++) {
        if (t[i] & LIT_FLAG) { put(w, lc[t[i] & 0xFF], ll[t[i] & 0xFF]); continue; }
        unsigned len = t[i] & 0xFFFF, dist = (t[i] >> 16) + 1;
        int a = lcode(len), b = dcode(dist);
        put(w, lc[257 + a], ll[257 + a]);
        if (LEXTRA[a]) put(w, len - LBASE[a], LEXTRA[a]);
        put(w, dc[b], dl[b]);
        if (DEXTRA[b]) put(w, dist - DBASE[b], DEXTRA[b]);
    }
    put(w, lc[256], ll[256]);
}

/* encode_fixed_huffman_packed_with_capacity, deflate.rs:1200-1237 */
static void fixed_block(Bw *w, const uint32_t *t, size_t nt)
{
    uint8_t ll[288], dl[32];
    uint32_t lc[288], dc[32];
    for (int i = 0; i < 288; i++) ll[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
    for (int i = 0; i < 32; i++) dl[i] = 5;
    canonical_rev(ll, 288, lc), canonical_rev(dl, 32, dc);
    put(w, 1, 1), put(w, 1, 2);
    tokens(w, t, nt, lc, ll, dc, dl);
    flush(w);
}

void pd_histogram(const uint32_t *t, size_t nt, uint32_t *lit, uint32_t *dist)
{
    memset(lit, 0, 286 * 4), memset(dist, 0, 30 * 4);
    for (size_t i = 0; i < nt; i++) {
        if (t[i] & LIT_FLAG) { lit[t[i] & 0xFF]++; continue; }
        lit[257 + lcode(t[i] & 0xFFFF)]++;
        dist[dcode((t[i] >> 16) + 1)]++;
    }
}

/* encode_dynamic_huffman_packed_with_capacity, deflate.rs:1364-1468, with rle_code_lengths :1490-1550 */
static void dynamic_block(Bw *w, const uint32_t *t, size_t nt)
{
    uint32_t lf[286], df[30], cf[19] = {0}, lc[286], dc[30], cc[19];
    uint8_t ll[286], dl[30], cl[19], seq[316], rs[316 + 8], rx[316 + 8], rn[316 + 8];
    pd_histogram(t, nt, lf, df);
    lf[256]++;
    int any = 0;
    for (int i = 0; i < 30; i++) any |= df[i] != 0;
    if (!any) df[0] = 1;
    pd_code_lengths(lf, 286, 15, ll), pd_code_lengths(df, 30, 15, dl);
    canonical_rev(ll, 286, lc), canonical_rev(dl, 30, dc);
    int ln = 1, dn = 1;   /* last_nonzero, deflate.rs:1470-1476 */
    for (int i = 285; i >= 0; i--) if (ll[i]) { ln = i + 1; break; }
    for (int i = 29; i >= 0; i--) if (dl[i]) { dn = i + 1; break; }
    int hlit = ln > 257 ? ln - 257 : 0, hdist = dn > 1 ? dn - 1 : 0;
    if (hlit > 29) hlit = 29;
    if (hdist > 29) hdist = 29;
    int ns = 0, nr = 0;
    for (int i = 0; i < 257 + hlit; i++) seq[ns++] = ll[i];
    for (int i = 0; i < 1 + hdist; i++) seq[ns++] = dl[i];
    for (int i = 0; i < ns;) {
        int cur = seq[i], run = 1;
        while (i + run < ns && seq[i + run] == cur) run++;
        int rem = run;
        if (cur == 0) {
            while (rem > 0) {
                if (rem >= 11) { int k = rem < 138 ? rem : 138; rs[nr] = 18, rx[nr] = (uint8_t)(k - 11), rn[nr++] = 7, rem -= k; }
                else if (rem >= 3) { int k = rem < 10 ? rem : 10; rs[nr] = 17, rx[nr] = (uint8_t)(k - 3), rn[nr++] = 3, rem -= k; }
                else rs[nr] = 0, rx[nr] = 0, rn[nr++] = 0, rem--;
                cf[rs[nr - 1]]++;
            }
        } else {
            rs[nr] = (uint8_t)cur, rx[nr] = 0, rn[nr++] = 0, cf[cur]++;
            rem = run - 1;
            while (rem >= 3) { int k = rem < 6 ? rem : 6; rs[nr] = 16, rx[nr] = (uint8_t)(k - 3), rn[nr++] = 2, cf[16]++, rem -= k; }
            while (rem > 0) rs[nr] = (uint8_t)cur, rx[nr] = 0, rn[nr++] = 0, cf[cur]++, rem--;
        }
        i += run;
    }
    pd_code_lengths(cf, 19, 7, cl);
    canonical_rev(cl, 19, cc);
    static const int ORD[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    int hclen = 0;
    for (int i = 18; i >= 0; i--) if (cl[ORD[i]]) { hclen = i < 15 ? i : 15; break; }
    put(w, 1, 1), put(w, 2, 2), put(w, (uint32_t)hlit, 5), put(w, (uint32_t)hdist, 5), put(w, (uint32_t)hclen, 4);
    for (int i = 0; i < hclen + 4; i++) put(w, cl[ORD[i]], 3);
    for (int i = 0; i < nr; i++) {
        put(w, cc[rs[i]], cl[rs[i]]);
        if (rn[i]) put(w, rx[i], rn[i]);
    }
    tokens(w, t, nt, lc, ll, dc, dl);
    flush(w);
}

/* deflate_stored, deflate.rs:1664-1688 */
static void stored(Bw *w, const uint8_t *d, size_t n)
{
    size_t k = n ? (n + 65534) / 65535 : 0;
    for (size_t i = 0; i < k; i++) {
        size_t m = n - i * 65535 < 65535 ? n - i * 65535 : 65535;
        put(w, i == k - 1, 8), put(w, (uint32_t)m, 16), put(w, (uint32_t)(~m & 0xFFFF), 16);
        for (size_t j = 0; j < m; j++) put(w, d[i * 65535 + j], 8);
    }
}

/* is_high_entropy_data, deflate.rs:1108-1145 (the f32 division restated in float) */
int pd_high_entropy(const uint8_t *d, size_t n)
{
    if (n < 4096) return 0;
    size_t s = n < 8192 ? n : 8192, coll = 0;
    uint8_t seen[4096] = {0};
    for (size_t i = 0; i + 4 <= s; i++) {
        uint32_t h = ((rd32(d + i) * 0x1E35A7BDu) >> 20) & 4095;
        if (seen[h]) coll++;
        else seen[h] = 1;
    }
    return (float)coll / (float)(s - 3) < 0.05f;
}

static uint32_t adler(const uint8_t *d, size_t n)
{
    uint32_t a = 1, b = 0;
    for (size_t i = 0; i < n; i++) a = (a + d[i]) % 65521, b = (b + a) % 65521;
    return b << 16 | a;
}

/* zlib_header, deflate.rs:1642-1658 */
static void zhdr(Bw *w, int level)
{
    unsigned flg = (unsigned)(level <= 2 ? 1 : level <= 6 ? 2 : 3) << 6;
    flg |= (31 - ((0x78u << 8 | flg) % 31)) % 31;
    put(w, 0x78, 8), put(w, flg, 8);
}

/* deflate_zlib_packed, deflate.rs:1074-1079 -> compress_packed_zlib :1008-1047.  Writes at most cap bytes of the
 * stream to out and returns its full length.  *kind (may be null): 0 stored, 1 fixed, 2 dynamic. */
size_t pd_deflate_zlib(const uint8_t *d, size_t n, int level, uint8_t *out, size_t cap, int *kind)
{
    level = level < 1 ? 1 : level > 9 ? 9 : level;
    Bw w = {out, cap, 0, 0, 0};
    int k = 0;
    zhdr(&w, level);
    if (n >= 4096 && pd_high_entropy(d, n)) {
        stored(&w, d, n);
    } else if (n == 0) {   /* empty_zlib, deflate.rs:1593-1610 */
        fixed_block(&w, NULL, 0);
        k = 1;
    } else {
        uint32_t *t = malloc(n * 4);
        size_t nt = pd_lz77(d, n, level, t), matches = 0;
        for (size_t i = 0; i < nt; i++) matches += !(t[i] & LIT_FLAG);
        if (matches == 0 && n >= 8192) {   /* STORED_LITERAL_ONLY_BYTES */
            stored(&w, d, n);
        } else {
            size_t start = w.n;
            k = nt <= 128 ? 1 : 2;   /* encode_best_huffman_packed, deflate.rs:121-144 */
            if (k == 1) fixed_block(&w, t, nt);
            else dynamic_block(&w, t, nt);
            size_t deflated = w.n - start;
            if (deflated + 6 >= n + (n / 65535 + 1) * 5 + 6) {   /* should_use_stored, deflate.rs:1091-1097 */
                w.n = start, w.acc = 0, w.bits = 0, k = 0;
                stored(&w, d, n);
            }
        }
        free(t);
    }
    uint32_t a = adler(d, n);
    put(&w, a >> 24, 8), put(&w, (a >> 16) & 0xFF, 8), put(&w, (a >> 8) & 0xFF, 8), put(&w, a & 0xFF, 8);
    if (kind) *kind = k;
    return w.n;
}
