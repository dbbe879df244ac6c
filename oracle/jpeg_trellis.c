/*
 * jpeg_trellis.c — CPU restatement of pixo's trellis quantiser (src/jpeg/trellis.rs:67-321) and of
 * compute_all_coefficients(.., use_trellis = true) (src/jpeg/mod.rs:932-1125, quantize_dct :970).
 *
 * TEST INFRASTRUCTURE ONLY (see pixo_oracle.h).  Written from the algorithm as the reference states
 * it: a state list that grows by insertion with merging on (value, zero run), a stable sort by cost,
 * truncation to 8, and backtracking through every step's list.  Built by oracle/jpeg_trellis.py with
 * the block extraction and DCT of pixo_oracle.c, strict binary32 (no contraction, SSE scalar math).
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "pixo_oracle.h"

#define MAX_STATES 8
#define MAX_LIST (MAX_STATES * 5)

typedef struct {
    float cost;
    uint8_t zero_run;
    uint16_t parent;
    int16_t value;
} state_t;

/* Rust's `f32 as i16`: saturating, NaN -> 0 */
static int16_t sat_i16(float f)
{
    if (f != f) return 0;
    if (f >= 32767.0f) return 32767;
    if (f <= -32768.0f) return -32768;
    return (int16_t)f;
}

static int contains(const int16_t *c, int n, int16_t v)
{
    for (int i = 0; i < n; ++i)
        if (c[i] == v) return 1;
    return 0;
}

/* generate_candidates, trellis.rs:210-244 */
static int gen_candidates(float fq, int16_t c[5])
{
    const int16_t rounded = sat_i16(roundf(fq)), fl = sat_i16(floorf(fq)), ce = sat_i16(ceilf(fq));
    int n = 0;
    c[n++] = 0;
    if (fl != 0 && !contains(c, n, fl)) c[n++] = fl;
    if (rounded != 0 && !contains(c, n, rounded)) c[n++] = rounded;
    if (ce != 0 && !contains(c, n, ce)) c[n++] = ce;
    if (fabsf(fq) > 1.5f) {
        const int16_t ext = (int16_t)(fq >= 0.0f ? ce + 1 : fl - 1);
        if (!contains(c, n, ext)) c[n++] = ext;
    }
    return n;
}

static int category(int16_t v)
{
    int a = v < 0 ? -(int)v : v, n = 0;
    while (a) { ++n; a >>= 1; }
    return n;
}

/* estimate_ac_huffman_length, trellis.rs:260-279 */
static float huffman_length(int rs)
{
    switch (rs) {
    case 0x00: return 4.0f;
    case 0x01: return 2.0f;
    case 0x02: return 2.5f;
    case 0x03: return 3.0f;
    case 0x04: return 4.0f;
    case 0x11: return 3.0f;
    case 0x12: return 4.0f;
    case 0x21: return 4.0f;
    case 0xF0: return 10.0f;
    default: {
        const float run = (float)(rs >> 4), size = (float)(rs & 15);
        return 3.0f + run * 0.5f + size * 0.3f;
    }
    }
}

/* estimate_ac_rate, trellis.rs:246-258 */
static float ac_rate(int16_t value, int zero_run)
{
    const int cat = category(value);
    return huffman_length((zero_run << 4) | cat) + (float)cat;
}

/* stable insertion sort by cost (Rust's sort_by is stable) */
static void stable_sort(state_t *s, int n)
{
    for (int i = 1; i < n; ++i) {
        const state_t x = s[i];
        int j = i;
        while (j > 0 && x.cost < s[j - 1].cost) { s[j] = s[j - 1]; --j; }
        s[j] = x;
    }
}

/* trellis_quantize, trellis.rs:67-208 */
void po_trellis_quantize(const float dct[64], const float q[64], float lambda, int16_t out[64])
{
    static state_t all[64][MAX_LIST];
    int counts[64];
    memset(out, 0, 64 * sizeof(int16_t));
    out[0] = sat_i16(roundf(dct[0] / q[0]));
    all[0][0] = (state_t){0.0f, 0, 0, 0};
    counts[0] = 1;
    for (int zz = 1; zz < 64; ++zz) {
        const int nat = PO_ZIGZAG[zz];
        const float coef = dct[nat], qq = q[nat];
        int16_t cand[5];
        const int nc = gen_candidates(coef / qq, cand);
        const state_t *cur = all[zz - 1];
        state_t *next = all[zz];
        int nn = 0;
        for (int p = 0; p < counts[zz - 1]; ++p) {
            for (int k = 0; k < nc; ++k) {
                const int16_t c = cand[k];
                const float rec = (float)c * qq;
                const float d = coef - rec;
                const float distortion = d * d;
                float rate;
                int new_run;
                if (c == 0) {
                    const int r = cur[p].zero_run + 1;
                    if (r >= 16) { rate = 10.0f; new_run = 0; }
                    else { rate = 0.0f; new_run = r; }
                } else {
                    rate = ac_rate(c, cur[p].zero_run);
                    new_run = 0;
                }
                const float cost = cur[p].cost + rate + lambda * distortion;
                int found = -1;
                for (int i = 0; i < nn; ++i)
                    if (next[i].value == c && next[i].zero_run == new_run) { found = i; break; }
                const state_t st = {cost, (uint8_t)new_run, (uint16_t)p, c};
                if (found < 0) next[nn++] = st;
                else if (cost < next[found].cost) next[found] = st;
            }
        }
        stable_sort(next, nn);
        counts[zz] = nn < MAX_STATES ? nn : MAX_STATES;
    }
    state_t *fin = all[63];
    for (int i = 0; i < counts[63]; ++i)
        if (fin[i].zero_run > 0) fin[i].cost += 4.0f;
    int best = 0;
    for (int i = 1; i < counts[63]; ++i)
        if (fin[i].cost < fin[best].cost) best = i;
    int idx = best;
    for (int zz = 63; zz >= 1; --zz) {
        out[PO_ZIGZAG[zz]] = all[zz][idx].value;
        idx = all[zz][idx].parent;
    }
}

/* trellis_quantize_adaptive's lambda, trellis.rs:304-321 */
float po_trellis_lambda(int quality)
{
    if (quality >= 80) return 0.5f + (float)(100 - quality) * 0.025f;
    if (quality >= 50) return 1.0f + (float)(80 - quality) * 0.033f;
    return 2.0f + (float)(50 - quality) * 0.04f;
}

/* compute_all_coefficients(.., use_trellis = true): natural order, MCU order (as po_jpeg_coefficients) */
void po_jpeg_coefficients_trellis(const uint8_t *data, uint32_t w, uint32_t h, int color_type, int subsampling,
                                  const float lum_q[64], const float chr_q[64], int16_t *y, int16_t *cb,
                                  int16_t *cr)
{
    float yb[64], cbb[64], crb[64], d[64];
    if (color_type == PO_GRAY || subsampling == PO_S444) {
        const size_t bw = (w + 7) / 8, bh = (h + 7) / 8;
        for (size_t by = 0; by < bh; ++by)
            for (size_t bx = 0; bx < bw; ++bx) {
                const size_t i = by * bw + bx;
                po_extract_block(data, w, h, bx * 8, by * 8, color_type, yb, cbb, crb);
                po_dct_2d(yb, d);
                po_trellis_quantize(d, lum_q, 1.0f, y + i * 64);
                if (color_type == PO_GRAY) continue;
                po_dct_2d(cbb, d);
                po_trellis_quantize(d, chr_q, 1.0f, cb + i * 64);
                po_dct_2d(crb, d);
                po_trellis_quantize(d, chr_q, 1.0f, cr + i * 64);
            }
        return;
    }
    float y4[4][64];
    const size_t mw = (w + 15) / 16, mh = (h + 15) / 16;
    for (size_t my = 0; my < mh; ++my)
        for (size_t mx = 0; mx < mw; ++mx) {
            const size_t m = my * mw + mx;
            po_extract_mcu_420(data, w, h, mx * 16, my * 16, y4, cbb, crb);
            for (int k = 0; k < 4; ++k) {
                po_dct_2d(y4[k], d);
                po_trellis_quantize(d, lum_q, 1.0f, y + (m * 4 + k) * 64);
            }
            po_dct_2d(cbb, d);
            po_trellis_quantize(d, chr_q, 1.0f, cb + m * 64);
            po_dct_2d(crb, d);
            po_trellis_quantize(d, chr_q, 1.0f, cr + m * 64);
        }
}
