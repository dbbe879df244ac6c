/* CPU oracle of pixo's palette mapping (test infrastructure only): PaletteLut, the plain map, the
 * early-out map and Floyd-Steinberg dithering, in pixo's own f32 form (src/png/mod.rs:1405-1500,
 * 1582-1701).  The CUDA kernels carry the dither in integer sixteenths instead; the two forms are
 * independent, so their agreement is evidence for both.  Built by oracle/png_quantize.py.
 * Palettes are n x 4 bytes RGBA. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static uint32_t dist(const uint8_t *c, const uint8_t *p)
{
    int dr = c[0] - p[0], dg = c[1] - p[1], db = c[2] - p[2], da = c[3] - p[3];
    int rm = (c[0] + p[0]) >> 1;
    int d = ((512 + rm) * dr * dr + 1024 * dg * dg + (767 - rm) * db * db) >> 8;
    return (uint32_t)(d + da * da);
}

static uint8_t nearest(const uint8_t *c, const uint8_t *pal, int n)
{
    uint32_t best = UINT32_MAX;
    uint8_t bi = 0;
    for (int i = 0; i < n; ++i) {
        uint32_t d = dist(c, pal + 4 * i);
        if (d < best) { best = d; bi = (uint8_t)i; }
    }
    return bi;
}

void pq_lut(const uint8_t *pal, int n, uint8_t *lut)
{
    for (int r6 = 0; r6 < 64; ++r6)
        for (int g6 = 0; g6 < 64; ++g6)
            for (int b6 = 0; b6 < 64; ++b6) {
                uint8_t c[4] = {(uint8_t)((r6 << 2) | (r6 >> 4)), (uint8_t)((g6 << 2) | (g6 >> 4)),
                                (uint8_t)((b6 << 2) | (b6 >> 4)), 255};
                lut[(r6 << 12) | (g6 << 6) | b6] = nearest(c, pal, n);
            }
}

static uint8_t lookup(const uint8_t *lut, const uint8_t *pal, int n, const uint8_t *c)
{
    if (c[3] == 255) return lut[((c[0] >> 2) << 12) | ((c[1] >> 2) << 6) | (c[2] >> 2)];
    return nearest(c, pal, n);
}

static void load(const uint8_t *data, size_t p, int bpp, uint8_t *c)
{
    c[0] = data[p * bpp]; c[1] = data[p * bpp + 1]; c[2] = data[p * bpp + 2];
    c[3] = bpp == 4 ? data[p * bpp + 3] : 255;
}

/* early_out != 0: pal is the histogram in key order; exact binary search, nearest entry on a miss.
 * Otherwise the table for opaque pixels, a nearest-entry search for the rest. */
void pq_map(const uint8_t *data, size_t npix, int bpp, const uint8_t *pal, int n, const uint8_t *lut, int early_out,
            uint8_t *out)
{
    for (size_t p = 0; p < npix; ++p) {
        uint8_t c[4];
        load(data, p, bpp, c);
        if (!early_out) { out[p] = lookup(lut, pal, n, c); continue; }
        uint32_t key = ((uint32_t)c[0] << 24) | ((uint32_t)c[1] << 16) | ((uint32_t)c[2] << 8) | c[3];
        int lo = 0, hi = n - 1, hit = -1;
        while (lo <= hi) {
            int mid = (lo + hi) / 2;
            const uint8_t *q = pal + 4 * mid;
            uint32_t k = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
            if (k == key) { hit = mid; break; }
            if (k < key) lo = mid + 1; else hi = mid - 1;
        }
        out[p] = hit >= 0 ? (uint8_t)hit : nearest(c, pal, n);
    }
}

static float clampf(float v) { return v < 0.0f ? 0.0f : v > 255.0f ? 255.0f : v; }

void pq_dither(const uint8_t *data, uint32_t w, uint32_t h, int bpp, const uint8_t *pal, int n, const uint8_t *lut,
               uint8_t *out)
{
    size_t W = (size_t)w + 2;
    float *buf = calloc(6 * W, sizeof(float));
    float *er[3] = {buf, buf + W, buf + 2 * W}, *ne[3] = {buf + 3 * W, buf + 4 * W, buf + 5 * W};
    size_t p = 0;
    for (uint32_t y = 0; y < h; ++y) {
        for (size_t x = 0; x < w; ++x, ++p) {
            uint8_t c[4];
            load(data, p, bpp, c);
            for (int k = 0; k < 3; ++k) c[k] = (uint8_t)clampf((float)c[k] + er[k][x + 1]);
            uint8_t id = lookup(lut, pal, n, c);
            out[p] = id;
            for (int k = 0; k < 3; ++k) {
                float e = (float)c[k] - (float)pal[4 * id + k];
                er[k][x + 2] += e * 7.0f / 16.0f;
                ne[k][x] += e * 3.0f / 16.0f;
                ne[k][x + 1] += e * 5.0f / 16.0f;
                ne[k][x + 2] += e * 1.0f / 16.0f;
            }
        }
        for (int k = 0; k < 3; ++k) {
            float *t = er[k];
            memset(t, 0, W * sizeof(float));
            er[k] = ne[k];
            ne[k] = t;
        }
    }
    free(buf);
}
