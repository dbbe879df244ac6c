// png_host.hpp — host half of the PNG palette reduction: the palette ordering on <= 256 colours.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <vector>

#ifdef __CUDACC__
#define PIXO_HOST_DEVICE __host__ __device__
#else
#define PIXO_HOST_DEVICE
#endif

namespace pixo {

// Index of the unordered pair (a, b), a < b, of an n-colour palette in the upper-triangle array of
// co-occurrence counts (n * (n - 1) / 2 entries).
PIXO_HOST_DEVICE inline size_t tri_index(uint32_t a, uint32_t b, uint32_t n)
{
    return (size_t)a * (2 * n - a - 1) / 2 + (b - a - 1);
}

// optimize_palette_order (src/png/mod.rs:909-1099) from the GPU statistics: n sorted palette entries,
// counts[256] of every pre-remap index, tri = the off-diagonal co-occurrence counts (right and below
// neighbours, wrapping u32), npix = pixel count.  order[k] = pre-remap index of new entry k.
void palette_order(uint32_t n, const uint32_t *counts, const uint32_t *tri, uint64_t npix, uint8_t order[256]);

// median_cut_palette's box splitting (src/png/mod.rs:1301-1333, ColorBox :1172-1299) on a histogram in key
// order (keys r<<24|g<<16|b<<8|a, counts as quantize_image accumulates them); returns the box means in
// box order, before the k-means refinement.
std::vector<uint32_t> median_cut_palette(const std::vector<uint32_t> &keys, const std::vector<uint32_t> &counts,
                                         uint32_t max_colors);

// maybe_trim_transparency (src/png/mod.rs:1888-1902): tRNS entries to write, 0 when every alpha is 255.
uint32_t trimmed_trns_len(const uint32_t *alpha, uint32_t n);

}  // namespace pixo
