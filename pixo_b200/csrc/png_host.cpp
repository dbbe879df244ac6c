// png_host.cpp — the modified Zeng palette ordering (Pinho et al., IEEE 2004) exactly as pixo runs it:
//   weighted_edges            src/png/mod.rs:980-991   (stable sort, heaviest first)
//   mzeng_reindex             src/png/mod.rs:998-1059  (first maximum wins, Vec::swap_remove order)
//   apply_most_popular_first  src/png/mod.rs:1063-1099 (last of equal maxima, 15 % threshold)
// O(n^2) on n <= 256 colours; the statistics it reads come from k_reduce_index.
#include "png_host.hpp"

#include <algorithm>
#include <vector>

namespace pixo {

void palette_order(uint32_t n, const uint32_t *counts, const uint32_t *tri, uint64_t npix, uint8_t order[256])
{
    for (uint32_t i = 0; i < n; ++i) order[i] = (uint8_t)i;
    if (n <= 2) return;
    // the matrix is symmetric and only its off-diagonal entries are read
    auto M = [&](uint32_t a, uint32_t b) -> uint32_t {
        if (a == b) return 0;
        return a < b ? tri[tri_index(a, b, n)] : tri[tri_index(b, a, n)];
    };
    struct Edge { uint32_t j, i, w; };
    std::vector<Edge> edges;
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = 0; j < i; ++j)
            if (const uint32_t w = M(i, j)) edges.push_back({j, i, w});
    if (edges.empty()) return;
    std::stable_sort(edges.begin(), edges.end(), [](const Edge &a, const Edge &b) { return a.w > b.w; });

    std::vector<uint32_t> remap = {edges[0].j, edges[0].i};
    struct Cand { uint32_t c, sum; };
    std::vector<Cand> sums;
    size_t best_pos = 0;
    Cand best = {0, 0};
    for (uint32_t i = 0; i < n; ++i) {
        if (i == remap[0] || i == remap[1]) continue;
        const uint32_t s = M(i, remap[0]) + M(i, remap[1]);   // wrapping u32, as the reference
        if (s > best.sum) { best_pos = sums.size(); best = {i, s}; }
        sums.push_back({i, s});
    }
    while (!sums.empty()) {
        const uint32_t b = best.c;
        const int64_t placed = (int64_t)n - (int64_t)sums.size();
        int64_t delta = 0;
        for (size_t k = 0; k < remap.size(); ++k) delta += (placed - 1 - 2 * (int64_t)k) * (int64_t)M(b, remap[k]);
        if (delta > 0) remap.insert(remap.begin(), b);
        else remap.push_back(b);
        sums[best_pos] = sums.back();   // Vec::swap_remove
        sums.pop_back();
        if (!sums.empty()) {
            best_pos = 0;
            best = {0, 0};
            for (size_t k = 0; k < sums.size(); ++k) {
                sums[k].sum += M(b, sums[k].c);
                if (sums[k].sum > best.sum) { best_pos = k; best = sums[k]; }
            }
        }
    }

    // most popular colour first: counts over the pre-remap indices, max_by_key keeps the last maximum
    uint32_t top = 0, top_count = 0;
    bool any = false;
    for (uint32_t c : remap)
        if (!any || counts[c] >= top_count) { top = c; top_count = counts[c]; any = true; }
    const uint32_t threshold = (uint32_t)npix * 3u / 20u;   // `len as u32 * 3 / 20`, wrapping
    if (top_count >= threshold) {
        const size_t pos = (size_t)(std::find(remap.begin(), remap.end(), top) - remap.begin());
        if (pos >= remap.size() / 2) {
            std::reverse(remap.begin(), remap.end());
            const size_t k = (pos + 1) % remap.size();        // rotate_right(pos + 1)
            std::rotate(remap.begin(), remap.end() - k, remap.end());
        } else {
            std::rotate(remap.begin(), remap.begin() + pos, remap.end());   // rotate_left(pos)
        }
    }
    for (uint32_t k = 0; k < n; ++k) order[k] = (uint8_t)remap[k];
}

}  // namespace pixo
