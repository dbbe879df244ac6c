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

namespace {

struct ColorCount {
    uint32_t key, count;
};

uint32_t channel_of(uint32_t key, int ch) { return (key >> (24 - 8 * ch)) & 255u; }

// ColorBox::range: (channel, score) with weights r 2, g 4, b 1, a 3; a later channel wins only when
// strictly larger
void box_range(const std::vector<ColorCount> &c, int &channel, uint32_t &score)
{
    uint32_t lo[4] = {255, 255, 255, 255}, hi[4] = {0, 0, 0, 0};
    for (const ColorCount &e : c)
        for (int ch = 0; ch < 4; ++ch) {
            lo[ch] = std::min(lo[ch], channel_of(e.key, ch));
            hi[ch] = std::max(hi[ch], channel_of(e.key, ch));
        }
    static const uint32_t weight[4] = {2, 4, 1, 3};
    channel = 0;
    score = (hi[0] - lo[0]) * weight[0];
    for (int ch = 1; ch < 4; ++ch)
        if ((hi[ch] - lo[ch]) * weight[ch] > score) { score = (hi[ch] - lo[ch]) * weight[ch]; channel = ch; }
}

}  // namespace

std::vector<uint32_t> median_cut_palette(const std::vector<uint32_t> &keys, const std::vector<uint32_t> &counts,
                                         uint32_t max_colors)
{
    std::vector<std::vector<ColorCount>> boxes(1);
    std::vector<std::pair<int, uint32_t>> range(1);   // each box's (channel, score)
    for (size_t i = 0; i < keys.size(); ++i) boxes[0].push_back({keys[i], counts[i]});
    if (boxes[0].empty()) return {255u};
    box_range(boxes[0], range[0].first, range[0].second);
    while (boxes.size() < max_colors) {
        // max_by_key: the LAST box of the largest score
        size_t idx = 0;
        for (size_t b = 1; b < boxes.size(); ++b)
            if (range[b].second >= range[idx].second) idx = b;
        if (boxes[idx].size() <= 1) break;
        std::vector<ColorCount> c = std::move(boxes[idx]);
        const int ch = range[idx].first;
        boxes.erase(boxes.begin() + (ptrdiff_t)idx);
        range.erase(range.begin() + (ptrdiff_t)idx);
        std::stable_sort(c.begin(), c.end(), [ch](const ColorCount &a, const ColorCount &b) {
            return channel_of(a.key, ch) < channel_of(b.key, ch);
        });
        // u32 arithmetic as pixo's release build does it (wrapping)
        uint32_t total = 0, acc = 0;
        for (const ColorCount &e : c) total += e.count;
        size_t split = 0;
        for (size_t i = 0; i < c.size(); ++i) {
            acc += c[i].count;
            if (acc >= total / 2) { split = i; break; }
        }
        split = std::min(split, c.size() - 2);
        boxes.emplace_back(c.begin(), c.begin() + (ptrdiff_t)split + 1);
        boxes.emplace_back(c.begin() + (ptrdiff_t)split + 1, c.end());
        for (size_t b = boxes.size() - 2; b < boxes.size(); ++b) {
            range.emplace_back();
            box_range(boxes[b], range.back().first, range.back().second);
        }
    }
    // make_palette_entry: u64 integer mean of each box
    std::vector<uint32_t> pal;
    for (const auto &b : boxes) {
        uint64_t sum[4] = {0, 0, 0, 0}, total = 0;
        for (const ColorCount &e : b) {
            for (int ch = 0; ch < 4; ++ch) sum[ch] += (uint64_t)channel_of(e.key, ch) * e.count;
            total += e.count;
        }
        if (!total) { pal.push_back(255u); continue; }
        uint32_t key = 0;
        for (int ch = 0; ch < 4; ++ch) key |= (uint32_t)(sum[ch] / total) << (24 - 8 * ch);
        pal.push_back(key);
    }
    return pal;
}

uint32_t trimmed_trns_len(const uint32_t *alpha, uint32_t n)
{
    uint32_t len = 0;
    for (uint32_t i = 0; i < n; ++i)
        if (alpha[i] != 255u) len = i + 1;
    return len;
}

}  // namespace pixo
