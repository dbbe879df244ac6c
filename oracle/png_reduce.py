"""Plain restatement of pixo's lossless PNG colour-type and palette reduction (test infrastructure,
numpy only): maybe_reduce_color_type and its helpers, src/png/mod.rs:683-836,838-1147 and
src/png/bit_depth.rs.  It is written from the reference's documented behaviour, not translated
from its code, and is checked against real pixo output by tests/test_png_reduce.py.

reduce(data, w, h, color_type, reduce_color_type, reduce_palette) -> Reduced
"""
from __future__ import annotations

import dataclasses

import numpy as np

GRAY, GRAY_ALPHA, RGB, RGBA = 0, 1, 2, 3
PNG_COLOR_BYTE = (0, 4, 2, 6)     # ColorType::png_color_type, src/color.rs
M32 = 0xFFFFFFFF


@dataclasses.dataclass
class Reduced:
    color_type_byte: int          # IHDR colour type
    bit_depth: int                # IHDR bit depth
    effective_color_type: int     # what maybe_optimize_alpha sees (a palette counts as Rgb)
    bytes_per_pixel: int
    row_bytes: int
    palette: np.ndarray | None    # (n, 4) uint8 RGBA, PLTE order
    data: np.ndarray              # the reduced rows, height * row_bytes bytes

    @property
    def trns(self) -> bytes | None:
        """tRNS payload: written iff some palette alpha is below 255 (src/png/mod.rs:535-545)."""
        if self.palette is None or not (self.palette[:, 3] != 255).any():
            return None
        return self.palette[:, 3].tobytes()


def palette_bit_depth(n: int) -> int:
    """bit_depth.rs palette_bit_depth."""
    if n == 0:
        return 8
    return 1 if n <= 2 else 2 if n <= 4 else 4 if n <= 16 else 8


def gray_bit_depth(vmax: int) -> int:
    """bit_depth.rs reduce_gray_bit_depth, from the largest sample."""
    return 1 if vmax <= 1 else 2 if vmax <= 3 else 4 if vmax <= 15 else 8


def pack_rows(vals: np.ndarray, w: int, bits: int) -> np.ndarray:
    """bit_depth.rs pack_bits_rows: MSB first, every row's last byte padded with zero bits."""
    if bits == 8:
        return vals.reshape(-1).copy()
    v = vals.reshape(-1, w).astype(np.uint8) & ((1 << bits) - 1)
    per = 8 // bits
    wp = -(-w // per) * per
    v = np.pad(v, ((0, 0), (0, wp - w)))
    v = v.reshape(v.shape[0], -1, per).astype(np.uint16)
    shifts = (8 - bits * (np.arange(per) + 1)).astype(np.uint16)
    return (v << shifts).sum(axis=2).astype(np.uint8).reshape(-1)


def _keys(px: np.ndarray, ct: int) -> np.ndarray:
    """r<<24 | g<<16 | b<<8 | a (a = 255 for Rgb), build_palette's key."""
    p = px.astype(np.uint32)
    a = p[:, 3] if ct == RGBA else np.uint32(255)
    return (p[:, 0] << 24) | (p[:, 1] << 16) | (p[:, 2] << 8) | a


def co_occurrence(idx: np.ndarray, n: int, w: int, h: int) -> np.ndarray:
    """build_co_occurrence_matrix: right and below neighbours, both directions, wrapping u32."""
    g = idx.reshape(h, w).astype(np.int64)
    pairs = [(g[:, :-1].ravel(), g[:, 1:].ravel()), (g[:-1, :].ravel(), g[1:, :].ravel())]
    m = np.zeros(n * n, np.uint64)
    for a, b in pairs:
        m += np.bincount(a * n + b, minlength=n * n).astype(np.uint64)
        m += np.bincount(b * n + a, minlength=n * n).astype(np.uint64)
    return (m & M32).reshape(n, n)


def weighted_edges(m: np.ndarray) -> list[tuple[int, int]]:
    """(j, i) for j < i in row-major order of i then j, weight > 0, stably sorted by weight, heaviest first."""
    n = m.shape[0]
    e = [((j, i), int(m[i, j])) for i in range(n) for j in range(i) if m[i, j] > 0]
    e.sort(key=lambda t: -t[1])   # list.sort is stable, like slice::sort_by
    return [t[0] for t in e]


def mzeng_reindex(n: int, edges, m: np.ndarray) -> list[int]:
    """Modified Zeng ordering (Pinho et al., IEEE 2004) as mzeng_reindex runs it: first maximum wins,
    removal by swap_remove, prepend when delta > 0."""
    M = m.tolist()
    remap = [edges[0][0], edges[0][1]]
    sums = []
    best_pos, best = 0, (0, 0)
    for i in range(n):
        if i == remap[0] or i == remap[1]:
            continue
        s = (M[i][remap[0]] + M[i][remap[1]]) & M32
        if s > best[1]:
            best_pos, best = len(sums), (i, s)
        sums.append([i, s])
    while sums:
        bi = best[0]
        placed = n - len(sums)
        delta = 0
        for k, c in enumerate(remap):
            delta += (placed - 1 - 2 * k) * M[bi][c]
        if delta > 0:
            remap.insert(0, bi)
        else:
            remap.append(bi)
        sums[best_pos] = sums[-1]     # Vec::swap_remove
        sums.pop()
        if sums:
            best_pos, best = 0, (0, 0)
            row = M[bi]
            for k, s in enumerate(sums):
                s[1] = (s[1] + row[s[0]]) & M32
                if s[1] > best[1]:
                    best_pos, best = k, (s[0], s[1])
    return remap


def most_popular_first(idx: np.ndarray, remap: list[int]) -> list[int]:
    """apply_most_popular_first: counts over the pre-remap indices; the last of equal maxima; 15 %."""
    counts = np.bincount(idx, minlength=256)
    best_i, best_c = 0, -1
    for c in remap:                       # Iterator::max_by_key keeps the last maximum
        if counts[c] >= best_c:
            best_i, best_c = c, int(counts[c])
    thr = ((idx.size & M32) * 3 & M32) // 20
    if best_c < thr:
        return remap
    pos = remap.index(best_i)
    if pos >= len(remap) // 2:
        r = remap[::-1]
        k = (pos + 1) % len(r)
        return r[len(r) - k:] + r[:len(r) - k]          # rotate_right(pos + 1)
    return remap[pos:] + remap[:pos]                       # rotate_left(pos)


def palette_order(idx: np.ndarray, n: int, w: int, h: int) -> list[int]:
    """optimize_palette_order: the new order as a list of old indices."""
    if n <= 2:
        return list(range(n))
    m = co_occurrence(idx, n, w, h)
    edges = weighted_edges(m)
    if not edges:
        return list(range(n))
    return most_popular_first(idx, mzeng_reindex(n, edges, m))


def build_palette(px: np.ndarray, ct: int, w: int, h: int):
    """build_palette: sorted unique keys (<= 256), pre-remap indices, Zeng order.  None past 256."""
    keys = _keys(px, ct)
    uniq, inv = np.unique(keys, return_inverse=True)
    if uniq.size > 256:
        return None
    idx = inv.astype(np.uint8).reshape(-1)
    order = palette_order(idx, uniq.size, w, h)
    byte_map = np.zeros(256, np.uint8)
    byte_map[np.array(order)] = np.arange(len(order), dtype=np.uint8)
    pal = uniq[np.array(order)]
    pal = np.stack([(pal >> s) & 255 for s in (24, 16, 8, 0)], axis=1).astype(np.uint8)
    return byte_map[idx], pal


def reduce(data, w: int, h: int, ct: int, reduce_color_type: bool, reduce_palette: bool) -> Reduced:
    """maybe_reduce_color_type (src/png/mod.rs:683-836)."""
    bpp = (1, 2, 3, 4)[ct]
    d = np.ascontiguousarray(np.asarray(data, np.uint8)).reshape(-1)
    assert d.size == w * h * bpp
    unchanged = Reduced(PNG_COLOR_BYTE[ct], 8, ct, bpp, w * bpp, None, d.copy())
    if ct == GRAY and reduce_color_type:
        return unchanged                 # Gray input is not bit-reduced
    px = d.reshape(-1, bpp)
    if reduce_palette and ct in (RGB, RGBA):
        r = build_palette(px, ct, w, h)
        if r is not None:
            idx, pal = r
            bits = palette_bit_depth(len(pal))
            return Reduced(3, bits, RGB, 1, -(-w * bits // 8), pal, pack_rows(idx, w, bits))
    if not reduce_color_type or ct not in (RGB, RGBA):
        return unchanged
    gray = bool((px[:, 0] == px[:, 1]).all() and (px[:, 1] == px[:, 2]).all())
    opaque = ct == RGB or bool((px[:, 3] == 255).all())

    def to_gray():
        bits = gray_bit_depth(int(px[:, 0].max()))
        return Reduced(0, bits, GRAY, 1, -(-w * bits // 8), None, pack_rows(px[:, 0], w, bits))

    if ct == RGB:
        return to_gray() if gray else unchanged
    if opaque and gray:
        return to_gray()
    if opaque:
        return Reduced(2, 8, RGB, 3, w * 3, None, px[:, :3].reshape(-1).copy())
    if gray:
        return Reduced(4, 8, GRAY_ALPHA, 2, w * 2, None, px[:, [0, 3]].reshape(-1).copy())
    return unchanged


def filter_input(r: Reduced, optimize_alpha: bool) -> np.ndarray:
    """maybe_optimize_alpha on the reduced rows, by their effective colour type (src/png/mod.rs:633-671)."""
    d = r.data.copy()
    if optimize_alpha and r.effective_color_type in (RGBA, GRAY_ALPHA):
        b = r.bytes_per_pixel
        v = d.reshape(-1, b)
        v[v[:, b - 1] == 0, :b - 1] = 0
    return d
