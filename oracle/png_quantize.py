"""Plain restatement of pixo's lossy PNG path (test infrastructure): the Auto decision, the sampled
histogram, median cut, the k-means refinement, maybe_trim_transparency and the filter-strategy remap of
encode_indexed_into (src/png/mod.rs:469-511,1172-1390,1505-1762,1866-1902), in Python and numpy.  The
palette mapping itself (PaletteLut, the plain map and the dither) runs in pixo's f32 form in
oracle/png_quantize.c, built here into oracle/libpng_quantize.so.  Written from the reference's documented
behaviour, and checked against real pixo output by tests/test_png_quantize.py.

quantize(data, w, h, ct, max_colors, dithering, palette=None) -> (palette (n, 4) uint8, indices)
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libpng_quantize.so")
RGB, RGBA = 2, 3
F_NONE, F_MINSUM, F_ADAPTIVE, F_ADAPTIVE_FAST, F_BIGRAMS = 0, 5, 6, 7, 8


class TruncationCase(Exception):
    """More than 8192 histogram colours: pixo's unstable-sort truncation, which is not restated."""


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "png_quantize.c")
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-fno-fast-math", "-msse2",
                               "-mfpmath=sse", "-fPIC", "-Wall", "-shared", "-o", SO, src])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        p = C.c_void_p
        L.pq_lut.argtypes = [p, C.c_int, p]
        L.pq_map.argtypes = [p, C.c_size_t, C.c_int, p, C.c_int, p, C.c_int, p]
        L.pq_dither.argtypes = [p, C.c_uint32, C.c_uint32, C.c_int, p, C.c_int, p, p]
        _lib = L
    return _lib


def _keys(px: np.ndarray) -> np.ndarray:
    """r<<24|g<<16|b<<8|a per pixel (a = 255 for RGB)."""
    a = px[:, 3].astype(np.uint32) if px.shape[1] == 4 else np.full(len(px), 255, np.uint32)
    return (px[:, 0].astype(np.uint32) << 24) | (px[:, 1].astype(np.uint32) << 16) | \
        (px[:, 2].astype(np.uint32) << 8) | a


def _pixels(data, ct) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(data, np.uint8)).reshape(-1, ct + 1)


def should_quantize_auto(data, ct: int, max_colors: int) -> bool:
    px = _pixels(data, ct)
    stride = max(len(px) // 20000, 1)
    unique = len(np.unique(_keys(px[::stride])))
    return max_colors < unique <= max_colors * 32


def should_quantize(data, ct: int, mode: str, max_colors: int) -> bool:
    """encode_into's decision; mode 'off', 'auto' or 'force'; max_colors already min(256)."""
    if mode == "off" or ct not in (RGB, RGBA):
        return False
    return mode == "force" or should_quantize_auto(data, ct, max_colors)


def histogram(data, ct: int):
    """(keys in key order, counts): samples at stride max(N/50000, 1), each counting `stride`."""
    px = _pixels(data, ct)
    stride = max(len(px) // 50000, 1)
    keys, cnt = np.unique(_keys(px[::stride]), return_counts=True)
    return keys, np.minimum(cnt.astype(np.uint64) * stride, 0xFFFFFFFF).astype(np.uint64)


def _rgba(keys) -> np.ndarray:
    k = np.asarray(keys, np.uint32)
    return np.stack([(k >> 24) & 255, (k >> 16) & 255, (k >> 8) & 255, k & 255], 1).astype(np.uint8)


def _score(box):
    """ColorBox::range: (channel, weighted range); a later channel must be strictly larger."""
    c = np.array([b[0] for b in box], np.int64)
    rng = c.max(0) - c.min(0)
    best, ch = int(rng[0]) * 2, 0
    for k, wgt in ((1, 4), (2, 1), (3, 3)):
        if int(rng[k]) * wgt > best:
            best, ch = int(rng[k]) * wgt, k
    return ch, best


def median_cut(keys, counts, max_colors: int) -> np.ndarray:
    """median_cut_palette's boxes (before k-means): box means in box order."""
    cols = [(tuple(int(v) for v in c), int(n)) for c, n in zip(_rgba(keys), counts)]
    boxes = [(cols, _score(cols))]
    while len(boxes) < max_colors:
        idx = max(range(len(boxes)), key=lambda i: (boxes[i][1][1], i))   # the LAST largest (max_by_key)
        box, (ch, _) = boxes[idx]
        if len(box) <= 1:
            break
        boxes.pop(idx)
        box = sorted(box, key=lambda c: c[0][ch])                          # stable, as sort_by_key
        total = sum(n for _, n in box) & 0xFFFFFFFF
        acc, split = 0, 0
        for i, (_, n) in enumerate(box):
            acc = (acc + n) & 0xFFFFFFFF
            if acc >= total // 2:
                split = i
                break
        split = min(split, len(box) - 2)
        for part in (box[:split + 1], box[split + 1:]):
            boxes.append((part, _score(part)))
    pal = []
    for box, _ in boxes:
        c = np.array([b[0] for b in box], np.uint64)
        n = np.array([b[1] for b in box], np.uint64)
        t = int(n.sum())
        pal.append([int((c[:, k] * n).sum()) // t for k in range(4)] if t else [0, 0, 0, 255])
    return np.array(pal, np.uint8).reshape(-1, 4)


def distances(colors: np.ndarray, pal: np.ndarray) -> np.ndarray:
    """perceptual_distance_sq of every colour (rows) to every entry (columns)."""
    c = colors.astype(np.int64)[:, None, :]
    p = pal.astype(np.int64)[None, :, :]
    d = c - p
    rm = (c[..., 0] + p[..., 0]) >> 1
    return (((512 + rm) * d[..., 0] ** 2 + 1024 * d[..., 1] ** 2 + (767 - rm) * d[..., 2] ** 2) >> 8) + d[..., 3] ** 2


def kmeans(pal: np.ndarray, keys, counts, iterations: int = 2) -> np.ndarray:
    """refine_palette_kmeans: first nearest entry, u64 integer centroids, empty entries unchanged."""
    pal = pal.copy()
    cols = _rgba(keys).astype(np.uint64)
    n = np.asarray(counts, np.uint64)
    for _ in range(iterations):
        best = distances(cols, pal).argmin(1)
        for i in range(len(pal)):
            m = best == i
            t = int(n[m].sum())
            if t:
                pal[i] = [int((cols[m, k] * n[m]).sum()) // t for k in range(4)]
    return pal


def lut(pal: np.ndarray) -> np.ndarray:
    out = np.zeros(1 << 18, np.uint8)
    p = np.ascontiguousarray(pal, np.uint8)
    lib().pq_lut(p.ctypes.data, len(p), out.ctypes.data)
    return out


def map_indices(data, w: int, h: int, ct: int, pal: np.ndarray, dithering: bool, early_out: bool) -> np.ndarray:
    d = np.ascontiguousarray(np.asarray(data, np.uint8)).reshape(-1)
    p = np.ascontiguousarray(pal, np.uint8)
    out = np.zeros(w * h, np.uint8)
    t = np.zeros(1, np.uint8) if early_out else lut(p)
    if dithering and not early_out:
        lib().pq_dither(d.ctypes.data, w, h, ct + 1, p.ctypes.data, len(p), t.ctypes.data, out.ctypes.data)
    else:
        lib().pq_map(d.ctypes.data, w * h, ct + 1, p.ctypes.data, len(p), t.ctypes.data, int(early_out),
                     out.ctypes.data)
    return out


def quantize(data, w: int, h: int, ct: int, max_colors: int, dithering: bool, palette=None):
    """quantize_image: (palette (n, 4) uint8, indices).  `palette`: a given median-cut palette, mapped as
    quantize_image maps one (table, then plain map or dither).  Raises TruncationCase when pixo would
    truncate a histogram of more than 8192 colours and no palette is given."""
    max_colors = min(int(max_colors), 256)
    if palette is not None:
        pal = np.asarray(palette, np.uint8).reshape(-1, 4)
        return pal, map_indices(data, w, h, ct, pal, dithering, False)
    keys, counts = histogram(data, ct)
    if len(keys) > 8192:
        raise TruncationCase(f"{len(keys)} histogram colours")
    if len(keys) <= max_colors:
        pal = _rgba(keys)
        return pal, map_indices(data, w, h, ct, pal, False, True)
    pal = kmeans(median_cut(keys, counts, max_colors), keys, counts)
    return pal, map_indices(data, w, h, ct, pal, dithering, False)


def trimmed_trns(pal: np.ndarray) -> bytes | None:
    """maybe_trim_transparency."""
    a = pal[:, 3]
    nz = np.nonzero(a != 255)[0]
    return None if len(nz) == 0 else a[:nz[-1] + 1].tobytes()


def indexed_strategy(strategy: int) -> int:
    """encode_indexed_into's remap: Adaptive, AdaptiveFast, MinSum and Bigrams become None."""
    return F_NONE if strategy in (F_MINSUM, F_ADAPTIVE, F_ADAPTIVE_FAST, F_BIGRAMS) else strategy
