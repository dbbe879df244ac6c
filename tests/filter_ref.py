"""An independent numpy restatement of pixo's PNG filter stage, with a model of how the GPU kernels route and score
each row, and mutants that restate single faults of those kernels.

It is written from pixo's semantics (src/png/filter.rs:64-208,302-527,610-649: score_filter, score_bigrams, the
five predictors, adaptive_filter / minsum_filter, adaptive_filter_fast, bigrams_filter and the pre-rules of
apply_filters_with_row_bytes; src/png/mod.rs:633-671: maybe_optimize_alpha), not from oracle/pixo_oracle.c, and is
checked against that oracle byte for byte.  For every row it records the route the kernels take, the five scores,
the winner, the ladder's exit and the smallest margin that decided it, so tests can assert what their rows exercise.

Routes (csrc/png_filter.cu, launch_png_filter_rows):
  "first"  k_png_band, the first row of a 16-row band: cheap candidates, then Paeth in a second pass if still open
  "fused"  k_png_band, the row above left its ladder open: all five candidates in one pass
  "two"    k_png_band, the row above ended its ladder early: cheap candidates, then Paeth if still open
  "row"    k_png_filter: rows too long for the band kernel's three shared-memory buffers (32 KiB segments)
  "sticky" k_png_filter, AdaptiveFast on an image of at most 32 rows: row 0 decides for every row
  "bigrams" k_png_filter's Bigrams scoring;  "fixed": a fixed filter type (no scores)

Mutants (a set of names and tuples) restate one fault each:
  "adaptive_lt" / "fast_lt"   the ladder ends on best < early instead of <=
  "no_plus_one"               early = row_bytes/4 (/8) without the + 1
  "up_le"                     AdaptiveFast: Up replaces Sub on <=
  "paeth_le:<route>"          Paeth replaces the best on <= on that route ("fused", "two" (also "first"), "row")
  "lane0_shfl"                k_png_band score4: lane 0 keeps its own shuffled word as vector v's left word
  "alpha_x0"                  k_png_band score4: optimize_alpha not applied to vector v's left word
  "no_trailing" / "no_ragged" k_png_band: the whole words after the last vector / the ragged last word unscored
  "pass0_unmasked"            k_png_filter: scores of the last segment's ragged word not masked to the row
  "bigram_seam"               k_png_filter: the bigram straddling each 32 KiB segment seam not counted
  ("drop", lo, hi)            bytes [lo, hi) of the row missing from every candidate's score, on every route
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

NONE, SUB, UP, AVG, PAETH = range(5)
MINSUM, ADAPTIVE, FAST, BIGRAMS = 5, 6, 7, 8
BAND_ROWS, SEG, THREADS = 16, 32768, 256
BAND_SMEM = 200 * 1024


# ---- predictors and scores ------------------------------------------------------------------------------------
def zero_alpha(row: np.ndarray, oa: int) -> np.ndarray:
    """maybe_optimize_alpha on one row: a pixel (oa = 2: GrayAlpha, 4: Rgba) whose alpha is 0 becomes all zero."""
    if not oa:
        return row
    px = row[:row.size - row.size % oa].reshape(-1, oa)
    out = row.copy()
    out[:px.size] = np.where(px[:, -1:] == 0, 0, px).reshape(-1)
    return out


def paeth(a, b, c):
    """paeth_predictor (src/png/filter.rs:281-298) on int arrays."""
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def neighbours(x: np.ndarray, b: np.ndarray, bpp: int):
    """left (a) and upper-left (c) of every byte; zero left of the first pixel"""
    a, c = np.zeros_like(x), np.zeros_like(b)
    a[bpp:], c[bpp:] = x[:-bpp], b[:-bpp]
    return a, c


def filtered(x, b, bpp, a=None, c=None) -> np.ndarray:
    """(5, n) uint8: the row under None, Sub, Up, Average and Paeth (wrapping differences)."""
    x, b = x.astype(np.int32), b.astype(np.int32)
    if a is None:
        a, c = neighbours(x, b, bpp)
    a, c = np.asarray(a, np.int32), np.asarray(c, np.int32)
    preds = (np.zeros_like(x), a, b, (a + b) >> 1, paeth(a, b, c))
    return np.stack([(x - p) & 255 for p in preds]).astype(np.uint8)


def abs_i8(f: np.ndarray) -> np.ndarray:
    f = f.astype(np.int32)
    return np.where(f >= 128, 256 - f, f)


def score(f: np.ndarray) -> int:
    """score_filter: sum of |i8| (src/png/filter.rs:610-627)"""
    return int(abs_i8(f).sum())


def bigrams(f: np.ndarray, skip=()) -> int:
    """score_bigrams: distinct windows(2) (src/png/filter.rs:629-649); `skip` lists pair indices left out"""
    if f.size < 2:
        return 0
    keys = f[:-1].astype(np.int32) << 8 | f[1:]
    if len(skip):
        keys = np.delete(keys, list(skip))
    return int(np.unique(keys).size)


def scores(x, b, bpp, a=None, c=None, keep=None) -> list[int]:
    fs = abs_i8(filtered(x, b, bpp, a, c))
    if keep is not None:
        fs = fs * keep
    return [int(v) for v in fs.sum(axis=1)]


# ---- the ladders ------------------------------------------------------------------------------------------------
@dataclass
class Pick:
    winner: int
    exit: str           # "early" (the ladder ended before Paeth) or "paeth" (Paeth was compared)
    margin: int         # smallest |difference| among the comparisons that decided the row
    open: bool          # the cheap ladder left Paeth in (the band kernel's next row scores fused)


def early_of(strategy: int, rb: int, mut=frozenset()) -> int:
    return rb // (8 if strategy == FAST else 4) + (0 if "no_plus_one" in mut else 1)


def ladder(s, strategy: int, rb: int, mut=frozenset(), route: str = "") -> Pick:
    """adaptive_filter / minsum_filter (src/png/filter.rs:302-404) and adaptive_filter_fast (:474-527)."""
    early = early_of(strategy, rb, mut)
    fast = strategy == FAST
    stop_lt = ("fast_lt" if fast else "adaptive_lt") in mut
    ends = (lambda v: v == 0 or v < early) if stop_lt else (lambda v: v <= early)
    margins = []
    if fast:
        win, best = SUB, s[SUB]
        margins.append(abs(best - early))
        done = ends(best)
        if not done:
            margins.append(abs(s[UP] - best))
            if s[UP] < best or ("up_le" in mut and s[UP] == best):
                win, best = UP, s[UP]
                margins.append(abs(best - early))
            done = ends(best)
    else:
        win, best = NONE, s[NONE]
        margins.append(abs(best - early))
        done = ends(best)
        for f in (SUB, UP, AVG):
            if done:
                break
            margins.append(abs(s[f] - best))
            if s[f] < best:
                win, best = f, s[f]
                margins.append(abs(best - early))
                done = ends(best)
    if done:
        return Pick(win, "early", min(margins), False)
    margins.append(abs(s[PAETH] - best))
    rname = {"first": "two", "sticky": "row"}.get(route, route)
    if s[PAETH] < best or (f"paeth_le:{rname}" in mut and s[PAETH] == best):
        win = PAETH
    return Pick(win, "paeth", min(margins), True)


# ---- how the kernels score a row --------------------------------------------------------------------------------
def band_scores(xr, br, bpp, oa=0, mut=frozenset()):
    """k_png_band's scores of one row (raw bytes xr, raw row above br), with its scoring mutants."""
    x, b = zero_alpha(xr, oa), zero_alpha(br, oa)
    a, c = neighbours(x, b, bpp)
    rb = x.size
    full, keep = rb >> 2, np.ones(rb, np.int32)
    nv = full >> 2
    if "lane0_shfl" in mut or "alpha_x0" in mut:
        a, c = a.copy(), c.copy()
        ar, cr = neighbours(xr, br, bpp)
        for v in range(1 if "alpha_x0" in mut else 0, nv, 1 if "alpha_x0" in mut else 32):
            for j in range(16 * v, 16 * v + bpp):
                if "alpha_x0" in mut:        # the left word read raw
                    a[j], c[j] = ar[j], cr[j]
                else:                         # lane 0's left word = its own word 3
                    a[j], c[j] = x[j - bpp + 16], b[j - bpp + 16]
    if "no_trailing" in mut:
        keep[16 * nv:4 * full] = 0
    if "no_ragged" in mut:
        keep[4 * full:] = 0
    for m in mut:
        if isinstance(m, tuple) and m[0] == "drop":
            keep[m[1]:m[2]] = 0
    return scores(x, b, bpp, a, c, keep)


def row_scores(xr, br, bpp, oa=0, mut=frozenset()):
    """k_png_filter's pass-0 scores of one row (32 KiB segments, masked ragged word), with its mutants."""
    x, b = zero_alpha(xr, oa), zero_alpha(br, oa)
    rb = x.size
    keep = np.ones(rb, np.int32)
    for m in mut:
        if isinstance(m, tuple) and m[0] == "drop":
            keep[m[1]:m[2]] = 0
    if "pass0_unmasked" in mut and rb % 4:
        pad = 4 - rb % 4
        x, b = np.concatenate([x, np.zeros(pad, np.uint8)]), np.concatenate([b, np.zeros(pad, np.uint8)])
        keep = np.concatenate([keep, np.ones(pad, np.int32)])
    return scores(x, b, bpp, keep=keep)


def bigram_scores(xr, br, bpp, oa=0, mut=frozenset()):
    x, b = zero_alpha(xr, oa), zero_alpha(br, oa)
    fs = filtered(x, b, bpp)
    skip = [k * SEG - 1 for k in range(1, (x.size - 1) // SEG + 1)] if "bigram_seam" in mut else ()
    return [bigrams(f, skip) for f in fs]


# ---- routing ----------------------------------------------------------------------------------------------------
def effective_strategy(strategy: int, width: int, rule_height: int) -> int:
    """the area pre-rule of apply_filters_with_row_bytes (src/png/filter.rs:75-86)"""
    if width * rule_height <= 4096 and strategy in (ADAPTIVE, FAST, BIGRAMS):
        return SUB
    return strategy


def use_band(rb: int) -> bool:
    return 3 * (32 + (rb + 15) // 16 * 16) <= BAND_SMEM and rb < (1 << 18)


@dataclass
class RowInfo:
    route: str
    scores: list = field(default_factory=list)
    winner: int = 0
    exit: str = ""
    margin: int = -1


def apply_filters(data, width, height, bpp, strategy, rb=None, oa=0, rule_height=None, above=None,
                  mut=frozenset()):
    """apply_filters_with_row_bytes as the kernels run it (optimize_alpha fused when oa = 2 / 4): the filtered
    stream, and a RowInfo per row.  `above` and `rule_height` describe a band of a taller image, as
    png_filter_rows_dev takes it (bands of 16 rows count from the band's first row)."""
    rb = width * bpp if rb is None else rb
    rule_height = height if rule_height is None else rule_height
    rows = np.asarray(data, np.uint8).reshape(height, rb)
    st = effective_strategy(strategy, width, rule_height)
    sticky = st == FAST and rule_height <= 32
    band = not sticky and st != BIGRAMS and use_band(rb)
    out = np.zeros((height, rb + 1), np.uint8)
    infos = []
    prev_open, forced = False, None
    zero = np.zeros(rb, np.uint8)
    for r in range(height):
        xr = rows[r]
        br = rows[r - 1] if r else (zero if above is None else np.asarray(above, np.uint8))
        x, b = zero_alpha(xr, oa), zero_alpha(br, oa)
        if st < 5:
            info = RowInfo("fixed", winner=st)
        elif forced is not None:
            info = RowInfo("sticky", winner=forced)
        elif st == BIGRAMS:
            s = bigram_scores(xr, br, bpp, oa, mut)
            info = RowInfo("bigrams", s, int(np.argmin(s)), "", int(np.partition(np.array(s) - min(s), 1)[1]))
        else:
            if band:
                route = "first" if r % BAND_ROWS == 0 else ("fused" if prev_open else "two")
                s = band_scores(xr, br, bpp, oa, mut)
            else:
                route = "sticky" if sticky else "row"
                s = row_scores(xr, br, bpp, oa, mut)
            p = ladder(s, st, rb, mut, route)
            prev_open = p.open
            info = RowInfo(route, s, p.winner, p.exit, p.margin)
            if sticky:
                forced = p.winner
        out[r, 0] = info.winner
        out[r, 1:] = filtered(x, b, bpp)[info.winner]
        infos.append(info)
    return out.reshape(-1), infos
