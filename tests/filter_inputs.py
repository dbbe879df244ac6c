"""Rows built to sit on the PNG filter kernels' decision edges, each with the faults (filter_ref mutants) that change
its output.

All constructions are exact and checked with filter_ref when they are built:
  * threshold rows: the best cheap score equals `early` (the ladder ends although a later candidate is lower) or
    `early + 1` (it does not), for Adaptive/MinSum (row_bytes/4 + 1) and AdaptiveFast (row_bytes/8 + 1);
  * Paeth ties: over a zero row Paeth predicts the left byte, so Paeth ties Sub on every row; over a row of 0/128
    steps its inverse does the same with the row above left open (the band kernel's fused route);
  * Up ties: a ramp over the same ramp shifted by its slope ties Sub, Up and Paeth (AdaptiveFast, `up_le`);
  * position rows: AdaptiveFast rows over a zero row where Sub = Up - 1, built from runs of equal pixels (a run of
    value v and n pixels adds n v to None and Up and 2 v to Sub).  The bytes at one named position are a run of 2s
    (their Sub is 0, their Up 2 each), so a kernel that skips those bytes, or reads a wrong left neighbour there,
    lets Up win;
  * Bigrams rows across a 32 KiB segment seam where the seam's bigram decides, found by a seeded search.
Everything is deterministic and cached per process.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

import filter_ref as R


@dataclass
class Row:
    x: np.ndarray
    label: str
    flips: tuple = ()     # mutants the row's output must change under
    strategies: tuple = (R.ADAPTIVE, R.MINSUM, R.FAST)   # ... with these strategies


def threshold_rows(rb, bpp, fast):
    """[(above, Row)]: best == early (flips the `<` and the dropped `+ 1` faults) and best == early + 1"""
    E = R.early_of(R.FAST if fast else R.ADAPTIVE, rb)
    out = []
    for at, flips in ((E, ("fast_lt", "no_plus_one") if fast else ("adaptive_lt", "no_plus_one")), (E + 1, ())):
        x = np.zeros(rb, np.uint8)
        if fast:   # isolated ones (Sub 2 each) and a last byte of 1 (Sub 1); the row above is the same row: Up 0
            k, t = divmod(at, 2)
            pos = [2 * bpp * m for m in range(k)]
            assert pos[-1] < rb - 3 * bpp
            x[pos] = 1
            if t:
                x[rb - 1] = 1
            out.append((x.copy(), Row(x, f"fast sub=={'early' if at == E else 'early+1'}", flips, (R.FAST,))))
        else:      # a run of `at` ones: None = Up = Avg = at, Sub = Paeth = 2 bpp
            x[:at] = 1
            out.append((np.zeros(rb, np.uint8), Row(x, f"adaptive none=={'early' if at == E else 'early+1'}", flips,
                                                    (R.ADAPTIVE, R.MINSUM))))
    return out


def ramp(rb, bpp, slope, shift=0):
    return ((np.arange(rb) // bpp * slope + shift) & 255).astype(np.uint8)


def paeth_tie_zero_above(rb, bpp):
    """a ramp over a zero row: Sub is the best cheap score and Paeth ties it"""
    x = ramp(rb, bpp, 3)
    s = R.scores(x, np.zeros(rb, np.uint8), bpp)
    assert s[R.PAETH] == s[R.SUB] < min(s[R.NONE], s[R.UP], s[R.AVG]), s
    return x


def paeth_tie_open_above(rb, bpp):
    """(above, x): the row above alternates runs of 8 pixels of 0 and 128, so its own ladder stays open (Sub scores
    128 per byte at each step); x is its inverse.  Where the row above is flat Paeth predicts the left byte, and at
    each step the left byte is as far from the upper-left one as the step is high, so Paeth predicts the left byte
    there too: Paeth ties Sub, the best cheap score, on the band kernel's fused route."""
    above = ((np.arange(rb) // bpp // 8) % 2 * 128).astype(np.uint8)
    x = (128 - above.astype(np.int32)).astype(np.uint8)
    s, sa = R.scores(x, above, bpp), R.scores(above, np.zeros(rb, np.uint8), bpp)
    assert s[R.PAETH] == s[R.SUB] < min(s[R.NONE], s[R.UP], s[R.AVG]), s
    assert all(R.ladder(sa, st, rb).open and R.ladder(s, st, rb).open for st in (R.ADAPTIVE, R.FAST))
    return above, x


def up_tie(rb, bpp):
    """(above, x): Sub, Up and Paeth tie, above early (AdaptiveFast keeps Sub; Up on <= would take it)"""
    for s_ in (3, 5, 7, 9):
        x, above = ramp(rb, bpp, s_, s_), ramp(rb, bpp, s_, 0)
        s = R.scores(x, above, bpp)
        if s[R.SUB] == s[R.UP] == s[R.PAETH] > R.early_of(R.FAST, rb):
            return above, x
    raise AssertionError("no ramp ties Up")


def position_row(rb, bpp, zone, flips, oa=0, scorer=R.band_scores):
    """An AdaptiveFast row over a zero row with Sub = Up - 1, open; `zone(x)` writes the bytes of one position
    (runs of 2s whose left neighbours are 2 as well), which must stay clear of the bulk."""
    E = R.early_of(R.FAST, rb)
    x = np.zeros(rb, np.uint8)
    busy = zone(x)                          # byte ranges the bulk must avoid
    ch = bpp - 1 if oa else 0               # with optimize_alpha only alpha bytes are set: no pixel is cleared
    def free(p0, n):                        # pixels p0 .. p0+n-1 and the pixel on each side are clear
        lo, hi = (p0 - 1) * bpp, (p0 + n + 1) * bpp
        return lo >= 0 and hi <= rb - 2 * bpp and all(hi <= a - 8 or lo >= b + 8 for a, b in busy)
    p, need = 0, E + 40                     # runs of two 1-pixels: None += 2, Sub += 2
    def put(n):
        nonlocal p
        while not free(p, n):
            p += 1
            assert p * bpp < rb, "row too short for its bulk"
        x[[(p + k) * bpp + ch for k in range(n)]] = 1
        p += n + 1
    zero = np.zeros(rb, np.uint8)
    s = R.scores(R.zero_alpha(x, oa), zero, bpp)
    for _ in range(max(0, -(-(need - s[R.NONE]) // 2))):
        put(2)
    s = R.scores(R.zero_alpha(x, oa), zero, bpp)
    diff = s[R.UP] - s[R.SUB]
    for _ in range(abs(diff - 1)):          # a run of three moves Up - Sub up by 1, a single pixel down by 1
        put(3 if diff < 1 else 1)
    s = scorer(x, zero, bpp, oa)
    assert s[R.UP] - s[R.SUB] == 1 and s[R.SUB] > E, s
    return x


def run_of_twos(lo, hi, bpp):
    """a zone writer: bytes [lo - bpp, hi) = 2 (the pixel left of the zone too, so the zone's Sub is 0)"""
    def w(x):
        a = max(lo - bpp, 0)
        x[a:hi] = 2
        return [(a, hi + bpp)]
    return w


def lane0_zone(j, bpp):
    """vector start j: its left pixel and first pixel are 2s, the bytes a lane-0 fault would read (j - bpp + 16)
    stay 0, and so does every other lane-0 vector start of the row"""
    def w(x):
        x[j - bpp:j + bpp] = 2
        return [(j - bpp, j + 16 + bpp)] + [(512 * k - 8, 512 * k + 24) for k in range(x.size // 512 + 1)]
    return w


def alpha_zone(j, bpp):
    """the pixel left of vector start j is transparent with colour 2 (optimize_alpha clears it); pixel j is zero"""
    def w(x):
        x[j - bpp:j - 1] = 2
        x[j - 1] = 0
        return [(j - bpp, j + 2 * bpp)]
    return w


BAND_POSITIONS = ("first_pixel", "warp_boundary", "lane1_31", "lane0", "iteration_4096", "trailing", "ragged")
ROW_POSITIONS = ("first_pixel", "segment_last_word", "segment_halo", "ragged")


def band_position(rb, bpp, cls):
    """(zone writer, mutants) for a class of k_png_band's scoring, or None if the row has no such position"""
    full, nv = rb >> 2, rb >> 4
    v = {"warp_boundary": 32, "lane1_31": 37, "lane0": 64, "iteration_4096": 256}.get(cls)
    if cls == "first_pixel":   # the bytes of word 0 right of the first pixel (none when bpp is 4)
        return (run_of_twos(0, 4, bpp), (("drop", 0, 4),)) if bpp < 4 else None
    if v is not None:
        if v >= nv:
            return None
        j = 16 * v
        if v % 32 == 0:
            return lane0_zone(j, bpp), ("lane0_shfl",)
        return run_of_twos(j, j + 4, bpp), (("drop", j, j + 4),)
    if cls == "trailing":
        return (run_of_twos(16 * nv, 4 * full, bpp), ("no_trailing",)) if full > 4 * nv else None
    if cls == "ragged":
        return (run_of_twos(4 * full, rb, bpp), ("no_ragged",)) if rb % 4 else None
    raise KeyError(cls)


def row_position(rb, bpp, cls):
    full = rb >> 2
    if cls == "first_pixel":   # the bytes of word 0 right of the first pixel (none when bpp is 4)
        return (run_of_twos(0, 4, bpp), (("drop", 0, 4),)) if bpp < 4 else None
    if cls == "segment_last_word":
        return run_of_twos(R.SEG - 4, R.SEG, bpp), (("drop", R.SEG - 4, R.SEG),)
    if cls == "segment_halo":   # the first pixel of segment 2 reads its left neighbour from the halo
        return run_of_twos(R.SEG, R.SEG + 4, bpp), (("drop", R.SEG, R.SEG + 4),)
    if cls == "ragged":
        return (run_of_twos(4 * full, rb, bpp), ("pass0_unmasked", ("drop", 4 * full, rb))) if rb % 4 else None
    raise KeyError(cls)


def bigram_seam_row(rb, bpp, seed):
    """a row over a zero row where the bigram straddling the 32 KiB seam decides Bigrams' winner"""
    rng = np.random.default_rng(seed)
    zero = np.zeros(rb, np.uint8)
    vals = np.array([1, 2, 3, 128, 255], np.uint8)
    for _ in range(20000):
        x = zero.copy()
        k = int(rng.integers(2, 6))
        x[rng.integers(R.SEG - 6, min(R.SEG + 6, rb), k)] = rng.choice(vals, k)
        s = R.bigram_scores(x, zero, bpp)
        m = R.bigram_scores(x, zero, bpp, mut=frozenset(["bigram_seam"]))
        if int(np.argmin(s)) != int(np.argmin(m)) and sorted(s)[1] - min(s) <= 1:
            return x
    raise AssertionError("no seam row found")


# ---- images ---------------------------------------------------------------------------------------------------
@dataclass
class Image:
    name: str
    width: int
    height: int
    bpp: int
    rb: int
    data: np.ndarray
    strategies: tuple
    flips: dict            # row index -> (mutants that must change that row, under these strategies)
    oa: int = 0


def _assemble(name, rb, bpp, pieces, strategies, min_height=33, oa=0, width=None):
    """pieces: [(above or None, Row)]; an `above` row goes in just before its row, a zero row separates pieces"""
    rows, flips = [], {}
    for above, row in pieces:
        if above is None:
            above = np.zeros(rb, np.uint8)
        if len(rows) % R.BAND_ROWS == R.BAND_ROWS - 1 and above.any():
            rows.append(np.zeros(rb, np.uint8))   # keep the row and its row above in one band
        rows.append(above)
        flips[len(rows)] = (row.flips, row.strategies)
        rows.append(row.x)
    while len(rows) < min_height:
        rows.append(np.zeros(rb, np.uint8))
    width = width or -(-rb // bpp)
    return Image(name, width, len(rows), bpp, rb, np.concatenate(rows), strategies, flips, oa)


ALL = tuple(range(9))


def band_image(rb, bpp):
    """threshold rows, Paeth ties on the fused and two-phase routes, an Up tie and every band position class"""
    pieces = []
    for fast in (False, True):
        pieces += threshold_rows(rb, bpp, fast)
    x = paeth_tie_zero_above(rb, bpp)
    pieces.append((None, Row(x, "paeth tie, two-phase", ("paeth_le:two",))))
    above, x = paeth_tie_open_above(rb, bpp)
    pieces.append((above, Row(x, "paeth tie, fused", ("paeth_le:fused",))))
    above, x = up_tie(rb, bpp)
    pieces.append((above, Row(x, "up tie", ("up_le",), (R.FAST,))))
    for cls in BAND_POSITIONS:
        p = band_position(rb, bpp, cls)
        if p:
            pieces.append((None, Row(position_row(rb, bpp, p[0], p[1]), cls, p[1], (R.FAST,))))
    img = _assemble(f"band rb={rb} bpp={bpp}", rb, bpp, pieces, ALL)
    # a band's first row: the Paeth tie again at row 16 k
    return img


def band_first_image(rb, bpp):
    """Paeth ties as the first row of each 16-row band (over a zero row)"""
    x = paeth_tie_zero_above(rb, bpp)
    rows = [np.zeros(rb, np.uint8) if r % 16 else x for r in range(48)]
    return Image(f"band-first rb={rb} bpp={bpp}", -(-rb // bpp), 48, bpp, rb, np.concatenate(rows),
                 (R.ADAPTIVE, R.FAST, R.MINSUM), {r: (("paeth_le:two",), (R.ADAPTIVE, R.MINSUM, R.FAST)) for r in (16, 32)})


def row_image(rb, bpp):
    """k_png_filter rows (too long for the band kernel): thresholds, Paeth tie, positions at the segment seams"""
    pieces = []
    for fast in (False, True):
        pieces += threshold_rows(rb, bpp, fast)
    pieces.append((None, Row(paeth_tie_zero_above(rb, bpp), "paeth tie, row", ("paeth_le:row",))))
    for cls in ROW_POSITIONS:
        p = row_position(rb, bpp, cls)
        if p:
            pieces.append((None, Row(position_row(rb, bpp, p[0], p[1], scorer=R.row_scores), cls, p[1],
                                                (R.FAST,))))
    return _assemble(f"row rb={rb} bpp={bpp}", rb, bpp, pieces, (R.ADAPTIVE, R.FAST, R.MINSUM, R.PAETH, R.SUB),
                     min_height=33)


def alpha_image(rb, bpp):
    """optimize_alpha: transparent pixels with colour left of a lane-0 and of a lane-37 vector start"""
    pieces = []
    for v in (37, 64, 256):
        j = 16 * v
        pieces.append((None, Row(position_row(rb, bpp, alpha_zone(j, bpp), ("alpha_x0",), oa=bpp), f"alpha v={v}",
                                 ("alpha_x0",), (R.FAST,))))
    return _assemble(f"alpha rb={rb} bpp={bpp}", rb, bpp, pieces, (R.FAST, R.ADAPTIVE), oa=bpp)


def sticky_image(rb, bpp, height):
    """AdaptiveFast on a short image: row 0 is a threshold row or a Paeth tie and decides every row"""
    out = []
    (_, t), = [p for p in threshold_rows(rb, bpp, True) if p[1].flips][:1]
    for name, x0, flips in (("sticky threshold", t.x, ("fast_lt",)), ("sticky paeth tie", paeth_tie_zero_above(rb, bpp),
                                                                        ("paeth_le:row",))):
        rows = [x0] + [ramp(rb, bpp, 1 + r) for r in range(1, height)]
        out.append(Image(f"{name} h={height} bpp={bpp}", -(-rb // bpp), height, bpp, rb, np.concatenate(rows),
                         (R.FAST,), {0: (flips, (R.FAST,))}))
    return out


def bigram_image(rb, bpp):
    x = bigram_seam_row(rb, bpp, rb + bpp)
    rows = [x, np.zeros(rb, np.uint8), x]
    return Image(f"bigrams rb={rb} bpp={bpp}", -(-rb // bpp), 3, bpp, rb, np.concatenate(rows), (R.BIGRAMS,),
                 {0: (("bigram_seam",), (R.BIGRAMS,)), 2: (("bigram_seam",), (R.BIGRAMS,))})


BAND_RBS = (4133, 4138, 4143, 4144)   # trailing words 1-3 and 0, ragged bytes 1-3 and 0


@functools.lru_cache(maxsize=None)
def band_images():
    return [band_image(rb, bpp) for bpp in (1, 2, 3, 4) for rb in BAND_RBS] + \
           [band_first_image(4143, bpp) for bpp in (1, 2, 3, 4)]


@functools.lru_cache(maxsize=None)
def row_images():
    return [row_image(rb, bpp) for bpp in (1, 2, 3, 4) for rb in (68225,)]


@functools.lru_cache(maxsize=None)
def longest_band_image():
    return band_image(68224, 4)


@functools.lru_cache(maxsize=None)
def alpha_images():
    return [alpha_image(4144, 2), alpha_image(4144, 4)]


@functools.lru_cache(maxsize=None)
def sticky_images():
    return [im for bpp in (1, 4) for h in (5, 32) for im in sticky_image(4144, bpp, h)]


@functools.lru_cache(maxsize=None)
def bigram_images():
    return [bigram_image(rb, bpp) for bpp in (1, 3, 4) for rb in (32769, 40000)]
