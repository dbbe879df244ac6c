"""An independent restatement of pixo's lossy PNG path (src/png/mod.rs:1296-1762) in numpy and Python integers,
written from pixo's semantics rather than from oracle/png_quantize.*, with a model of the routes the CUDA stage
(png_quantize.cu, png_host.cpp) takes and single-fault mutants of that code.

  distance(c, p)            perceptual_distance_sq (redmean, truncated by >> 8, alpha unweighted)
  nearest(c, pal, shape)    the first nearest entry as nearest_seq (one thread, k-means and the 6-6-6 table) or
                            nearest_warp (32 lanes split the entries, min of (d << 8) | i) finds it, with the tie set
  table_index / map_pixels  PaletteLut and the map: the table, the translucent search, the early out's exact hit
                            and its search on a miss
  dither                    Floyd-Steinberg in the kernel's integer form: E16 = 7 e(x-1, y) + 1 e(x-1, y-1)
                            + 5 e(x, y-1) + 3 e(x+1, y-1), adj = clamp(16 v + E16, 0, 4080) >> 4
  kmeans / median_cut       refine_palette_kmeans (u64 floor centroids, an entry with no members keeps its colour)
                            and median_cut_palette
  decision / histogram      should_quantize_auto and quantize_image's histogram, with their strides and sample counts
  batch_samples             the device sampler: 64-bit keys image << 33 | set << 32 | colour, a stable radix sort on
                            bits [0, end_bit), run-length counts, each run credited to the image its key names
  quantize                  the whole stage for one image: decision, palette, indices, the route and tie set of every
                            pixel, and what the case exercised (ties, empty entries, split events, dither extremes)

Every pixel's route is one of ROUTES.  `mut` is a set of MUTANTS, each restating one fault in the kernels or the host
code; EQUIVALENT names faults that cannot change any output, and why.
"""
from __future__ import annotations

import dataclasses

import numpy as np

ROUTES = ("table", "warp", "early", "early-miss", "dither-table", "dither-warp")

MUTANTS = {
    "seq_last": "nearest_seq keeps the last minimum (k-means and the table)",
    "warp_last": "each lane of nearest_warp keeps the last minimum of its entries",
    "warp_lane": "nearest_warp reduces on distance alone and takes the lowest lane's entry",
    "dist_exact": "redmean compared without the >> 8 truncation",
    "rm_ceil": "r_mean rounded up",
    "cell_plain": "table cell colour r6 << 2",
    "cell_mid": "table cell colour r6 << 2 | 2",
    "table_alpha": "translucent pixels take the table",
    "km_round": "k-means centroids rounded to nearest",
    "km_empty_zero": "a k-means entry with no members zeroed",
    "km_one_pass": "one k-means pass",
    "km_unweighted": "k-means ignores the histogram counts",
    "box_first_max": "median cut splits the first box of the largest score",
    "channel_ge": "median cut: a later channel wins on a tied score",
    "split_gt": "median cut splits at acc > total / 2",
    "auto_ge": "Auto quantises at unique >= m",
    "auto_lt": "Auto quantises only below 32 m",
    "early_lt": "early out only below m histogram colours",
    "trunc_ge": "refusal at 8192 histogram colours or more",
    "nd_floor": "decision sample count npix / stride",
    "nh_floor": "histogram sample count npix / stride",
    "pack8": "dither errors packed in 8-bit fields",
    "err_unclamped": "dither error taken from the unclamped sum",
    "err_src": "dither error taken from the source value",
    "w13": "the 1/16 and 3/16 dither weights swapped",
    "seam_zero": "the first row of each 32-row group receives no error from above",
}

EQUIVALENT = {
    "early_search": "any fault in the early out's binary search: a miss falls back to the nearest search, and distance 0 "
                    "holds only for identical colours, so the search finds the entry the binary search missed",
    "clamp_after_shift": "clamp((16 v + E16) >> 4, 0, 255) equals clamp(16 v + E16, 0, 4080) >> 4 for every integer",
    "sort_bits_38": "the radix sort is stable and the samples go in image-major order, so keys that agree on bits 0-37 "
                    "keep image i's before image i+32's; every run holds one full key, and the host credits runs by the "
                    "image bits of the key, so each image's colours, counts and key order are unchanged",
}

DECISION_CAP, HISTOGRAM_CAP, MAX_HIST_COLORS = 20000, 50000, 8192


class Refused(Exception):
    """More than 8192 histogram colours and no palette: pixo's truncation case, which the library refuses."""


def keys_of(px: np.ndarray) -> np.ndarray:
    px = np.asarray(px, np.uint32)
    return (px[:, 0] << 24) | (px[:, 1] << 16) | (px[:, 2] << 8) | px[:, 3]


def rgba_of(keys) -> np.ndarray:
    k = np.asarray(keys, np.uint64).astype(np.uint32)
    return np.stack([k >> 24, (k >> 16) & 255, (k >> 8) & 255, k & 255], 1).astype(np.uint8)


def pixels(data, ct: int) -> np.ndarray:
    """(npix, 4) RGBA, alpha 255 for RGB."""
    px = np.asarray(data, np.uint8).reshape(-1, ct + 1)
    if ct == 2:
        px = np.concatenate([px, np.full((len(px), 1), 255, np.uint8)], 1)
    return px


# ---- distance and the nearest search -----------------------------------------------------------------
def distance(c, p, mut=frozenset()) -> np.ndarray:
    """perceptual_distance_sq of colours c (k, 4) to entries p (n, 4) as a (k, n) int64 matrix.  Under dist_exact the
    redmean sum is compared untruncated (alpha on the same scale)."""
    c = np.asarray(c, np.int64)[:, None, :]
    p = np.asarray(p, np.int64)[None, :, :]
    d = c - p
    s = c[..., 0] + p[..., 0]
    rm = (s + 1) >> 1 if "rm_ceil" in mut else s >> 1
    w = (512 + rm) * d[..., 0] ** 2 + 1024 * d[..., 1] ** 2 + (767 - rm) * d[..., 2] ** 2
    if "dist_exact" in mut:
        return w + 256 * d[..., 3] ** 2
    return (w >> 8) + d[..., 3] ** 2


def nearest(c, pal, shape: str, mut=frozenset()):
    """(indices, tie sets) of colours c (k, 4) among pal (n, 4); shape "seq" or "warp".  A tie set is the tuple of all
    entries at the minimum distance."""
    D = distance(c, pal, mut)
    n = D.shape[1]
    dmin = D.min(1)
    tie = D == dmin[:, None]
    first = tie.argmax(1)
    last = n - 1 - tie[:, ::-1].argmax(1)
    if shape == "seq":
        idx = last if "seq_last" in mut else first
    elif not ({"warp_last", "warp_lane"} & mut):
        idx = first
    else:
        # lane l holds entries l, l + 32, ...; each lane's pick, then the reduction
        big = np.iinfo(np.int64).max
        lane_d = np.full((len(D), 32), big, np.int64)
        lane_pick = np.zeros((len(D), 32), np.int64)
        for lane in range(min(n, 32)):
            ent = np.arange(lane, n, 32)
            Dl = D[:, ent]
            lane_d[:, lane] = Dl.min(1)
            t = Dl == lane_d[:, lane][:, None]
            lane_pick[:, lane] = ent[len(ent) - 1 - t[:, ::-1].argmax(1)] if "warp_last" in mut else ent[t.argmax(1)]
        if "warp_lane" in mut:       # distance alone: the lowest lane at the minimum
            idx = lane_pick[np.arange(len(D)), (lane_d == dmin[:, None]).argmax(1)]
        else:                        # (d << 8) | i: the lowest lane pick at the minimum
            idx = np.where(lane_d == dmin[:, None], lane_pick, big).min(1)
    ties = [tuple(np.flatnonzero(r)) for r in tie]
    return idx.astype(np.int64), ties


# ---- PaletteLut and the map --------------------------------------------------------------------------
def cell_colour(cells, mut=frozenset()) -> np.ndarray:
    """The colour PaletteLut::new searches for 6-6-6 cells (k,) -> (k, 4)."""
    cells = np.asarray(cells, np.int64)
    six = np.stack([cells >> 12, (cells >> 6) & 63, cells & 63], 1)
    if "cell_plain" in mut:
        v = six << 2
    elif "cell_mid" in mut:
        v = (six << 2) | 2
    else:
        v = (six << 2) | (six >> 4)
    return np.concatenate([v, np.full((len(v), 1), 255)], 1)


def cell_of(px) -> np.ndarray:
    px = np.asarray(px, np.int64)
    return ((px[:, 0] >> 2) << 12) | ((px[:, 1] >> 2) << 6) | (px[:, 2] >> 2)


class Table:
    """The 6-6-6 table, searched lazily: only the cells a case reaches."""

    def __init__(self, pal, mut=frozenset()):
        self.pal, self.mut, self.cache = pal, mut, {}

    def lookup(self, cells):
        cells = np.asarray(cells, np.int64)
        new = np.setdiff1d(np.unique(cells), np.fromiter(self.cache, np.int64, len(self.cache)))
        if len(new):
            idx, ties = nearest(cell_colour(new, self.mut), self.pal, "seq", self.mut)
            self.cache.update(zip(new.tolist(), zip(idx.tolist(), ties)))
        got = [self.cache[c] for c in cells.tolist()]
        return np.array([g[0] for g in got], np.int64), [g[1] for g in got]


def table_entries(pal, mut=frozenset()) -> np.ndarray:
    """The whole table (262 144 cells) of pal."""
    return Table(pal, mut).lookup(np.arange(1 << 18))[0]


def map_pixels(px, pal, early: bool, mut=frozenset(), table=None):
    """The plain map (early False: the table for opaque pixels, the warp search otherwise) or the early out (pal is
    the key-ordered histogram: an exact hit, the warp search on a miss).  Returns (indices, routes, ties)."""
    px = np.asarray(px, np.uint8)
    n = len(px)
    idx = np.zeros(n, np.int64)
    routes = np.empty(n, object)
    ties: list = [()] * n
    if early:
        pk, k = keys_of(pal), keys_of(px)
        hit = np.minimum(np.searchsorted(pk, k), len(pk) - 1)
        search = pk[hit] != k
        idx[~search] = hit[~search]
        routes[~search] = "early"
        routes[search] = "early-miss"
    else:
        search = (px[:, 3] != 255) & ("table_alpha" not in mut)
        routes[~search] = "table"
        routes[search] = "warp"
        tab = table or Table(pal, mut)
        on = np.flatnonzero(~search)
        if len(on):
            i, t = tab.lookup(cell_of(px[on]))
            idx[on] = i
            for k, tt in zip(on.tolist(), t):
                ties[k] = tt
    on = np.flatnonzero(search)
    if len(on):
        cols, inv = np.unique(px[on], axis=0, return_inverse=True)
        i, t = nearest(cols, pal, "warp", mut)
        idx[on] = i[inv.reshape(-1)]
        for k, u in zip(on.tolist(), inv.reshape(-1).tolist()):
            ties[k] = t[u]
    return idx, routes, ties


@dataclasses.dataclass
class DitherStats:
    max_err: int = 0          # largest |error| carried
    low: int = 0              # pixels where 16 v + E16 < 0
    high: int = 0             # pixels where 16 v + E16 > 4080


def _wrap(e: int, bits: int) -> int:
    m = 1 << bits
    e &= m - 1
    return e - m if e >= m >> 1 else e


def dither(px, w: int, h: int, pal, mut=frozenset(), table=None):
    """Floyd-Steinberg as k_quant_dither computes it.  Returns (indices, routes, ties, DitherStats)."""
    px = np.asarray(px, np.int64).reshape(h, w, 4).tolist()
    pal64 = np.asarray(pal, np.int64).tolist()
    tab = table or Table(pal, mut)
    bits = 8 if "pack8" in mut else 10
    wt = (7, 3, 5, 1) if "w13" in mut else (7, 1, 5, 3)   # e(x-1, y), e(x-1, y-1), e(x, y-1), e(x+1, y-1)
    idx = np.zeros((h, w), np.int64)
    routes = np.empty(h * w, object)
    ties: list = [()] * (h * w)
    st = DitherStats()
    above = [[0, 0, 0] for _ in range(w)]
    zero = [0, 0, 0]
    for y in range(h):
        row = [None] * w
        cut = y % 32 == 0 and "seam_zero" in mut
        for x in range(w):
            left = row[x - 1] if x else zero
            ul = zero if cut or x == 0 else above[x - 1]
            up = zero if cut else above[x]
            ur = zero if cut or x + 1 >= w else above[x + 1]
            v = px[y][x]
            adj, raw = [0, 0, 0], [0, 0, 0]
            for ch in range(3):
                e16 = wt[0] * left[ch] + wt[1] * ul[ch] + wt[2] * up[ch] + wt[3] * ur[ch]
                s = 16 * v[ch] + e16
                st.low += s < 0
                st.high += s > 4080
                raw[ch] = s >> 4
                adj[ch] = min(max(s, 0), 4080) >> 4
            k = y * w + x
            if v[3] == 255 or "table_alpha" in mut:
                cell = ((adj[0] >> 2) << 12) | ((adj[1] >> 2) << 6) | (adj[2] >> 2)
                if cell not in tab.cache:
                    tab.lookup([cell])
                i, ties[k] = tab.cache[cell]
                routes[k] = "dither-table"
            else:
                i, t = nearest(np.array([adj + [v[3]]], np.int64), pal, "warp", mut)
                i, ties[k] = int(i[0]), t[0]
                routes[k] = "dither-warp"
            idx[y, x] = i
            base = v[:3] if "err_src" in mut else raw if "err_unclamped" in mut else adj
            e = [base[ch] - pal64[i][ch] for ch in range(3)]
            st.max_err = max(st.max_err, max(abs(q) for q in e))
            row[x] = [_wrap(q, bits) for q in e]
        above = row
    return idx.reshape(-1), routes, ties, st


# ---- k-means and median cut ----------------------------------------------------------------------------
@dataclasses.dataclass
class KmeansInfo:
    tied: list            # per pass: indices of histogram colours with more than one nearest entry
    empty: list           # per pass: entries with no members


def kmeans(pal, keys, counts, mut=frozenset()):
    """refine_palette_kmeans: two passes; returns (palette, KmeansInfo)."""
    pal = np.asarray(pal, np.int64).copy()
    cols = rgba_of(keys).astype(np.int64)
    wts = np.ones(len(cols), object) if "km_unweighted" in mut else np.asarray(counts, np.uint64).astype(object)
    info = KmeansInfo([], [])
    for _ in range(1 if "km_one_pass" in mut else 2):
        best, ties = nearest(cols, pal, "seq", mut)
        info.tied.append([k for k, t in enumerate(ties) if len(t) > 1])
        empty = []
        for i in range(len(pal)):
            m = best == i
            t = int(wts[m].sum()) if m.any() else 0
            if not t:
                empty.append(i)
                if "km_empty_zero" in mut:
                    pal[i] = 0
                continue
            sums = [int((cols[m, ch].astype(object) * wts[m]).sum()) for ch in range(4)]
            pal[i] = [(s + t // 2) // t if "km_round" in mut else s // t for s in sums]
        info.empty.append(empty)
    return pal.astype(np.uint8), info


@dataclasses.dataclass
class CutInfo:
    box_tie: int = 0        # splits where more than one box had the largest score
    channel_tie: int = 0    # splits whose box had a later channel tied with the chosen one
    split_eq: int = 0       # splits where acc equalled total / 2 at the split
    clamped: int = 0       # splits moved back by the len - 2 clamp


def _range(box, mut):
    c = np.array([b[0] for b in box], np.int64)
    r = c.max(0) - c.min(0)
    sc = [int(r[0]) * 2, int(r[1]) * 4, int(r[2]), int(r[3]) * 3]
    ch, best = 0, sc[0]
    for k in (1, 2, 3):
        if sc[k] > best or ("channel_ge" in mut and sc[k] == best):
            ch, best = k, sc[k]
    tied = any(sc[k] == best for k in range(4) if k != ch)
    return ch, best, tied


def median_cut(keys, counts, m: int, mut=frozenset()):
    """median_cut_palette's boxes (before k-means): (box means in box order, CutInfo)."""
    info = CutInfo()
    cols = [(tuple(int(v) for v in c), int(n)) for c, n in zip(rgba_of(keys), counts)]
    if not cols:
        return np.array([[0, 0, 0, 255]], np.uint8), info
    boxes = [(cols, _range(cols, mut))]
    while len(boxes) < m:
        scores = [b[1][1] for b in boxes]
        top = max(scores)
        at = [i for i, s in enumerate(scores) if s == top]
        idx = at[0] if "box_first_max" in mut else at[-1]
        box, (ch, _, ctie) = boxes[idx]
        if len(box) <= 1:
            break
        info.box_tie += len(at) > 1
        info.channel_tie += ctie
        boxes.pop(idx)
        box = sorted(box, key=lambda c: c[0][ch])
        total = sum(n for _, n in box) & 0xFFFFFFFF
        acc, split = 0, 0
        for i, (_, n) in enumerate(box):
            acc = (acc + n) & 0xFFFFFFFF
            if acc > total // 2 if "split_gt" in mut else acc >= total // 2:
                split = i
                info.split_eq += acc == total // 2
                break
        if split > len(box) - 2:
            info.clamped += 1
            split = len(box) - 2
        for part in (box[:split + 1], box[split + 1:]):
            boxes.append((part, _range(part, mut)))
    pal = []
    for box, _ in boxes:
        t = sum(n for _, n in box)
        pal.append([sum(c[ch] * n for c, n in box) // t for ch in range(4)] if t else [0, 0, 0, 255])
    return np.array(pal, np.uint8), info


# ---- decision and samplers -----------------------------------------------------------------------------
def sample_positions(npix: int, cap: int, floor: bool = False) -> np.ndarray:
    """Pixel indices a sampler reads: stride max(npix / cap, 1), ceil(npix / stride) samples (floor under the
    nd_floor / nh_floor faults)."""
    stride = max(npix // cap, 1)
    n = npix // stride if floor else -(-npix // stride)
    return np.arange(n, dtype=np.int64) * stride


def decision_unique(px, mut=frozenset()) -> int:
    return len(np.unique(keys_of(px[sample_positions(len(px), DECISION_CAP, "nd_floor" in mut)])))


def auto_quantises(unique: int, m: int, mut=frozenset()) -> bool:
    lo = unique >= m if "auto_ge" in mut else unique > m
    hi = unique < 32 * m if "auto_lt" in mut else unique <= 32 * m
    return lo and hi


def histogram(px, mut=frozenset()):
    """(keys in key order, counts): each sample counts `stride`, saturating at 2^32 - 1."""
    stride = max(len(px) // HISTOGRAM_CAP, 1)
    k, n = np.unique(keys_of(px[sample_positions(len(px), HISTOGRAM_CAP, "nh_floor" in mut)]), return_counts=True)
    return k.astype(np.uint32), np.minimum(n.astype(np.uint64) * stride, 0xFFFFFFFF)


def batch_samples(frames, ct: int, end_bit: int = 39, chunk: int = 64):
    """The device sampler over a batch: per image, (decision unique count, histogram keys, counts), as the host reads
    them back from a stable radix sort on key bits [0, end_bit) and a run-length encode of the sorted keys."""
    out = []
    for i0 in range(0, len(frames), chunk):
        ks = []
        for j, f in enumerate(frames[i0:i0 + chunk]):
            px = pixels(f, ct)
            for s, cap in ((0, DECISION_CAP), (1, HISTOGRAM_CAP)):
                col = keys_of(px[sample_positions(len(px), cap)]).astype(np.uint64)
                ks.append((np.uint64(j) << np.uint64(33)) | (np.uint64(s) << np.uint64(32)) | col)
        k = np.concatenate(ks)
        k = k[np.argsort(k & np.uint64((1 << end_bit) - 1), kind="stable")]
        starts = np.flatnonzero(np.concatenate([[True], k[1:] != k[:-1]]))
        runs = np.diff(np.concatenate([starts, [len(k)]]))
        nb = min(chunk, len(frames) - i0)
        uniq = [0] * nb
        hk = [[] for _ in range(nb)]
        hn = [[] for _ in range(nb)]
        for key, cnt in zip(k[starts].tolist(), runs.tolist()):
            img = key >> 33
            if not (key >> 32) & 1:
                uniq[img] += 1
            else:
                hk[img].append(key & 0xFFFFFFFF)
                hn[img].append(cnt)
        for j in range(nb):
            npix = len(pixels(frames[i0 + j], ct))
            out.append((uniq[j], hk[j], [c * max(npix // HISTOGRAM_CAP, 1) for c in hn[j]]))
    return out


# ---- the stage -----------------------------------------------------------------------------------------
@dataclasses.dataclass
class Result:
    kind: str                       # "lossless", "early", "lut" (median cut) or "given" (the caller's palette)
    unique: int = 0                 # decision sample's distinct colours (Auto)
    hist: int = 0                   # histogram colours
    palette: np.ndarray | None = None
    indices: np.ndarray | None = None
    routes: np.ndarray | None = None
    ties: list | None = None
    kmeans: KmeansInfo | None = None
    cut: CutInfo | None = None
    dither: DitherStats | None = None

    def key(self):
        """What the stage hands the filter: comparable across mutants."""
        if self.kind == "lossless":
            return ("lossless",)
        return (self.kind, self.palette.tobytes(), self.indices.astype(np.uint8).tobytes())


def quantize(data, w: int, h: int, ct: int, max_colors: int, mode: str, dithering: bool, palette=None,
             mut=frozenset(), map_pixels_too: bool = True) -> Result:
    """encode_into's quantisation branch for one RGB (ct 2) or RGBA (ct 3) image; mode "auto" or "force".  Raises
    Refused in the truncation case."""
    mut = frozenset(mut)
    m = min(int(max_colors), 256)
    px = pixels(data, ct)
    r = Result("lossless")
    if mode == "auto":
        r.unique = decision_unique(px, mut)
        if not auto_quantises(r.unique, m, mut):
            return r
    if palette is not None:
        r.kind, pal = "given", np.asarray(palette, np.uint8).reshape(-1, 4)
    else:
        keys, counts = histogram(px, mut)
        r.hist = len(keys)
        if len(keys) >= MAX_HIST_COLORS if "trunc_ge" in mut else len(keys) > MAX_HIST_COLORS:
            raise Refused(f"{len(keys)} histogram colours exceed 8192")
        if len(keys) < m if "early_lt" in mut else len(keys) <= m:
            r.kind, pal = "early", rgba_of(keys)
        else:
            mc, r.cut = median_cut(keys, counts, m, mut)
            pal, r.kmeans = kmeans(mc, keys, counts, mut)
            r.kind = "lut"
    r.palette = pal
    if not map_pixels_too:
        return r
    if r.kind != "early" and dithering:
        r.indices, r.routes, r.ties, r.dither = dither(px, w, h, pal, mut)
    else:
        r.indices, r.routes, r.ties = map_pixels(px, pal, r.kind == "early", mut)
    return r


def trimmed_trns(pal) -> bytes | None:
    a = np.asarray(pal, np.uint8)[:, 3]
    nz = np.flatnonzero(a != 255)
    return None if len(nz) == 0 else a[:nz[-1] + 1].tobytes()
