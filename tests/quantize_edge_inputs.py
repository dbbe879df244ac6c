"""Seeded, deterministic inputs that sit on the PNG quantiser's decisions (numpy only).  Each Case is one image and the
options it is quantised with; `targets` names the quantize_ref mutants whose output it must change, and `expect` what
it is built to exercise.

  tie_cases          caller palettes under Force with the None filter, so the index rows are the output: a colour at
                     exactly the same distance from two entries i < j (exact ties: green- and alpha-symmetric pairs and
                     duplicated entries; truncation ties: red + 1 against blue + 1, which redmean's >> 8 makes equal;
                     pairs found by search whose weighted sums differ but floor to the same value, and near misses one
                     apart), placed in one lane of nearest_warp (j = i + 32, i + 64), with i in a higher lane than j
                     (5, 33), adjacent, and first and last, in palettes of 1 to 256 entries; searched on the table, by
                     translucent pixels (a = 0, 1, 254) with every lane, lane 0 or lane 31 of a warp searching, and in
                     a partial last warp
  sweep_cases        one truncation tie for every r <= 254 (translucent) and every cell r6 <= 62 (table); the cell
                     colours themselves against neighbours r6 << 2 and r6 << 2 | 2
  early_cases        early-out misses (100 000+ pixels: the stride-2 histogram skips the odd pixels), tied between two
                     histogram colours whose key order places them in one lane, in crossed lanes or adjacent
  kmeans_cases       histograms found by search: a tie between two median-cut entries in k-means pass 1 and in pass
                     2 that changes the palette, an entry emptied in pass 1, floor against round, counts, one pass
  cut_cases          median cut: two boxes of equal best score, tied channel scores, acc == total / 2, the len - 2 clamp
  decision_cases     Auto at unique = m, m + 1, 32 m, 32 m + 1; the decision and histogram samplers' strides and last
                     samples; early out at m against m + 1; 8 192 against 8 193 histogram colours
  batch_frames       frames of one batch whose decisions alternate, for batches across the 64-image sort chunk
  dither_cases       one- and two-entry palettes far from the image: errors of 255, 16 v + E16 below 0 and above 4080,
                     first and last columns, heights around the 32-row groups, translucent pixels tied after adjustment
  all_cells / all_colours   every 6-6-6 cell colour once (512 x 512) and every opaque colour (4096 x 4096), RGB
"""
from __future__ import annotations

import dataclasses

import numpy as np

import quantize_ref as R


@dataclasses.dataclass
class Case:
    name: str
    w: int
    h: int
    ct: int                              # 2 RGB, 3 RGBA
    data: np.ndarray                     # flat uint8
    mode: str = "force"
    m: int = 256
    dither: bool = False
    palette: np.ndarray | None = None
    targets: tuple = ()
    expect: dict = dataclasses.field(default_factory=dict)
    keys: dict = dataclasses.field(default_factory=dict)     # mutant -> output, where already computed

    def run(self, mut=frozenset(), **kw):
        return R.quantize(self.data, self.w, self.h, self.ct, self.m, self.mode, self.dither, self.palette, mut, **kw)


def expand(v6: int) -> int:
    return (v6 << 2) | (v6 >> 4)


SIZES = (2, 31, 32, 33, 64, 255, 256)
TIE_KINDS = ("trunc", "green", "alpha", "dup", "floor")


def _pair(kind: str, t):
    """Two entries at equal distance from colour t (r, g, b, a), or None where the kind does not fit t."""
    r, g, b, a = t
    if kind == "trunc":
        return (r + 1, g, b, a), (r, g, b + 1, a)
    if kind == "green":
        return (r, g - 1, b, a), (r, g + 1, b, a)
    if kind == "alpha":
        return None if a in (0, 255) else ((r, g, b, a - 1), (r, g, b, a + 1))
    if kind == "dup":
        return (r, g, b + 1, a), (r, g, b + 1, a)
    if kind == "floor":     # weighted sums that differ but floor alike: found by search
        return FLOOR_PAIR[0](t)
    raise ValueError(kind)


def _floor_search():
    """Offsets (dr, db) and (dr', db') from a colour of r = 100 whose redmean sums differ and floor to the same
    value, and a near miss: floors one apart."""
    t = np.array([[100, 100, 100, 255]])
    offs = [(dr, 0, db, 0) for dr in range(-3, 4) for db in range(-3, 4) if (dr, db) != (0, 0)]
    p = t + np.array(offs)
    exact = R.distance(t, p, frozenset(["dist_exact"]))[0]
    d = R.distance(t, p)[0]
    for i in range(len(offs)):
        for j in range(len(offs)):
            if d[i] == d[j] and exact[j] < exact[i] and d[i] == d.min():
                return offs[i], offs[j]
    raise AssertionError("no floor tie")


_FI, _FJ = _floor_search()
FLOOR_PAIR = [lambda t: (tuple(int(t[k]) + _FI[k] for k in range(4)), tuple(int(t[k]) + _FJ[k] for k in range(4)))]


def _fillers(rng, n: int, t, a: int = 255) -> np.ndarray:
    """n colours far from t: green at least 96 away (a redmean distance above 36 000)."""
    g = (t[1] + 96 + rng.integers(0, 64, n)) % 256
    return np.stack([rng.integers(0, 256, n), g, rng.integers(0, 256, n), np.full(n, a)], 1).astype(np.uint8)


def placements(n: int):
    """(i, j, name) pairs for an n-entry palette."""
    out = [(0, n - 1, "first-last")]
    if n > 33:
        out.append((5, 33, "cross-lane"))
    for i in (0, n - 33):
        if n > 32 and i >= 0 and (i, i + 32) not in [(p[0], p[1]) for p in out]:
            out.append((i, i + 32, "same-lane"))
    if n > 64:
        out.append((n - 65, n - 1, "same-lane-64"))
    if n > 2:
        out.append((n // 2, n // 2 + 1, "adjacent"))
    return out


def warp_targets(i: int, j: int):
    """The nearest_warp faults a tie between i < j exposes."""
    t = []
    if i % 32 == j % 32:
        t.append("warp_last")
    if i % 32 > j % 32:
        t.append("warp_lane")
    return t


def _also(c: Case, candidates) -> Case:
    """Add to c's targets the candidate mutants whose output it changes.  Used where whether a fault shows depends on
    which way it breaks a tie (dist_exact) or on the palette around it (table_alpha, the dither faults)."""
    base = c.run().key()
    for m in candidates:
        if m not in c.targets:
            c.keys[m] = c.run(frozenset([m])).key()
    c.targets = tuple(c.targets) + tuple(m for m in candidates if m in c.keys and c.keys[m] != base)
    return c


def _layout(tie, other, w=131, h=3):
    """393 pixels: warp 0 all tie pixels, warp 1 only lane 0 (pixels 128-131), warp 2 only lane 31 (380-383), and the
    partial warp 3 (9 pixels) all tie pixels; the rest `other`."""
    px = np.tile(np.array(other, np.uint8), (w * h, 1))
    for s in (slice(0, 128), slice(128, 132), slice(380, 384), slice(384, w * h)):
        px[s] = tie
    return px


def tie_cases():
    rng = np.random.default_rng(1)
    cases = []
    t_tab = (expand(40), expand(20), expand(33), 255)          # a cell colour; r6 >= 16 so cell_plain moves it
    for kind in TIE_KINDS:
        for route in ("table", "warp"):
            for n in SIZES:
                for p, (i, j, where) in enumerate(placements(n)):
                    # translucent pixels take a = 0, 1 and 254 in turn (the alpha pair needs 1 <= a <= 254)
                    a = 255 if route == "table" else (1, 254, 0)[(p + n) % (2 if kind == "alpha" else 3)]
                    t = t_tab[:3] + (a,)
                    pr = _pair(kind, t)
                    if pr is None:
                        continue
                    pal = _fillers(rng, n, t)
                    pal[i], pal[j] = pr
                    far = pal[(j + 1) % n] if n > 2 else (t[0], (t[1] + 128) % 256, t[2], 255)
                    ct = 3 if route == "warp" else 2 + (n % 2)
                    data = _layout(t, far)
                    tg = ["seq_last"] if route == "table" else warp_targets(i, j)
                    cases.append(_also(Case(f"tie-{kind}-{route}-a{a}-n{n}-{where}-{i}-{j}", 131, 3, ct,
                                      data[:, :ct + 1].reshape(-1).copy(), palette=pal, targets=tuple(tg),
                                      expect={"tie": (i, j), "route": route, "n": n, "kind": kind,
                                              "where": where}), ("dist_exact", "table_alpha")))
    # a single entry: every pixel maps to it on both routes
    t = t_tab
    cases.append(Case("tie-n1", 131, 3, 3, _layout(t[:3] + (1,), t).reshape(-1).copy(),
                      palette=np.array([t], np.uint8), expect={"n": 1}))
    # near misses: entries 5 and 37 one apart after the floor, the later one closer and then the earlier one
    base = np.array([100, 100, 100, 255])
    offs = np.array([(dr, dg, db, 0) for dr in range(-3, 4) for dg in range(-1, 2) for db in range(-3, 4)])
    d = R.distance(base[None], base + offs)[0]
    for name, sign in (("miss-later", 1), ("miss-earlier", -1)):
        a, b = next((a, b) for a in range(len(offs)) for b in range(len(offs)) if d[a] > 0 and d[a] == d[b] + sign)
        pal = _fillers(rng, 40, base)
        pal[5], pal[37] = base + offs[a], base + offs[b]
        cases.append(Case(f"tie-{name}", 131, 3, 3, _layout(base, pal[0]).reshape(-1).copy(), palette=pal,
                          expect={"miss": (5, 37), "n": 40}))
    return cases


def sweep_cases():
    """One truncation tie per r <= 254: translucent colours (r, g(r), 100, 254) with pairs at (k, k + 32) of each
    64-entry block, every lane searching a different colour; and every cell r6 <= 62 on the table, pairs adjacent.
    Then the cell colours against entries at r6 << 2 and r6 << 2 | 2 (cell_plain and cell_mid)."""
    cases = []
    for r0 in (0, 128):
        rs = [r for r in range(r0, min(r0 + 128, 255))]
        pal = np.zeros((256, 4), np.uint8)
        px = []
        for k, r in enumerate(rs):
            t = (r, 2 * (k % 128), 100, 254)
            i = (k // 32) * 64 + k % 32
            pal[i], pal[i + 32] = _pair("trunc", t)
            px.append(t)
        px = np.resize(np.array(px, np.uint8), (512, 4))
        # dist_exact turns red + 1 vs blue + 1 toward blue (entry j) only where 512 + r > 767 - r
        cases.append(Case(f"sweep-warp-r{r0}", 128, 4, 3, px.reshape(-1).copy(), palette=pal,
                          targets=("warp_last",) + (("dist_exact",) if r0 else ()), expect={"route": "warp", "rs": rs}))
    pal, px = np.zeros((126, 4), np.uint8), []
    for r6 in range(63):
        t = (expand(r6), expand(r6 % 32 * 2), expand(17), 255)
        pal[2 * r6], pal[2 * r6 + 1] = _pair("trunc", t)
        px.append(t)
    px = np.array(px, np.uint8)
    cases.append(Case("sweep-table", 63, 1, 2, px[:, :3].reshape(-1).copy(), palette=pal,
                      targets=("seq_last", "dist_exact"), expect={"route": "table"}))
    # cell colours: entry 2k the cell colour, entry 2k+1 where a wrong expansion lands
    for mut, shift in (("cell_plain", lambda v: v << 2), ("cell_mid", lambda v: (v << 2) | 2)):
        pal, px = [], []
        for v in range(64):
            c = (expand(v), expand(63 - v), expand((v * 7) % 64), 255)
            wrong = (shift(v), shift(63 - v), shift((v * 7) % 64), 255)
            if wrong == c:
                continue
            px.append(c)
            pal += [c, wrong]
        pal = np.array(pal[:256], np.uint8)
        px = np.array(px[:len(pal) // 2], np.uint8)
        cases.append(Case(f"cells-{mut}", len(px), 1, 2, px[:, :3].reshape(-1).copy(), palette=pal, targets=(mut,),
                          expect={"route": "table"}))
    return cases


def _key_ordered(rng, t, pi, pj, i, j, n):
    """n histogram colours, key-ordered, with pi at i and pj at j (key(pi) < key(pj)), the rest far from t, or None."""
    kt = lambda c: (int(c[0]) << 24) | (int(c[1]) << 16) | (int(c[2]) << 8) | int(c[3])
    ki, kj = kt(pi), kt(pj)
    pool = _fillers(rng, 40000, t)
    pool = pool[np.unique(R.keys_of(pool), return_index=True)[1]]
    k = R.keys_of(pool).astype(np.int64)
    lo, mid, hi = pool[k < ki], pool[(k > ki) & (k < kj)], pool[k > kj]
    need = (i, j - i - 1, n - 1 - j)
    if len(lo) < need[0] or len(mid) < need[1] or len(hi) < need[2]:
        return None
    pal = np.concatenate([lo[:need[0]], [pi], mid[:need[1]], [pj], hi[len(hi) - need[2]:]]).astype(np.uint8)
    assert (np.diff(R.keys_of(pal).astype(np.int64)) > 0).all()
    return pal


def early_cases():
    """400 x 250 RGBA (100 000 pixels, histogram stride 2): even pixels draw from the histogram colours, odd pixels are
    the tie colour t, which the histogram never sees."""
    rng = np.random.default_rng(2)
    cases = []
    w, h = 400, 250
    for kind, t in (("trunc", (60, 200, 90, 254)), ("trunc", (60, 200, 90, 255)), ("alpha", (60, 200, 90, 1)),
                    ("green", (60, 40, 90, 255)), ("floor", (100, 100, 100, 255))):
        pi, pj = sorted(_pair(kind, t), key=lambda c: tuple(c))
        for n in (2, 33, 64, 256):
            for i, j, where in placements(n):
                pal = _key_ordered(rng, t, pi, pj, i, j, n)
                if pal is None:
                    continue
                px = pal[(np.arange(w * h) // 2) % n]
                px[1::2] = t
                tg = warp_targets(i, j)
                cases.append(_also(Case(f"early-{kind}-a{t[3]}-n{n}-{where}-{i}-{j}", w, h, 3, px.reshape(-1).copy(),
                                  m=256, dither=True, targets=tuple(tg),
                                  expect={"tie": (i, j), "route": "early-miss", "n": n, "kind": kind}),
                                   ("dist_exact",)))
    return cases


# ---- k-means and median cut --------------------------------------------------------------------------
def _search(name, stride, m, pred, tries=4000, seed=0, span=6, ncol=(3, 9), cnt=(1, 6), alpha=False):
    """The first small histogram (3 to 8 colours in a small cube, counts 1-5) for which pred(case) holds.  Stride 1:
    each colour on `count` pixels.  Stride 2: every pixel doubled and the image tiled past 100 000 pixels, so the
    stride-2 histogram sees the same colours in the same proportions."""
    rng = np.random.default_rng(seed)
    for _ in range(tries):
        k = int(rng.integers(*ncol))
        a = rng.integers(0, span, (k, 1)) * 20 + 100 if alpha else np.full((k, 1), 255)
        cols = np.unique(np.concatenate([rng.integers(0, span, (k, 3)) * 3 + 90, a], 1), axis=0)
        if len(cols) <= m:
            continue
        px = np.repeat(cols.astype(np.uint8), rng.integers(*cnt, len(cols)), 0)
        if stride == 2:
            px = np.repeat(px, 2, 0)
            px = np.tile(px, (-(-100000 // len(px)), 1))
        c = Case(name, len(px), 1, 3, px.reshape(-1).copy(), m=m)
        if pred(c):
            return c
    raise AssertionError(f"no case found for {name}")


def _changes(c, mut):
    try:
        return c.run(frozenset([mut]), map_pixels_too=False).palette.tobytes() != \
            c.run(map_pixels_too=False).palette.tobytes()
    except R.Refused:
        return True


def kmeans_cases():
    out = []
    specs = [
        ("km-tie-pass1", "seq_last", lambda r: r.kmeans.tied[0]),
        ("km-tie-pass2", "seq_last", lambda r: r.kmeans.tied[1] and not r.kmeans.tied[0]),
        ("km-empty-pass1", "km_empty_zero", lambda r: r.kmeans.empty[0]),
        ("km-round", "km_round", lambda r: True),
        ("km-unweighted", "km_unweighted", lambda r: True),
        ("km-one-pass", "km_one_pass", lambda r: True),
    ]
    for stride in (1, 2):
        for k, (name, mut, info) in enumerate(specs):
            if stride == 2 and name not in ("km-tie-pass1", "km-empty-pass1", "km-round"):
                continue
            pred = lambda c, info=info, mut=mut: info(c.run(map_pixels_too=False)) and _changes(c, mut)
            c = _search(f"{name}-s{stride}", stride, 2 + k % 3, pred, seed=10 * k + stride,
                        tries=300 if stride == 2 else 4000)
            c.targets, c.expect = (mut,), {"kmeans": name}
            out.append(c)
    return out


def cut_cases():
    out = []
    specs = [("cut-box-tie", "box_first_max", lambda r: r.cut.box_tie),
             ("cut-channel-tie", "channel_ge", lambda r: r.cut.channel_tie),
             ("cut-split-eq", "split_gt", lambda r: r.cut.split_eq),
             ("cut-clamp", None, lambda r: r.cut.clamped)]
    for k, (name, mut, info) in enumerate(specs):
        for alpha in (False, True):
            pred = lambda c, info=info, mut=mut: info(c.run(map_pixels_too=False)) and (mut is None or _changes(c, mut))
            c = _search(f"{name}{'-alpha' if alpha else ''}", 1, 3 + k % 2, pred, seed=100 + 10 * k + alpha,
                        alpha=alpha)
            c.targets, c.expect = ((mut,) if mut else ()), {"cut": name}
            out.append(c)
    return out


# ---- decisions and samplers ----------------------------------------------------------------------------
def _distinct(k, rng, a=255):
    """k distinct opaque colours."""
    v = np.unique(rng.integers(0, 1 << 24, 2 * k + 64))
    v = rng.permutation(v)[:k]
    return np.stack([v >> 16, (v >> 8) & 255, v & 255, np.full(k, a)], 1).astype(np.uint8)


def decision_cases():
    rng = np.random.default_rng(3)
    out = []
    # Auto at unique = m, m + 1, 32 m, 32 m + 1 (stride 1)
    for m in (1, 2, 16, 255, 256):
        for u in (m, m + 1, 32 * m, 32 * m + 1):
            cols = _distinct(u, rng)
            npix = max(u, 64)
            px = cols[np.arange(npix) % u]
            tg = ("auto_ge",) if u == m else ("auto_lt",) if u == 32 * m else ()
            out.append(Case(f"auto-m{m}-u{u}", npix, 1, 2, px[:, :3].reshape(-1).copy(), mode="auto", m=m,
                            targets=tg, expect={"unique": u}))
    # the decision sampler: stride max(npix / 20000, 1), the deciding colour on the last sampled pixel
    m = 16
    for npix in (39999, 40000, 40001, 59999, 60000):
        stride = max(npix // 20000, 1)
        pos = R.sample_positions(npix, R.DECISION_CAP)
        base = _distinct(m + 1 + 700, rng)
        px = base[np.zeros(npix, np.int64)].copy()
        px[pos] = base[np.arange(len(pos)) % m]          # m colours on the sampled pixels
        px[pos[-1]] = base[m]                             # the deciding colour: m + 1
        mask = np.ones(npix, bool)
        mask[pos] = False
        px[mask] = base[m + 1 + np.arange(mask.sum()) % 700]   # unsampled pixels: 700 more colours (> 32 m)
        floor = npix % stride != 0
        out.append(Case(f"decide-{npix}", npix, 1, 2, px[:, :3].reshape(-1).copy(), mode="auto", m=m,
                        targets=("nd_floor",) if floor else (), expect={"unique": m + 1, "stride": stride}))
    # the histogram sampler and the early out: m against m + 1 colours, the deciding one on the last sample
    for npix in (99999, 100000, 100001):
        stride = max(npix // 50000, 1)
        pos = R.sample_positions(npix, R.HISTOGRAM_CAP)
        for extra in (0, 1):
            base = _distinct(m + 1 + 50, rng)
            px = np.repeat(base[m + 1:], -(-npix // 50), 0)[:npix].copy()   # unsampled: 50 more colours
            px[pos] = base[np.arange(len(pos)) % m]
            if extra:
                px[pos[-1]] = base[m]
            tg = ["nh_floor"] if extra and npix % stride else []
            if not extra:
                tg.append("early_lt")
            out.append(Case(f"early-{npix}-{m + extra}", npix, 1, 3, px.reshape(-1).copy(), m=m,
                            targets=tuple(tg), expect={"hist": m + extra, "stride": stride}))
    # 8 192 against 8 193 histogram colours, without and with a palette
    for k in (8192, 8193):
        cols = _distinct(k, rng)
        out.append(Case(f"trunc-{k}", k, 1, 2, cols[:, :3].reshape(-1).copy(), m=256,
                        targets=("trunc_ge",) if k == 8192 else (), expect={"hist": k}))
        out.append(Case(f"trunc-{k}-palette", k, 1, 2, cols[:, :3].reshape(-1).copy(), m=256,
                        palette=cols[::40][:200].copy(), expect={"hist": k}))
    return out


def batch_frames(n: int, m: int = 4, w: int = 16, h: int = 8):
    """n RGB frames from one shared set of colours; frame i holds m + (i % 2) of them, so Auto alternates."""
    rng = np.random.default_rng(4)
    cols = _distinct(m + 1, rng)
    frames = []
    for i in range(n):
        k = m + (i % 2)
        pick = cols[np.roll(np.arange(m + 1), i)[:k]]
        frames.append(pick[np.arange(w * h) % k][:, :3].reshape(-1).copy())
    return frames


# ---- dither at full scale -------------------------------------------------------------------------------
DITHER_W = (1, 2, 31, 32, 33, 63, 64, 65)
DITHER_H = (31, 33, 63, 65)


def dither_cases():
    rng = np.random.default_rng(5)
    black, white = (0, 0, 0, 255), (255, 255, 255, 255)
    out = []
    for k, w in enumerate(DITHER_W):
        h = DITHER_H[k % len(DITHER_H)]
        for name, img, pal in (("black-on-white", np.full((h * w, 3), 255), [black]),
                               ("white-on-black", np.zeros((h * w, 3)), [white]),
                               ("bw-on-grey", np.full((h * w, 3), 128), [black, white]),
                               ("bw-on-noise", rng.integers(0, 2, (h * w, 3)) * 255, [black, white])):
            # one entry: every index is 0 whatever the errors, so these cases only drive the clamps
            out.append(_also(Case(f"dither-{name}-{w}x{h}", w, h, 2, img.astype(np.uint8).reshape(-1).copy(), dither=True,
                            palette=np.array(pal, np.uint8), expect={"full": True}),
                             () if len(pal) == 1 else ("pack8", "err_unclamped", "err_src", "w13", "seam_zero")))
    # translucent pixels among opaque ones, tied under the adjusted colour (found by search)
    t = (expand(40), expand(20), expand(33), 200)
    pi, pj = _pair("trunc", t)
    for k, (i, j) in enumerate(((0, 32), (5, 33))):
        for seed in range(200):
            r2 = np.random.default_rng(1000 * k + seed)
            pal = _fillers(r2, 40, t)
            pal[i], pal[j] = pi, pj
            pal[1] = t[:3] + (255,)
            w, h = 37, 34
            px = np.tile(np.array(t, np.uint8), (w * h, 1))
            px[r2.random(w * h) < 0.5, 3] = 255
            c = Case(f"dither-translucent-{i}-{j}", w, h, 3, px.reshape(-1).copy(), dither=True, palette=pal,
                     targets=tuple(warp_targets(i, j)), expect={"tie": (i, j), "route": "dither-warp"})
            r = c.run()
            if any(len(tt) > 1 and rt == "dither-warp" and i in tt and j in tt for rt, tt in zip(r.routes, r.ties)) \
                    and all(c.run(frozenset([mm])).key() != r.key() for mm in c.targets):
                out.append(c)
                break
        else:
            raise AssertionError("no translucent dither tie found")
    return out


def all_cells():
    """512 x 512 RGB: pixel k is the colour of 6-6-6 cell k, so the index rows are the whole table."""
    return R.cell_colour(np.arange(1 << 18))[:, :3].astype(np.uint8).reshape(-1)


def all_colours():
    """4096 x 4096 RGB: every opaque colour once."""
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([v >> 16, (v >> 8) & 255, v & 255], 1).astype(np.uint8).reshape(-1)


def table_palettes():
    """Palettes for the whole-table and every-colour images: the cell-sweep ties, a random 256, two entries."""
    sweep = [c for c in sweep_cases() if c.name == "sweep-table"][0].palette
    rng = np.random.default_rng(6)
    return {"sweep": sweep, "random256": rng.integers(0, 256, (256, 4)).astype(np.uint8) | np.array([0, 0, 0, 255], np.uint8),
            "bw": np.array([[0, 0, 0, 255], [255, 255, 255, 255]], np.uint8)}
