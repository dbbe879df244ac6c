"""Frames built to sit on the JPEG transform kernels' edges (tests/transform_ref.py restates what they compute).

  * Quantiser cases: pixel blocks, found by a seeded search in pixel space, and per-position divisors d in 1..255
    for which pixo's quotient RN(x / d) is exactly +-(k + 1/2) (k = 0, 1, 2 or >= 64: half-away and half-even
    differ for even k, half toward +inf for every negative one), or one float32 ulp below or above it (-0.49999997
    and +0.49999997, 0x3EFFFFFF, among them: the one quotient where RZ and RN of q + 0.5 differ), on every route:
    K1 luma, K1 chroma (quad sums, the divisor folded x4), K2 luma, K2 chroma and gray.  Each case is certified
    with fractions.Fraction: the exact x / d, the float the division returns and the integer pixo rounds it to.
    Cases are packed into frames whose tables agree at the cases' positions; every frame is one row of blocks
    (gray and 4:4:4) or MCUs (4:2:0).
  * Colour frames: every colour as a flat block or MCU, and every colour once in a 2x2 quad tiled over an MCU, with
    all-ones tables.  These are generated on the device by the GPU tests; this file holds their layout.
  * Geometry frames: noise whose last column and last row differ from their neighbours, at every width and height
    residue of the MCU, around the 128-px half tile, the 256-px unit and the 512-px gray tile.
  * Walk shapes: units per MCU row x MCU rows x frames for the persistent kernels' unit walk.
Everything is deterministic and cached per process."""
from __future__ import annotations

import functools
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

import transform_ref as R

F32 = np.float32
ROUTES = ("gray", "k2_y", "k2_c", "k1_y", "k1_c")
LARGE_K = 64        # k >= LARGE_K counts as "a large k"
TARGET_KS = (0, 1, 2)


@dataclass
class Case:
    route: str
    block: int          # index of the block (gray / 4:4:4) or MCU (4:2:0) in its frame
    comp: int           # 0 Y, 1 Cb, 2 Cr
    sub: int            # Y block within the MCU (4:2:0), else 0
    pos: int            # natural-order position
    d: int
    x: float            # pixo's f32 DCT coefficient
    q: float            # RN(x / d)
    want: int           # pixo's integer
    kind: str           # "tie", "below" (one ulp below k + 1/2 in magnitude) or "above"
    k: int
    flips: tuple = ()   # transform_ref mutants whose result differs


@dataclass
class CaseFrame:
    mode: str           # "gray", "444" or "420"
    w: int
    h: int
    pixels: np.ndarray  # uint8, h * w * channels
    lum_q: np.ndarray   # float32[64]
    chr_q: np.ndarray
    cases: list = field(default_factory=list)


def classify(q):
    """float32 quotients -> (kind code 0 none / 1 tie / 2 below / 3 above, k)"""
    a = np.abs(q).astype(F32)
    up, down = np.nextafter(a, F32(np.inf)), np.nextafter(a, F32(0))

    def tie(v):
        t = v.astype(np.float64) * 2
        return (t == np.floor(t)) & (np.floor(t) % 2 == 1)

    kind = np.where(tie(a), 1, np.where(tie(up), 2, np.where(tie(down), 3, 0)))
    k = np.where(kind == 2, np.floor(up), np.floor(a)).astype(np.int64)
    return kind, k


def certify(x, d):
    """(q, integer) from exact arithmetic: q the float32 nearest x / d, pixo's integer its half-away rounding"""
    exact = Fraction(float(x)) / d
    q = R.rn(exact)
    assert float(F32(x) / F32(d)) == float(q), (x, d)
    a = int(abs(q) + Fraction(1, 2))
    return q, (-a if q < 0 else a)


def _flips(route, x, d):
    """the transform_ref mutants under which the kernel's integer differs from pixo's, exactly"""
    sc = 4 if route == "k1_c" else 1
    want = R.pixo_quant(x, d)
    assert R.kernel_quant(x, d, sc) == want, (route, x, d)
    return tuple(m for m in R.MUTANTS if (m != "no_fold" or sc == 4) and R.kernel_quant(x, d, sc, (m,)) != want)


def _cheap_flips(route, x, d, kind, k):
    """_flips predicted without fractions (checked against _flips for every chosen case)"""
    neg = x < 0
    out = []
    if kind == 2 and k == 0 and not neg:
        out.append("rz_to_rn")
    xf = F32(x)
    if R.round_half_away(F32(xf * (F32(1) / F32(d)))) != R.round_half_away(F32(xf / F32(d))):
        out.append("no_residual")
    if kind == 1 and k % 2 == 0:
        out.append("half_even")
    if kind == 1 and neg:
        out.append("half_up_neg")
    if route == "k1_c":
        out.append("no_fold")
    return tuple(out)


def _tiles(rng, n, px, style):
    """n RGB tiles of px x px: uniform noise, noise around a random level, or pixels of 0 and 255"""
    if style == 0:
        return rng.integers(0, 256, (n, px, px, 3), dtype=np.int32)
    if style == 1:
        lvl = rng.integers(0, 256, (n, 1, 1, 3))
        amp = rng.integers(1, 40, (n, 1, 1, 1))
        return np.clip(lvl + rng.integers(-64, 65, (n, px, px, 3)) * amp // 40, 0, 255)
    return rng.integers(0, 2, (n, px, px, 3), dtype=np.int32) * 255


def _component_blocks(route, tiles):
    """tiles -> (f32 blocks [n, nb, 64], (comp, sub) per block slot)"""
    if route == "gray":
        return R.gray_block(tiles[..., 0].reshape(len(tiles), 1, 64)), [(0, 0)]
    ycc = R.rgb_to_ycbcr(tiles).astype(np.int32)
    if route in ("k2_y", "k2_c"):
        comps = (0,) if route == "k2_y" else (1, 2)
        return np.stack([R.gray_block(ycc[..., c].reshape(len(tiles), 64)) for c in comps], 1), \
            [(c, 0) for c in comps]
    if route == "k1_y":
        y = ycc[..., 0].reshape(len(tiles), 2, 8, 2, 8).transpose(0, 1, 3, 2, 4).reshape(len(tiles), 4, 64)
        return R.gray_block(y), [(0, s) for s in range(4)]
    sums = ycc[..., 1:].reshape(len(tiles), 8, 2, 8, 2, 2).sum(axis=(2, 4))       # [n, 8, 8, 2]
    return np.stack([R.chroma_420_block(sums[..., c].reshape(len(tiles), 64)) for c in (0, 1)], 1), [(1, 0), (2, 0)]


def _hits(x):
    """(block, slot, position, d, kind, k) for every coefficient of x [n, nb, 64] whose quotient by some d is a
    target.  Every target is d (2j + 1) / 2 within an ulp of the quotient, so x lies within a few of its own ulps
    of a multiple of 1/2: that filter goes first."""
    ax = np.abs(x.astype(np.float64))
    ulp = np.spacing(np.abs(x)).astype(np.float64)
    near = (np.abs(2 * ax - np.rint(2 * ax)) <= 8 * ulp) & (ax > 0)
    t, b, p = np.nonzero(near)
    xs, a = x[t, b, p], ax[t, b, p]
    out = []
    cands = [np.rint(a / (k + 0.5)) for k in TARGET_KS] + [np.full(a.shape, d, np.float64) for d in range(1, 16)]
    for dd in cands:
        ok = (dd >= 1) & (dd <= 255)
        q = (xs / np.where(ok, dd, 1).astype(F32)).astype(F32)
        kind, k = classify(q)
        hit = ok & (kind > 0) & ((k <= TARGET_KS[-1]) | (k >= LARGE_K))
        out += zip(t[hit].tolist(), b[hit].tolist(), p[hit].tolist(), dd[hit].astype(int).tolist(),
                   kind[hit].tolist(), k[hit].tolist())
    return sorted(set(out))


def _search(route, seed, n_tiles, chunk=20000):
    """tiles, their component slots, their DCT coefficients and the hits among them"""
    rng = np.random.default_rng(seed)
    px = 16 if route.startswith("k1") else 8
    tiles, xs, found = [], [], []
    for c0 in range(0, n_tiles, chunk):
        t = _tiles(rng, chunk, px, (c0 // chunk) % 3)
        if route == "gray":
            t = t[..., :1]
        blocks, slots = _component_blocks(route, t)
        x = R.dct_2d(blocks)
        found += [(h[0] + c0,) + h[1:] for h in _hits(x)]
        tiles.append(t.astype(np.uint8))
        xs.append(x)
    return np.concatenate(tiles), slots, np.concatenate(xs), found


KIND = {1: "tie", 2: "below", 3: "above"}


def _select(route, found, x, slots):
    """Enough cases to cover every (sign, kind, k class) twice, every mutant twice, every position and d = 1 and
    d = 255; each case is certified with fractions"""
    chosen, count = [], {}
    for t, b, p, d, kind, k in found:
        xv = float(x[t, b, p])
        kc = k if k < LARGE_K else LARGE_K
        keys = [("class", xv < 0, kind, kc), ("pos", p)] + ([("d", d)] if d in (1, 255) else [])
        keys += [("mut", m) for m in _cheap_flips(route, xv, d, kind, k)]
        if all(count.get(key, 0) >= (1 if key[0] in ("pos", "d") else 2) for key in keys):
            continue
        flips = _flips(route, xv, d)
        assert flips == _cheap_flips(route, xv, d, kind, k), (route, xv, d, flips)
        q, want = certify(xv, d)
        comp, sub = slots[b]
        chosen.append((t, Case(route, -1, comp, sub, p, d, xv, float(q), want, KIND[kind], k, flips)))
        for key in keys:
            count[key] = count.get(key, 0) + 1
    return chosen


def _pack(route, chosen, tiles, seed):
    """Cases -> frames: a case joins the first frame whose table is free or equal at its position"""
    rng = np.random.default_rng(seed)
    mode = {"gray": "gray", "k2_y": "444", "k2_c": "444"}.get(route, "420")
    chroma = route in ("k2_c", "k1_c")
    groups = []   # [table dict, [(tile, case)]]
    for t, c in chosen:
        for tab, members in groups:
            if tab.get(c.pos, c.d) == c.d and all(m[0] != t for m in members):
                tab[c.pos] = c.d
                members.append((t, c))
                break
        else:
            groups.append(({c.pos: c.d}, [(t, c)]))
    frames = []
    px = 16 if mode == "420" else 8
    for tab, members in groups:
        q = rng.integers(1, 256, 64).astype(F32)
        for p, d in tab.items():
            q[p] = d
        other = rng.integers(1, 256, 64).astype(F32)
        lum_q, chr_q = (other, q) if chroma else (q, other)
        if mode == "gray":   # pixo ignores chr_q for gray; the table still goes through validation
            chr_q = other
        ch = 1 if mode == "gray" else 3
        strip = np.concatenate([tiles[t].reshape(px, px, ch) for t, _ in members], axis=1)
        fr = CaseFrame(mode, strip.shape[1], px, strip.astype(np.uint8).reshape(-1), lum_q, chr_q)
        for i, (t, c) in enumerate(members):
            c.block = i
            fr.cases.append(c)
        frames.append(fr)
    return frames


N_TILES = {"gray": 160000, "k2_y": 160000, "k2_c": 80000, "k1_y": 40000, "k1_c": 120000}


@functools.lru_cache(maxsize=None)
def quantiser_frames(route):
    """[CaseFrame] for one route"""
    seed = 1000 + ROUTES.index(route)
    tiles, slots, x, found = _search(route, seed, N_TILES[route])
    chosen = _select(route, found, x, slots)
    return _pack(route, chosen, tiles, seed)


def all_quantiser_frames():
    return [f for r in ROUTES for f in quantiser_frames(r)]


# ---- colour frames --------------------------------------------------------------------------------------
FLAT444_W = 4096          # 512 colours per 4096 x 8 frame
FLAT420_W = 8192          # 512 colours per 8192 x 16 frame
QUAD_W = 8192             # 512 quads (MCUs) per 8192 x 16 frame
CHUNK444 = 1 << 22        # colours per call: 805 MB of pixels
CHUNK420 = 1 << 20        # colours per call: 805 MB of pixels
CHUNK_QUAD = 1 << 20      # quads per call: 805 MB of pixels


@functools.lru_cache(maxsize=1)
def quad_permutation():
    """every colour exactly once: [2^22, 4] colour indices, quad m's pixels in the order TL, TR, BL, BR"""
    return np.random.default_rng(2024).permutation(1 << 24).astype(np.int32).reshape(-1, 4)


def extreme_quads():
    """quads whose chroma sums Sum(256 - c) reach the ends of their range, for Cb and for Cr: 4 (c = 255 four times)
    and 1020 (c = 1 four times); each quad holds four different colours"""
    ycc = R.all_colours_ycbcr()
    out = []
    for comp, val in ((1, 255), (1, 1), (2, 255), (2, 1)):
        idx = np.flatnonzero(ycc[:, comp] == val)
        out.append(idx[np.linspace(0, idx.size - 1, 4).astype(int)])
    return np.stack(out).astype(np.int32)


# ---- geometry frames ------------------------------------------------------------------------------------
def geometry_frame(w, h, ch, seed):
    """noise whose last column and last row differ from the column and row before them in every byte"""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (h, w, ch), dtype=np.int32)
    if w > 1:
        f[:, -1] = (f[:, -2] + rng.integers(1, 256, (h, ch))) % 256
    if h > 1:
        f[-1] = (f[-2] + rng.integers(1, 256, (w, ch))) % 256
    return f.astype(np.uint8).reshape(-1)


def geometry_shapes(mode):
    """(w, h) for one mode: every residue of the MCU in both directions, and widths around the kernels' tiles"""
    m = 16 if mode == "420" else 8
    shapes = [(2 * m + a, m + b) for a in range(m) for b in range(m)]
    if mode == "gray":
        shapes += [(w, 9) for w in (7, 504, 505, 511, 512, 513, 519, 520, 1023, 1024, 1025)]
    else:
        shapes += [(w, 17) for w in (112, 120, 127, 128, 129, 136, 240, 255, 256, 257, 264, 383, 384, 385, 512, 513)]
    return shapes


# ---- walk shapes ----------------------------------------------------------------------------------------
WALK_UNITS_X = (1, 2, 3, 15, 16, 17)
WALK_MCUS_Y = (1, 3, 7)
WALK_STRIDE_MAX = 4 * 3 * 132     # 4 warps x 3 CTAs per SM x 132 SMs


def walk_shapes(mode):
    """(w, h, n, units_x, mcus_y): frames whose units number at least three times the largest stride"""
    px, per_unit = (16, 16) if mode == "420" else (8, 32)
    out = []
    for ux in WALK_UNITS_X:
        for my in WALK_MCUS_Y:
            w = ((ux - 1) * per_unit + 1) * px - 3     # the last unit holds one (partial) MCU
            n = -(-3 * WALK_STRIDE_MAX // (ux * my))
            out.append((w, my * px, n, ux, my))
    return out
