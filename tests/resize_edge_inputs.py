"""Inputs for the resizer edge tests (tests/test_resize_edges.py, tests/test_resize_edges_gpu.py).

cap_cases(): Lanczos3 batches with the scratch cap PIXO_B200_RESIZE_SCRATCH sets, each naming the paths of
csrc/resize.cu it claims to take (resize_ref.lanczos_bands says whether it does):
  one-band     the whole intermediate in one band
  bands        several bands of destination rows, each frame through every band in turn
  exact        a band whose source-row window is exactly the cap
  overlap      consecutive bands whose windows share source rows
  chunks       a destination row whose taps alone exceed the cap: its columns in chunks
  ragged       chunks of unequal width, the last one column wide
  single-col   chunks of one column each (every destination pixel is its own pair of launches)
  passes       a one-band batch split into frame passes, the last of a single frame
Exact halves: frames holding every (a, b) byte pair, and the bytes integer arithmetic expects of them."""
from __future__ import annotations

import numpy as np

import resize_ref as rr
from oracle import resize as rz

GEOMS = {"down": (101, 61, 37, 23), "up": (43, 27, 101, 61), "mixed": (101, 23, 37, 61)}
TINY = {"tiny-down": (17, 9, 13, 7), "tiny-up": (7, 5, 17, 9)}
N = 3   # frames per capped call


def noise(sw, sh, bpp, seed):
    return np.random.default_rng(seed).integers(0, 256, sw * sh * bpp, dtype=np.uint8)


def frames(sw, sh, bpp, n, seed):
    """n frames: noise, and a 0/255 checkerboard with noise in channel 0 (sums near 0 and 255 clamp)"""
    out = []
    for i in range(n):
        f = noise(sw, sh, bpp, 1000 * seed + i)
        if i % 2:
            y, x = np.mgrid[0:sh, 0:sw]
            f = f.reshape(sh, sw, bpp)
            f[:, :, 1:] = ((((x // 3) + (y // 2)) % 2) * 255)[:, :, None]
            f[:, :, 0] = np.where(f[:, :, 0] < 128, 0, 255)
            f = f.reshape(-1)
        out.append(np.ascontiguousarray(f))
    return out


def plan(sw, sh, dw, dh, bpp, n, cap):
    """(bands, frames per pass, launches) of a Lanczos3 call under `cap`"""
    start, count = rz.contrib(sh, dh)[:2]
    bands = rr.lanczos_bands(start, count, sh, dw, dh, bpp, cap)
    per = rr.frames_per_pass(bands, n, bpp, cap)
    return bands, per, rr.lanczos_launches(bands, n, per)


def paths(bands, n, per, bpp, dw, cap):
    """The claims of the module docstring that a plan makes true"""
    got = set()
    rows = [b for b in bands if b[5] == dw]
    got.add("one-band" if len(bands) == 1 else "bands")
    if any((re - rs) * cw * bpp == cap for _, _, rs, re, _, cw in bands):
        got.add("exact")
    if any(b[2] < a[3] and b[0] == a[1] for a, b in zip(rows, rows[1:])):
        got.add("overlap")
    chunked = {}
    for b in bands:
        if b[5] < dw:
            chunked.setdefault(b[0], []).append(b[5])
    if chunked:
        got.add("chunks")
        if any(len(set(w)) > 1 and w[-1] == 1 for w in chunked.values()):
            got.add("ragged")
        if all(w == [1] * dw for w in chunked.values()):
            got.add("single-col")
    if per > 1 and n % per == 1:
        got.add("passes")
    return got


def _exact_k(sw, sh, dw, dh, bpp, lo, hi):
    """The first k in lo..hi-1 whose cap k * row closes a band with a window of exactly k rows"""
    for k in range(lo, hi):
        bands = plan(sw, sh, dw, dh, bpp, N, k * dw * bpp)[0]
        if len(bands) > 1 and "exact" in paths(bands, N, 1, bpp, dw, k * dw * bpp):
            return k
    raise AssertionError(("no exact band", sw, sh, dw, dh, bpp, lo, hi))


def cap_cases():
    """[(name, (sw, sh, dw, dh), bpp, n, cap, claims)]"""
    cases = []
    for g, (sw, sh, dw, dh) in GEOMS.items():
        count = rz.contrib(sh, dh)[1]
        taps = int(count.max())
        for bpp in range(1, 5):
            row = dw * bpp
            frame = sh * row
            k_mid = _exact_k(sw, sh, dw, dh, bpp, max(taps, sh // 2), sh)
            k_min = _exact_k(sw, sh, dw, dh, bpp, taps, sh)
            cases += [
                (f"{g}-{bpp}-whole", (sw, sh, dw, dh), bpp, N, frame, {"one-band", "exact"}),
                (f"{g}-{bpp}-whole-1", (sw, sh, dw, dh), bpp, N, frame - 1, {"bands", "overlap"}),
                (f"{g}-{bpp}-k{k_mid}", (sw, sh, dw, dh), bpp, N, k_mid * row, {"bands", "exact", "overlap"}),
                (f"{g}-{bpp}-k{k_mid}-1", (sw, sh, dw, dh), bpp, N, k_mid * row - 1, {"bands", "overlap"}),
                (f"{g}-{bpp}-k{k_min}", (sw, sh, dw, dh), bpp, N, k_min * row, {"bands", "exact", "overlap"}),
                (f"{g}-{bpp}-taps-1", (sw, sh, dw, dh), bpp, N, taps * row - 1, {"bands", "chunks", "ragged"}),
                (f"{g}-{bpp}-passes-2", (sw, sh, dw, dh), bpp, 5, 2 * frame, {"one-band", "passes"}),
                (f"{g}-{bpp}-passes-3", (sw, sh, dw, dh), bpp, 4, 4 * frame - 1, {"one-band", "passes"}),
                (f"{g}-{bpp}-passes-1", (sw, sh, dw, dh), bpp, 3, 2 * frame - 1, {"one-band"}),
            ]
    for g, (sw, sh, dw, dh) in TINY.items():
        for bpp in range(1, 5):
            cases.append((f"{g}-{bpp}-1byte", (sw, sh, dw, dh), bpp, 2, 1, {"bands", "chunks", "single-col"}))
    return cases


# ---- exact halves -------------------------------------------------------------------------------------
def pairs(bpp):
    """Every (a, b) byte pair once: (65536 / bpp, 2, bpp), pair p in channel p % bpp of row p // bpp"""
    p = np.arange(65536)
    ab = np.stack([p >> 8, p & 255], axis=1).astype(np.uint8)              # (65536, 2)
    return np.ascontiguousarray(ab.reshape(65536 // bpp, bpp, 2).transpose(0, 2, 1))


def bilinear_halves(a, b, dst):
    """Bilinear 2 -> dst (3 or 5) between a and b: the blends are k/(dst-1) of the way, exact in f32, so
    the byte is ((dst-1-k) a + k b) / (dst-1) rounded half away from zero, in integers"""
    q = dst - 1
    k = np.arange(dst)
    num = (q - k)[None, :] * a.astype(np.int64)[:, None] + k[None, :] * b.astype(np.int64)[:, None]
    return ((2 * num + q) // (2 * q)).astype(np.uint8)                       # (len(a), dst)


def nearest_halves(src, dst):
    """Nearest src -> dst = src / r for an even r: position d lands on r d + r/2 - 1/2, which rounds to
    r d + r/2 (odd r: exactly r d + (r-1)/2); index r d + r // 2 either way"""
    r = src // dst
    assert r * dst == src
    return r * np.arange(dst) + r // 2
