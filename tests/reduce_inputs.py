"""Deterministic inputs of the colour-type / palette reduction fixtures, shared by
oracle/wasm_ref/gen_golden_reduce.py (which produced tests/golden/reduce/ by running real pixo) and
the tests that consume them.  numpy only.

make_reduce_input(kind, w, h, ch, seed, n) -> flat uint8 pixels
  pal        n distinct colours scattered at random (RGBA: alphas 0, 255 and in between)
  palo       n distinct opaque colours (RGBA with alpha 255: no tRNS)
  palblk     n distinct colours in 4x3 blocks (neighbours mostly equal)
  pal0       n colours of which half have alpha 0 with differing RGB
  dom        one colour on n percent of the pixels, 20 others on the rest
  stripes    vertical stripes of n colours, one pixel wide (equal edge weights)
  checker    colour (x + y) % n (equal edge weights and candidate sums)
  graypal    gray pixels (r = g = b) of n levels 0..n-1
  noise      independent random bytes
  opaque     random RGB, alpha 255
  grayalpha  random gray with random alpha, a quarter of it 0
"""
import json
import os
import struct
import zlib

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PNG_STRATEGY = {0: 7, 1: 6, 2: 8}  # preset -> FilterStrategy (AdaptiveFast, Adaptive, Bigrams)


def load_manifest():
    return json.load(open(os.path.join(GOLD, "reduce", "manifest.json")))


def skipped_golden_cases():
    """The fixtures of tests/golden/manifest.json whose IHDR shows a reduction (3x2 RGBA inputs that
    pixo turned into a 4-bit palette)."""
    out = []
    for c in json.load(open(os.path.join(GOLD, "manifest.json")))["png"]:
        ihdr = png_parts(open(os.path.join(GOLD, c["file"]), "rb").read())["ihdr"]
        if (ihdr[2], ihdr[3]) != (8, (0, 4, 2, 6)[c["ct"]]):
            out.append(c)
    return out


def png_parts(png: bytes) -> dict:
    """IHDR fields, PLTE / tRNS payloads, the decompressed IDAT stream and its zlib Adler-32."""
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    p, idat, parts = 8, b"", {"PLTE": None, "tRNS": None}
    while p < len(png):
        ln = struct.unpack(">I", png[p:p + 4])[0]
        typ, data = png[p + 4:p + 8], png[p + 8:p + 8 + ln]
        assert struct.unpack(">I", png[p + 8 + ln:p + 12 + ln])[0] == zlib.crc32(typ + data)
        if typ == b"IDAT":
            idat += data
        elif typ == b"IHDR":
            parts["ihdr"] = struct.unpack(">IIBBBBB", data)
        else:
            parts[typ.decode()] = data
        p += 12 + ln
    parts["raw"] = zlib.decompress(idat)
    parts["adler"] = struct.unpack(">I", idat[-4:])[0]
    return parts


def _colours(rng, n: int, ch: int, alpha: str) -> np.ndarray:
    """n distinct ch-channel colours."""
    out = np.zeros((0, ch), np.uint8)
    while out.shape[0] < n:
        c = rng.integers(0, 256, (2 * n + 8, ch), dtype=np.uint8)
        if ch == 4:
            if alpha == "opaque":
                c[:, 3] = 255
            else:
                pick = rng.integers(0, 3, c.shape[0])
                c[:, 3] = np.where(pick == 0, 0, np.where(pick == 1, 255, c[:, 3]))
        allc = np.concatenate([out, c])
        _, first = np.unique(allc.view(np.dtype((np.void, ch))).reshape(-1), return_index=True)
        out = allc[np.sort(first)]
    return out[:n]


def _scatter(rng, n: int, npx: int) -> np.ndarray:
    """colour index per pixel, every colour present when npx >= n"""
    idx = rng.integers(0, n, npx)
    k = min(n, npx)
    idx[rng.permutation(npx)[:k]] = np.arange(k)
    return idx


def make_reduce_input(kind: str, w: int, h: int, ch: int, seed: int, n: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    npx = w * h
    if kind in ("pal", "palo", "palblk"):
        cols = _colours(rng, n, ch, "opaque" if kind == "palo" else "mixed")
        if kind == "palblk":
            y, x = np.mgrid[0:h, 0:w]
            idx = ((y // 3) * ((w + 3) // 4) + x // 4).reshape(-1) * 7 % n
            idx[rng.permutation(npx)[:min(n, npx)]] = np.arange(min(n, npx))
        else:
            idx = _scatter(rng, n, npx)
        return np.ascontiguousarray(cols[idx]).reshape(-1)
    if kind == "pal0":
        assert ch == 4
        cols = _colours(rng, n, 4, "opaque")
        cols[: n // 2, 3] = 0
        return np.ascontiguousarray(cols[_scatter(rng, n, npx)]).reshape(-1)
    if kind == "dom":
        cols = _colours(rng, 21, ch, "opaque")
        idx = 1 + rng.integers(0, 20, npx)
        idx[rng.permutation(npx)[: npx * n // 100]] = 0
        return np.ascontiguousarray(cols[idx]).reshape(-1)
    if kind in ("stripes", "checker"):
        cols = _colours(rng, n, ch, "opaque")
        y, x = np.mgrid[0:h, 0:w]
        idx = (x % n) if kind == "stripes" else ((x + y) % n)
        return np.ascontiguousarray(cols[idx.reshape(-1)]).reshape(-1)
    if kind == "graypal":
        v = rng.integers(0, n, npx).astype(np.uint8)
        v[: min(n, npx)] = np.arange(min(n, npx))
        img = np.repeat(v[:, None], ch, axis=1)
        if ch == 4:
            img[:, 3] = 255
        return np.ascontiguousarray(img).reshape(-1)
    if kind == "noise":
        return rng.integers(0, 256, npx * ch, dtype=np.uint8)
    if kind == "opaque":
        img = rng.integers(0, 256, (npx, 4), dtype=np.uint8)
        img[:, 3] = 255
        return img.reshape(-1)
    if kind == "grayalpha":
        v = rng.integers(0, 256, npx, dtype=np.uint8)
        a = rng.integers(0, 256, npx, dtype=np.uint8)
        a[rng.random(npx) < 0.25] = 0
        return np.ascontiguousarray(np.stack([v, v, v, a], 1)).reshape(-1)
    raise ValueError(kind)
