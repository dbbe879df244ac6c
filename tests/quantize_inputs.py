"""Deterministic inputs of the palette-quantisation fixtures, shared by
oracle/wasm_ref/gen_golden_quantize.py (which produced tests/golden/quantize/ by running real pixo with
lossy = 1) and the tests that consume them.  numpy only.

make_quantize_input(kind, w, h, ch, seed, n) -> flat uint8 pixels
  pal, palo, palblk, noise   as make_reduce_input (n distinct colours, scattered / opaque / in blocks)
  grad       a diagonal gradient with +-8 noise (RGBA: alpha a gradient from 0 to 255)
  stride     n colours in blocks; every pixel at an odd index instead carries one of n rare colours,
             which pixo's histogram sampler (stride 2 above 100 000 pixels) never sees
  missed     200 colours at even pixel indices and n others at odd ones: the decision sample sees
             more than 256 colours, the histogram sample (stride 2) only the 200, so the early-out
             path maps the odd pixels by nearest-entry search
  trunc      pixels at indices divisible by 3 draw from 8 000 colours, the others from n more: the
             decision sample (stride 3 at 256x256) stays at or under 8 192 colours while the full
             histogram exceeds 8 192, pixo's truncation case
  gray       Gray or GrayAlpha noise (ch 1 or 2), which never quantises
"""
import json
import os

import numpy as np

from reduce_inputs import _colours, make_reduce_input, png_parts  # noqa: F401  (png_parts re-exported)

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quantize")


def load_manifest():
    return json.load(open(os.path.join(GOLD, "manifest.json")))


def make_quantize_input(kind: str, w: int, h: int, ch: int, seed: int, n: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    npx = w * h
    if kind in ("pal", "palo", "palblk", "noise"):
        return make_reduce_input(kind, w, h, ch, seed, n)
    if kind == "gray":
        return rng.integers(0, 256, npx * ch, dtype=np.uint8)
    if kind == "grad":
        y, x = np.mgrid[0:h, 0:w]
        t = (x * 255 // max(w - 1, 1) + y * 255 // max(h - 1, 1)) // 2
        img = np.stack([t, 255 - t, (x * 7 + y * 3) % 256] + ([y * 255 // max(h - 1, 1)] if ch == 4 else []), -1)
        img = img.astype(np.int32)
        img[..., :3] += rng.integers(-8, 9, img[..., :3].shape)
        return np.ascontiguousarray(np.clip(img, 0, 255).astype(np.uint8)).reshape(-1)
    if kind in ("stride", "missed", "trunc"):
        if kind == "trunc":
            common, rare = 8000, n
            on_common = np.arange(npx) % 3 == 0
        else:
            common, rare = (n, n) if kind == "stride" else (200, n)
            on_common = np.arange(npx) % 2 == 0
        cols = _colours(rng, common + rare, ch, "opaque")
        if kind == "stride":
            yy, xx = np.mgrid[0:h, 0:w]
            idx = ((yy // 4) * ((w + 7) // 8) + xx // 8).reshape(-1) % common
        else:
            idx = rng.integers(0, common, npx)
        idx = np.where(on_common, idx, common + rng.integers(0, rare, npx))
        return np.ascontiguousarray(cols[idx]).reshape(-1)
    raise ValueError(kind)
