"""Inputs of the resize fixtures (oracle/wasm_ref/gen_golden_resize.py) and of the tests that reproduce them.
Every geometry runs under all three algorithms and all four colour types.  "edges" frames are 0/255 blocks
and stripes, so Lanczos3's ringing drives sums below 0 and above 255; "noise" frames are uniform noise."""
import numpy as np

GEOMETRIES = [
    # (sw, sh, dw, dh, kind)
    (37, 29, 37, 29, "noise"),        # identity
    (23, 17, 46, 34, "edges"),        # 2x up
    (97, 61, 37, 29, "edges"),        # non-integer down
    (37, 29, 100, 71, "noise"),       # non-integer up
    (1, 1, 9, 4, "noise"),            # 1x1 -> N
    (31, 19, 1, 1, "edges"),          # N -> 1x1
    (1000, 3, 7, 30, "edges"),        # extreme aspect ratios, both ways
    (2, 500, 50, 3, "noise"),
    (257, 263, 64, 61, "edges"),      # prime sizes
    (1024, 5, 3, 2, "noise"),         # 1024 -> 3: support 3 * 341.33 taps
    (300, 200, 301, 199, "edges"),    # near-identity, non-integer both ways
]
CASES = [dict(sw=sw, sh=sh, dw=dw, dh=dh, ct=ct, alg=alg, kind=kind, seed=17 + i)
         for i, (sw, sh, dw, dh, kind) in enumerate(GEOMETRIES) for ct in range(4) for alg in range(3)]


def make_resize_input(c) -> np.ndarray:
    bpp = c["ct"] + 1
    rng = np.random.default_rng(c["seed"])
    h, w = c["sh"], c["sw"]
    if c["kind"] == "noise":
        img = rng.integers(0, 256, (h, w, bpp), dtype=np.uint8)
    else:
        y, x = np.mgrid[0:h, 0:w]
        base = (((x // 3) + (y // 2)) % 2) * 255
        base = np.where((x % 7) == 0, 255 - base, base)
        img = np.repeat(base[:, :, None], bpp, axis=2).astype(np.uint8)
        img[:, :, -1] = np.where(rng.random((h, w)) < 0.1, 255 - img[:, :, -1], img[:, :, -1])
    return np.ascontiguousarray(img).reshape(-1)
