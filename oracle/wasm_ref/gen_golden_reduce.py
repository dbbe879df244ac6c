#!/usr/bin/env python
"""Generates tests/golden/reduce/* by running the reference ITSELF: pixo's committed WebAssembly build
(web/src/lib/pixo-wasm/pixo_bg.wasm of a pixo checkout) executed by oracle/wasm_ref, with presets 1
(balanced) and 2 (max), which both reduce the colour type and the palette before filtering.

    python oracle/wasm_ref/gen_golden_reduce.py <pixo checkout>

Every fixture is a complete PNG file from encodePng; manifest.json says how to regenerate each input
(tests/reduce_inputs.py) and gives the SHA-256 of that input.
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.wasm_ref import build as wb  # noqa: E402
from oracle.wasm_ref import gen_golden as gg  # noqa: E402
from reduce_inputs import make_reduce_input  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reduce")
WIDTHS = (1, 3, 5, 7, 9, 65, 200)

CASES = []


def case(kind, w, h, ct, n=0, seed=1, preset=1):
    CASES.append(dict(kind=kind, w=w, h=h, ct=ct, n=n, seed=seed, preset=preset))


# palette sizes, RGB and RGBA (RGBA "pal" has alpha 0 and alpha < 255 entries: tRNS)
for k, n in enumerate((1, 2, 3, 4, 5, 16, 17, 255, 256)):
    for ct in (2, 3):
        w = WIDTHS[(k + ct) % len(WIDTHS)]
        h = max(6, -(-n // w) + 3)
        if w * h > 65536:
            h = 65536 // w
        case("pal", w, h, ct, n, seed=10 + k)
    case("palo", 33, 29, 3, n, seed=20 + k)
    case("palblk", 64, 48, 2, n, seed=30 + k)
# row padding of 1/2/4-bit rows
for w in WIDTHS:
    for n in (2, 3, 5, 9):
        case("pal", w, 7, 2, n, seed=40 + w)
# alpha-0 entries with differing RGB
for n in (4, 17, 200):
    case("pal0", 40, 30, 3, n, seed=50 + n)
# most-popular rotation: a dominant colour above, at and just under 15 %
for pct in (10, 14, 16, 25, 40, 70):
    for seed in (1, 2, 3):
        case("dom", 60, 50, 2, pct, seed=seed)
# ties: equal edge weights and equal candidate sums
for n in (3, 4, 5, 6, 8):
    case("stripes", 24, 8, 2, n)
    case("checker", 16, 16, 2, n)
    case("checker", 17, 5, 3, n, seed=2)
# gray content: with both presets' flags every gray RGB image becomes a palette
for n in (2, 4, 16, 200):
    case("graypal", 50, 40, 2, n)
    case("graypal", 50, 40, 3, n)
# over 256 colours
case("pal", 64, 64, 2, 257, seed=3)
case("pal", 64, 64, 3, 257, seed=3)
case("noise", 64, 64, 2)                 # stays RGB
case("opaque", 64, 64, 3)                # -> RGB
case("grayalpha", 64, 64, 3)             # -> GrayAlpha
case("noise", 64, 64, 3)                 # no reduction
# inputs that never reduce
case("noise", 45, 30, 0)
case("noise", 45, 30, 1)
# full-size preset 1
case("palblk", 256, 256, 3, 200, seed=7)
case("pal", 256, 256, 2, 256, seed=8)
case("opaque", 256, 256, 3, seed=9)
# preset 2 (max): small, its Zopfli-style DEFLATE is slow under the interpreter
for kind, w, h, ct, n in (("pal", 9, 7, 2, 3), ("pal", 13, 9, 3, 17), ("checker", 16, 8, 2, 5),
                          ("dom", 20, 20, 2, 30), ("opaque", 16, 16, 3, 0), ("grayalpha", 16, 16, 3, 0),
                          ("graypal", 16, 16, 2, 4)):
    case(kind, w, h, ct, n, seed=60, preset=2)


def main():
    wb.build()
    os.makedirs(OUT, exist_ok=True)
    manifest = {"source": "pixo_bg.wasm from leerob/pixo @ 437bf63 (web/src/lib/pixo-wasm), sha256 " +
                hashlib.sha256(open(gg.WASM, "rb").read()).hexdigest(),
                "runner": "oracle/wasm_ref/wasm_ref.c", "inputs": "tests/reduce_inputs.py", "png": []}
    for i, c in enumerate(CASES):
        img = make_reduce_input(c["kind"], c["w"], c["h"], (1, 2, 3, 4)[c["ct"]], c["seed"], c["n"])
        out = gg.run(["png", c["w"], c["h"], c["ct"], c["preset"], 0], img)
        name = f"r{i:03d}.png"
        open(os.path.join(OUT, name), "wb").write(out)
        manifest["png"].append(dict(c, file=name, input_sha256=hashlib.sha256(img.tobytes()).hexdigest()))
    json.dump(manifest, open(os.path.join(OUT, "manifest.json"), "w"), indent=1)
    total = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print(f"{len(CASES)} PNG fixtures, {total / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
