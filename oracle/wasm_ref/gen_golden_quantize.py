#!/usr/bin/env python
"""Generates tests/golden/quantize/* by running the reference ITSELF: pixo's committed WebAssembly build
(web/src/lib/pixo-wasm/pixo_bg.wasm of a pixo checkout) executed by oracle/wasm_ref, with lossy = 1,
which selects QuantizationMode::Auto with Floyd-Steinberg dithering and max_colors 256.

    python oracle/wasm_ref/gen_golden_quantize.py <pixo checkout>

Every fixture is a complete PNG file from encodePng; manifest.json says how to regenerate each input
(tests/quantize_inputs.py) and gives the SHA-256 of that input.  A quantised fixture takes about 16 s
under the interpreter (PaletteLut::new alone is 262 144 nearest-entry searches), so the cases run in
parallel processes and stay small.
"""
import hashlib
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.wasm_ref import build as wb  # noqa: E402
from oracle.wasm_ref import gen_golden as gg  # noqa: E402
from quantize_inputs import make_quantize_input  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "quantize")

CASES = []


def case(kind, w, h, ct, n=0, seed=1, preset=1):
    CASES.append(dict(kind=kind, w=w, h=h, ct=ct, n=n, seed=seed, preset=preset))


# distinct colours (RGB), over the 32-row warp groups
case("pal", 33, 16, 2, 257, seed=1)
case("pal", 65, 33, 2, 300, seed=2)
case("pal", 200, 40, 2, 1000, seed=3)
case("pal", 65, 100, 2, 4000, seed=4)
case("pal", 200, 64, 2, 8000, seed=5)
# RGBA: opaque (no tRNS), and alpha 0 / partial alpha (trimmed tRNS, translucent search in the dither)
case("palo", 33, 65, 3, 1000, seed=6)
case("pal", 65, 40, 3, 300, seed=7)
case("pal", 200, 33, 3, 1000, seed=8)
case("pal", 65, 64, 3, 4000, seed=9)
# colours in blocks
case("palblk", 64, 48, 2, 500, seed=10)
case("palblk", 200, 65, 3, 2000, seed=11)
# narrow and one-row images
case("pal", 1, 300, 2, 257, seed=12)
case("pal", 2, 200, 3, 300, seed=13)
case("pal", 3, 150, 2, 400, seed=14)
case("pal", 7, 64, 3, 300, seed=15)
case("pal", 300, 1, 2, 257, seed=16)
case("pal", 290, 1, 3, 270, seed=17)
# gradients with noise
case("grad", 64, 48, 2, seed=18)
case("grad", 65, 65, 3, seed=19)
case("grad", 200, 31, 2, seed=20)
# sampling strides above 1 (104 000 pixels: histogram stride 2, decision stride 5)
case("stride", 400, 260, 2, 1000, seed=21)
case("missed", 400, 260, 2, 400, seed=22)
case("missed", 400, 260, 3, 400, seed=23)
# presets 0 and 2 (preset 2 small: its Zopfli-style DEFLATE is slow under the interpreter)
case("pal", 33, 16, 2, 300, seed=24, preset=0)
case("pal", 33, 16, 3, 300, seed=25, preset=0)
case("palblk", 65, 33, 2, 400, seed=26, preset=0)
case("pal", 20, 16, 2, 257, seed=27, preset=2)
case("pal", 20, 16, 3, 300, seed=28, preset=2)
# inputs that take the lossless path: <= 256 colours, > 8 192 in the decision sample, Gray, GrayAlpha
case("pal", 33, 16, 2, 200, seed=29)
case("pal", 33, 16, 3, 256, seed=30)
case("noise", 200, 64, 2, seed=31)
case("noise", 100, 100, 3, seed=32)
case("gray", 45, 30, 0, seed=33)
case("gray", 45, 30, 1, seed=34)
# pixo's truncation case: > 8 192 histogram colours (tests pass the palette read back from the file)
case("trunc", 256, 256, 2, 12000, seed=35)
case("trunc", 256, 256, 3, 12000, seed=36)


def _one(i):
    c = CASES[i]
    img = make_quantize_input(c["kind"], c["w"], c["h"], (1, 2, 3, 4)[c["ct"]], c["seed"], c["n"])
    out = gg.run(["png", c["w"], c["h"], c["ct"], c["preset"], 1], img)
    name = f"q{i:03d}.png"
    open(os.path.join(OUT, name), "wb").write(out)
    return dict(c, file=name, input_sha256=hashlib.sha256(img.tobytes()).hexdigest())


def main():
    wb.build()
    os.makedirs(OUT, exist_ok=True)
    manifest = {"source": "pixo_bg.wasm from leerob/pixo @ 437bf63 (web/src/lib/pixo-wasm), sha256 " +
                hashlib.sha256(open(gg.WASM, "rb").read()).hexdigest(),
                "runner": "oracle/wasm_ref/wasm_ref.c", "inputs": "tests/quantize_inputs.py",
                "lossy": 1, "png": []}
    with ProcessPoolExecutor(max(1, (os.cpu_count() or 2) - 1)) as ex:
        manifest["png"] = list(ex.map(_one, range(len(CASES))))
    json.dump(manifest, open(os.path.join(OUT, "manifest.json"), "w"), indent=1)
    total = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print(f"{len(CASES)} PNG fixtures, {total / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
