#!/usr/bin/env python
"""Generates tests/golden/trellis/* by running the reference ITSELF: pixo's committed WebAssembly build
(web/src/lib/pixo-wasm/pixo_bg.wasm of a pixo checkout) executed by oracle/wasm_ref, encodeJpeg at
preset 2 (max: progressive, trellis quantisation, optimised Huffman tables).  The subsampling argument
overrides the preset's 4:2:0, so 4:4:4 files are max-preset files too.

    python oracle/wasm_ref/gen_golden_trellis.py <pixo checkout>

Every fixture is a complete JPEG file; manifest.json says how to regenerate each input
(tests/trellis_inputs.py) and gives its SHA-256.  The tests re-encode coefficient arrays with a
restatement of pixo's progressive scan writer (tests/jpeg_progressive_scans.py) and compare the 7 scans.
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
from trellis_inputs import make_trellis_input  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "trellis")
MODES = [(2, 1), (2, 0), (0, 0)]          # (color_type, subsampling_420): RGB 4:2:0, RGB 4:4:4, Gray
KINDS = ["noise", "smooth", "gradient", "primaries", "hifreq"]
QUALS = [1, 25, 50, 75, 80, 90, 95, 100]

CASES = []
i = 0
for ct, s420 in MODES:
    for (w, h) in [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 17), (70, 45), (100, 75)]:
        CASES.append(dict(w=w, h=h, ct=ct, s420=s420, kind=KINDS[i % 5], q=QUALS[i % 8], seed=i))
        i += 1
    for kind, q in [("smooth", 80), ("hifreq", 90), ("noise", 50)]:
        CASES.append(dict(w=256, h=256, ct=ct, s420=s420, kind=kind, q=q, seed=i))
        i += 1
for q in QUALS:                              # every quality on 4:2:0 noise and on ZRL content
    CASES.append(dict(w=70, h=45, ct=2, s420=1, kind="noise", q=q, seed=100 + q))
    CASES.append(dict(w=40, h=33, ct=2, s420=0, kind="hifreq", q=q, seed=200 + q))
CASES.append(dict(w=512, h=384, ct=2, s420=1, kind="smooth", q=85, seed=3))
CASES.append(dict(w=520, h=390, ct=0, s420=0, kind="primaries", q=75, seed=4))


def _one(k):
    c = CASES[k]
    img = make_trellis_input(c["kind"], c["w"], c["h"], 1 if c["ct"] == 0 else 3, c["seed"])
    out = gg.run(["jpeg", c["w"], c["h"], c["ct"], c["q"], 2, c["s420"]], img)
    name = f"t{k:03d}.jpg"
    open(os.path.join(OUT, name), "wb").write(out)
    return dict(c, preset=2, file=name, input_sha256=hashlib.sha256(img.tobytes()).hexdigest())


def main():
    wb.build()
    os.makedirs(OUT, exist_ok=True)
    manifest = {"source": "pixo_bg.wasm from leerob/pixo @ 437bf63 (web/src/lib/pixo-wasm), sha256 " +
                hashlib.sha256(open(gg.WASM, "rb").read()).hexdigest(),
                "runner": "oracle/wasm_ref/wasm_ref.c", "inputs": "tests/trellis_inputs.py", "jpeg": []}
    with ProcessPoolExecutor(max(1, (os.cpu_count() or 2) - 1)) as ex:
        manifest["jpeg"] = list(ex.map(_one, range(len(CASES))))
    json.dump(manifest, open(os.path.join(OUT, "manifest.json"), "w"), indent=1)
    total = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print(f"{len(CASES)} JPEG fixtures, {total / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
