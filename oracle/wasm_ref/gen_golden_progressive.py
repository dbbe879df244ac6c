#!/usr/bin/env python
"""Generates tests/golden/progressive/* by running the reference ITSELF: pixo's committed WebAssembly
build (web/src/lib/pixo-wasm/pixo_bg.wasm of a pixo checkout) executed by oracle/wasm_ref, encodeJpeg at
preset 2 (max: progressive, trellis quantisation, optimised Huffman tables), on the mostly flat frames of
tests/progressive_inputs.py, whose Y AC scans hold EOB runs of 32 766, 32 767, 32 768 and 69 999 empty
blocks (0x7FFF flushes, and EOBRUN symbols the tables lack).  The subsampling argument overrides the
preset's 4:2:0.  Under the interpreter a file takes 20-80 s.

    python oracle/wasm_ref/gen_golden_progressive.py <pixo checkout>

The wasm API cannot set a restart interval, plain rounding or standard tables with progressive scans:
those options are pinned by oracle/jpeg_progressive.c alone.
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
from progressive_inputs import CASES, make_progressive_input  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "progressive")


def _one(k):
    c = CASES[k]
    img = make_progressive_input(c)
    out = gg.run(["jpeg", c["w"], c["h"], c["ct"], c["q"], 2, c["s420"]], img)
    name = f"g{k:03d}.jpg"
    open(os.path.join(OUT, name), "wb").write(out)
    return dict(c, preset=2, file=name, input_sha256=hashlib.sha256(img.tobytes()).hexdigest())


def main():
    wb.build()
    os.makedirs(OUT, exist_ok=True)
    manifest = {"source": "pixo_bg.wasm from leerob/pixo @ 437bf63 (web/src/lib/pixo-wasm), sha256 " +
                hashlib.sha256(open(gg.WASM, "rb").read()).hexdigest(),
                "runner": "oracle/wasm_ref/wasm_ref.c", "inputs": "tests/progressive_inputs.py", "jpeg": []}
    with ProcessPoolExecutor(max(1, min(len(CASES), (os.cpu_count() or 2) - 1))) as ex:
        manifest["jpeg"] = list(ex.map(_one, range(len(CASES))))
    json.dump(manifest, open(os.path.join(OUT, "manifest.json"), "w"), indent=1)
    total = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print(f"{len(CASES)} JPEG fixtures, {total / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
