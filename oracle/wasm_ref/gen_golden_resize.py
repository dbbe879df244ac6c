#!/usr/bin/env python
"""Generates tests/golden/resize/* by running the reference ITSELF: pixo's committed WebAssembly build
(web/src/lib/pixo-wasm/pixo_bg.wasm of a pixo checkout) executed by oracle/wasm_ref/resize_ref.c.

  r*.raw      resizeImage on the frames of tests/resize_inputs.py (every geometry x 4 colour types x 3
              algorithms), with manifest.json
  sinf.npy    (x, sin x) f32 pairs of the wasm's own sinf: every argument in a sweep of every 64th f32 of
              [-3pi, 3pi] where it differs from (float)sin((double)x), plus every 65536th argument

    python oracle/wasm_ref/gen_golden_resize.py <pixo checkout>            # the fixtures
    python oracle/wasm_ref/gen_golden_resize.py <pixo checkout> --check    # oracle sinf vs the wasm's, every
                                                                           # f32 in [-3pi, 3pi] (~10 CPU-min)
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from resize_inputs import CASES, make_resize_input  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(HERE, "resize_ref")
WASM = os.path.join(sys.argv[1] if len(sys.argv) > 1 else ".", "web", "src", "lib", "pixo-wasm", "pixo_bg.wasm")
OUT = os.path.join(ROOT, "tests", "golden", "resize")
TOP = 0x4116CBE4   # the f32 nearest 3pi


def build() -> str:
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-msse2", "-mfpmath=sse", "-w",
                           os.path.join(HERE, "resize_ref.c"), "-lm", "-o", EXE])
    return EXE


def _one(k):
    c = CASES[k]
    img = make_resize_input(c)
    with tempfile.TemporaryDirectory() as td:
        src, dst = os.path.join(td, "in.raw"), os.path.join(td, "out.raw")
        img.tofile(src)
        subprocess.check_call([EXE, WASM, "resize", src] + [str(c[f]) for f in ("sw", "sh", "dw", "dh", "ct", "alg")]
                              + [dst])
        out = open(dst, "rb").read()
    name = f"r{k:03d}.raw"
    open(os.path.join(OUT, name), "wb").write(out)
    return dict(c, file=name, input_sha256=hashlib.sha256(img.tobytes()).hexdigest())


def _sweep(args):
    first, last, step, which = args
    with tempfile.TemporaryDirectory() as td:
        p = os.path.join(td, "s.bin")
        subprocess.check_call([EXE, WASM, "sinf", hex(first), hex(last), str(step), which, p], stderr=subprocess.DEVNULL)
        return np.fromfile(p, np.uint32).reshape(-1, 2)


def _chunks(n):
    return [(s + k * (TOP + 1) // n, s + (k + 1) * (TOP + 1) // n - 1) for s in (0, 0x80000000) for k in range(n)]


def _check(rng):
    out = subprocess.run([EXE, WASM, "check", hex(rng[0]), hex(rng[1])], capture_output=True, text=True)
    return [int(v) for v in out.stdout.split()[1::2]]


def main():
    build()
    jobs = max(1, (os.cpu_count() or 2) - 1)
    if "--check" in sys.argv:
        with ProcessPoolExecutor(jobs) as ex:
            res = np.array(list(ex.map(_check, _chunks(2 * jobs)))).sum(0)
        print(f"checked {res[0]} f32 arguments: {res[1]} differ from oracle/resize.c's rz_sinf, "
              f"{res[2]} from (float)sin((double)x)")
        return
    os.makedirs(OUT, exist_ok=True)
    manifest = {"source": "pixo_bg.wasm from leerob/pixo @ 437bf63 (web/src/lib/pixo-wasm), sha256 " +
                hashlib.sha256(open(WASM, "rb").read()).hexdigest(),
                "runner": "oracle/wasm_ref/resize_ref.c", "inputs": "tests/resize_inputs.py"}
    with ProcessPoolExecutor(jobs) as ex:
        manifest["resize"] = list(ex.map(_one, range(len(CASES))))
        differ = np.concatenate(list(ex.map(_sweep, [(a, b, 64, "differ") for a, b in _chunks(2 * jobs)])))
        spread = np.concatenate(list(ex.map(_sweep, [(a, b, 65536, "all") for a, b in _chunks(2)])))
    pairs = np.unique(np.concatenate([differ, spread]), axis=0)
    np.save(os.path.join(OUT, "sinf.npy"), pairs)
    manifest["sinf"] = {"file": "sinf.npy", "pairs": int(len(pairs)), "dense_sweep_step": 64,
                        "differ_from_double_sin": int(len(differ)),
                        "spread_step": 65536}
    json.dump(manifest, open(os.path.join(OUT, "manifest.json"), "w"), indent=1)
    total = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print(f"{len(CASES)} resize fixtures, {len(pairs)} sinf pairs ({len(differ)} differ from double sin), "
          f"{total / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
