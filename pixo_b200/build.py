"""Builds libpixo_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

The library is compiled for exactly one target, the H100: -gencode arch=compute_90a,code=sm_90a.
`-fmad=false` keeps the compiler from contracting the reference's separate multiply/add steps
into FMAs (the DCT must round after every operation); the FMAs the quantiser's exact division
needs are written explicitly as `__fmaf_rn` / `__fmaf_rd` (see DESIGN.md section 3).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libpixo_b200.so")
SOURCES = ["api.cu", "api_jpeg.cu", "api_png.cu", "api_decode.cu", "jpeg_transform.cu", "jpeg_trellis.cu", "jpeg_entropy.cu", "jpeg_progressive.cu", "png_filter.cu", "png_reduce.cu", "png_quantize.cu",
           "resize.cu", "jpeg_decode.cu", "png_decode.cu", "png_deflate.cu", "png_encode.cu", "jpeg_host.cpp", "jpeg_decode_host.cpp", "png_decode_host.cpp", "png_host.cpp", "resize_host.cpp"]
HEADERS = ["api.hpp", "common.cuh", "decode_host.hpp", "jpeg_host.hpp", "jpeg_decode_host.hpp", "png_decode_host.hpp", "png_host.hpp", "resize_host.hpp", os.path.join("..", "..", "include", "pixo_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false", "-Xcompiler", "-fPIC,-O2,-fno-fast-math,-ffp-contract=off,-pthread",
    "--shared", "-Xptxas", "-v", "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return SO
    cmd = [_nvcc()] + NVCC_FLAGS + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", SO, "-lpthread"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    log = proc.stdout + proc.stderr
    with open(os.path.join(HERE, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if proc.returncode != 0:
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed building libpixo_b200.so")
    if verbose:
        print(log)
    return SO


if __name__ == "__main__":
    build(force=True, verbose=True)
