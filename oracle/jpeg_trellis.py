"""CPU restatement of pixo's trellis quantiser (test infrastructure): oracle/jpeg_trellis.c, built here
with the block extraction and DCT of oracle/pixo_oracle.c into oracle/libjpeg_trellis.so (strict
binary32).  Checked by tests/test_jpeg_trellis.py against real pixo output - the max-preset files of
tests/golden/trellis/ (pixo's wasm build, oracle/wasm_ref/gen_golden_trellis.py), every scan re-encoded
from this oracle's coefficients by tests/jpeg_progressive_scans.py - and against an independent
pure-Python restatement (tests/trellis_ref.py) on constructed blocks.

trellis_quantize(dct, q, lam=None) -> int16[64]        (lam None = pixo's DEFAULT_LAMBDA 1.0)
trellis_lambda(quality) -> float                        (trellis_quantize_adaptive's formula)
jpeg_coefficients(data, w, h, ct, ss, quality) -> (y, cb, cr)   use_trellis = true
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libjpeg_trellis.so")
SOURCES = ["jpeg_trellis.c", "pixo_oracle.c"]


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, s) for s in SOURCES]
    if force or not os.path.exists(SO) or any(os.path.getmtime(SO) < os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-fno-fast-math", "-msse2",
                               "-mfpmath=sse", "-fPIC", "-Wall", "-shared", "-o", SO] + srcs + ["-lm"])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        p = C.c_void_p
        L.po_trellis_quantize.argtypes = [p, p, C.c_float, p]
        L.po_trellis_lambda.argtypes = [C.c_int]
        L.po_trellis_lambda.restype = C.c_float
        L.po_jpeg_coefficients_trellis.argtypes = [p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, p, p, p, p, p]
        L.po_quant_tables.argtypes = [C.c_int, p, p, p, p]
        _lib = L
    return _lib


def trellis_lambda(quality: int) -> float:
    return float(np.float32(lib().po_trellis_lambda(int(quality))))


def trellis_quantize(dct, q, lam=None) -> np.ndarray:
    d = np.ascontiguousarray(dct, np.float32).reshape(64)
    qq = np.ascontiguousarray(q, np.float32).reshape(64)
    out = np.zeros(64, np.int16)
    lib().po_trellis_quantize(d.ctypes.data, qq.ctypes.data, 1.0 if lam is None else float(np.float32(lam)),
                              out.ctypes.data)
    return out


def trellis_quantize_blocks(dct, q, lam=None) -> np.ndarray:
    d = np.ascontiguousarray(dct, np.float32).reshape(-1, 64)
    return np.stack([trellis_quantize(b, q, lam) for b in d]) if len(d) else np.zeros((0, 64), np.int16)


def quant_tables(quality: int):
    lz = np.zeros(64, np.uint8); cz = np.zeros(64, np.uint8)
    ln = np.zeros(64, np.float32); cn = np.zeros(64, np.float32)
    lib().po_quant_tables(int(quality), lz.ctypes.data, cz.ctypes.data, ln.ctypes.data, cn.ctypes.data)
    return ln, cn


def jpeg_coefficients(data, w, h, color_type=2, subsampling=1, quality=80, lum_q=None, chr_q=None):
    """compute_all_coefficients(.., use_trellis = true) -> (y, cb, cr) int16 [n, 64], natural order."""
    d = np.ascontiguousarray(np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data,
                             np.uint8).reshape(-1)
    if lum_q is None:
        lum_q, chr_q = quant_tables(quality)
    lq = np.ascontiguousarray(lum_q, np.float32); cq = np.ascontiguousarray(chr_q, np.float32)
    if color_type == 0 or subsampling == 0:
        ny = ((w + 7) // 8) * ((h + 7) // 8)
        nc = 0 if color_type == 0 else ny
    else:
        ny = ((w + 15) // 16) * ((h + 15) // 16) * 4
        nc = ny // 4
    y = np.zeros((ny, 64), np.int16)
    cb = np.zeros((max(nc, 1), 64), np.int16)
    cr = np.zeros((max(nc, 1), 64), np.int16)
    lib().po_jpeg_coefficients_trellis(d.ctypes.data, w, h, color_type, subsampling, lq.ctypes.data,
                                       cq.ctypes.data, y.ctypes.data, cb.ctypes.data, cr.ctypes.data)
    return y, cb[:nc], cr[:nc]
