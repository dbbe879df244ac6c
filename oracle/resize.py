"""ctypes wrapper of oracle/resize.c, the C restatement of pixo's resizers and of the sinf its wasm build
runs (test infrastructure), built here into oracle/libresize.so.

resize(data, sw, sh, dw, dh, ct, alg) -> uint8 array, or raises OracleError(status)
contrib(src, dst) -> (start, count, offset, weights)      Lanczos3 tables of one axis
sinf(x) -> float32 array
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libresize.so")


class OracleError(Exception):
    def __init__(self, code: int):
        super().__init__(f"resize status {code}")
        self.code = code


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "resize.c")
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-fno-fast-math", "-msse2",
                               "-mfpmath=sse", "-fPIC", "-Wall", "-shared", "-o", SO, src, "-lm"])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        p, u32 = C.c_void_p, C.c_uint32
        L.rz_sinf_many.argtypes = [p, p, C.c_size_t]
        L.rz_contrib.argtypes = [u32, u32, p, p, p, p]
        L.rz_contrib.restype = C.c_size_t
        L.rz_resize.argtypes = [p, C.c_size_t, u32, u32, u32, u32, u32, u32, p]
        _lib = L
    return _lib


def sinf(x) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty_like(x)
    lib().rz_sinf_many(x.ctypes.data, y.ctypes.data, x.size)
    return y


def contrib(src: int, dst: int):
    start, count = np.empty(dst, np.uint32), np.empty(dst, np.uint32)
    offset = np.empty(dst, np.uint64)
    n = lib().rz_contrib(src, dst, start.ctypes.data, count.ctypes.data, offset.ctypes.data, None)
    w = np.empty(max(n, 1), np.float32)
    lib().rz_contrib(src, dst, None, None, None, w.ctypes.data)
    return start, count, offset, w[:n]


def resize(data, sw: int, sh: int, dw: int, dh: int, ct: int, alg: int) -> np.ndarray:
    d = np.ascontiguousarray(np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else data,
                             np.uint8).reshape(-1)
    bpp = ct + 1 if 0 <= ct <= 3 else 1
    out = np.empty(max(int(dw) * int(dh) * bpp, 1) if 0 < dw <= 1 << 24 and 0 < dh <= 1 << 24 else 1, np.uint8)
    rc = lib().rz_resize(d.ctypes.data, d.size, sw, sh, dw, dh, ct, alg, out.ctypes.data)
    if rc:
        raise OracleError(rc)
    return out[:int(dw) * int(dh) * bpp]
