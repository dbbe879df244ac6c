"""CPU restatement of pixo's progressive encoder (test infrastructure): oracle/jpeg_progressive.c, built
here with oracle/pixo_oracle.c and oracle/jpeg_trellis.c into oracle/libjpeg_progressive.so (strict
binary32).  Pinned by tests/test_jpeg_progressive.py to real pixo output - the max-preset files of
tests/golden/trellis/ and tests/golden/progressive/, reproduced whole - and to the Python scan
restatement tests/jpeg_progressive_scans.py on constructed coefficient arrays.

encode(data, w, h, ct, ss, quality, restart, optimize, trellis) -> bytes   (a whole progressive file)
scans(y, cb, cr, dht) -> [7 entropy-coded segments]   dht: uint8 [4, 272] (counts + values per table)
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libjpeg_progressive.so")
SOURCES = ["jpeg_progressive.c", "jpeg_trellis.c", "pixo_oracle.c"]


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
        L.po_jpeg_encode_progressive.restype = C.c_long
        L.po_jpeg_encode_progressive.argtypes = [p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int,
                                                 C.c_uint32, C.c_int, C.c_int, p, C.c_size_t]
        L.po_progressive_scans.restype = C.c_long
        L.po_progressive_scans.argtypes = [p, C.c_size_t, p, p, C.c_size_t, p, p, C.c_size_t, p]
        _lib = L
    return _lib


def encode(data, w, h, ct=2, ss=1, quality=80, restart=0, optimize=True, trellis=True) -> bytes:
    d = np.ascontiguousarray(np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data,
                             np.uint8).reshape(-1)
    cap = d.size * 4 + (1 << 20)
    out = np.empty(cap, np.uint8)
    n = lib().po_jpeg_encode_progressive(d.ctypes.data, d.size, w, h, ct, quality, ss, restart or 0,
                                         int(optimize), int(trellis), out.ctypes.data, cap)
    if n < 0:
        raise ValueError(f"po_jpeg_encode_progressive error {n}")
    return out[:n].tobytes()


def scans(y, cb, cr, dht) -> list[bytes]:
    y = np.ascontiguousarray(y, np.int16).reshape(-1, 64)
    cb = np.ascontiguousarray(cb, np.int16).reshape(-1, 64)
    cr = np.ascontiguousarray(cr, np.int16).reshape(-1, 64)
    nc = len(cb)
    cb_ = cb if nc else np.zeros((1, 64), np.int16)
    cr_ = cr if nc else np.zeros((1, 64), np.int16)
    d = np.ascontiguousarray(dht, np.uint8).reshape(4, 272)
    cap = (len(y) + 2 * nc) * 64 * 8 + 4096
    out = np.empty(cap, np.uint8)
    lens = (C.c_size_t * 7)()
    n = lib().po_progressive_scans(y.ctypes.data, len(y), cb_.ctypes.data, cr_.ctypes.data, nc, d.ctypes.data,
                                   out.ctypes.data, cap, lens)
    if n < 0:
        raise ValueError("po_progressive_scans: capacity")
    res, o = [], 0
    for s in range(7):
        res.append(out[o:o + lens[s]].tobytes())
        o += lens[s]
    return res
