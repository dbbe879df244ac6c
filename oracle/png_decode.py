"""CPU restatement of pixo's PNG decoder, pixo::decode::decode_png (test infrastructure): oracle/png_decode.c, built
here into oracle/libpng_decode.so.  Checked by tests/test_png_decode.py against real pixo files (the 225 PNG goldens
decode to their generator inputs), against zlib and PIL on valid streams, and against an independent pure-Python
restatement (tests/png_decode_ref.py) on constructed files.

decode(data) -> Decoded(kind, message, width, height, color_type, pixels)
    kind: OK, INVALID (Error::InvalidDecode), UNSUPPORTED (Error::UnsupportedDecode), DIMENSIONS
    (Error::InvalidDimensions), TOO_LARGE (Error::ImageTooLarge); message: pixo's Display text
inflate_zlib(data, expected) -> (kind, message, bytes)   inflate_zlib_with_size(data, Some(expected))
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libpng_decode.so")
SOURCES = ["png_decode.c"]
OK, INVALID, UNSUPPORTED, DIMENSIONS, TOO_LARGE = 0, 1, 2, 3, 4


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, s) for s in SOURCES]
    if force or not os.path.exists(SO) or any(os.path.getmtime(SO) < os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-fPIC", "-Wall", "-shared", "-o", SO] + srcs)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        p = C.c_void_p
        L.pd_decode.argtypes = [p, C.c_size_t, p, p, p]
        L.pd_decode.restype = None
        L.pd_inflate_zlib.argtypes = [p, C.c_size_t, C.c_uint64, p, C.c_size_t, p, p]
        L.pd_inflate_zlib.restype = None
        L.pd_crc32.argtypes = [p, C.c_size_t]
        L.pd_crc32.restype = C.c_uint32
        _lib = L
    return _lib


@dataclasses.dataclass
class Decoded:
    kind: int
    message: str
    width: int = 0
    height: int = 0
    color_type: int = 0
    pixels: np.ndarray | None = None


def _buf(data):
    b = np.frombuffer(bytes(data), np.uint8)
    return b, (b.ctypes.data if b.size else None)


def decode(data, pixels: bool = True) -> Decoded:
    b, ptr = _buf(data)
    info = np.zeros(8, np.uint64)
    msg = C.create_string_buffer(256)
    lib().pd_decode(ptr, b.size, None, info.ctypes.data, msg)
    kind = int(info[0])
    if kind != OK:
        return Decoded(kind, msg.value.decode("utf-8", "replace"))
    px = None
    if pixels:
        px = np.zeros(int(info[4]), np.uint8)
        lib().pd_decode(ptr, b.size, px.ctypes.data, info.ctypes.data, msg)
    return Decoded(kind, "", int(info[1]), int(info[2]), int(info[3]), px)


def inflate_zlib(data, expected: int):
    b, ptr = _buf(data)
    info = np.zeros(2, np.uint64)
    msg = C.create_string_buffer(256)
    lib().pd_inflate_zlib(ptr, b.size, expected, None, 0, info.ctypes.data, msg)
    out = np.zeros(max(int(info[1]), 1), np.uint8)
    lib().pd_inflate_zlib(ptr, b.size, expected, out.ctypes.data, out.size, info.ctypes.data, msg)
    return int(info[0]), msg.value.decode("utf-8", "replace"), out[:int(info[1])].tobytes()


def crc32(data) -> int:
    b, ptr = _buf(data)
    return int(lib().pd_crc32(ptr, b.size))
