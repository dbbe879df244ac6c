"""CPU restatement of pixo's baseline JPEG decoder, pixo::decode::decode_jpeg (test infrastructure):
oracle/jpeg_decode.c, built here into oracle/libjpeg_decode.so.  Checked by tests/test_jpeg_decode.py against
real pixo files (the coefficients it decodes from tests/golden/j*.jpg equal the encoder oracle's) and against
an independent pure-Python restatement (tests/jpeg_decode_ref.py) on constructed files.

decode(data) -> Decoded(status, message, width, height, color_type, pixels, coefs, stored)
    status: OK, INVALID (Error::InvalidDecode), UNSUPPORTED (Error::UnsupportedDecode), PANIC (a file pixo
    panics on); coefs: int16 [blocks, 64] in zig-zag order, in decode order; stored: blocks the scan stored
idct_block(coef, q) -> uint8[64]         dequantize + idct_2d_integer
find_entropy_end(data) -> int
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libjpeg_decode.so")
SOURCES = ["jpeg_decode.c"]
OK, INVALID, UNSUPPORTED, PANIC = 0, 1, 2, 3


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, s) for s in SOURCES]
    if force or not os.path.exists(SO) or any(os.path.getmtime(SO) < os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-fwrapv", "-fPIC", "-Wall", "-shared", "-o", SO] + srcs)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        p = C.c_void_p
        L.jd_decode.argtypes = [p, C.c_size_t, p, p, p, p]
        L.jd_decode.restype = None
        L.jd_idct_block.argtypes = [p, p, p]
        L.jd_idct_block.restype = None
        L.jd_find_entropy_end.argtypes = [p, C.c_size_t]
        L.jd_find_entropy_end.restype = C.c_size_t
        _lib = L
    return _lib


@dataclasses.dataclass
class Decoded:
    status: int
    message: str
    width: int = 0
    height: int = 0
    color_type: int = 0
    pixels: np.ndarray | None = None
    coefs: np.ndarray | None = None
    stored: int = 0
    blocks: int = 0


def _buf(data: bytes):
    b = np.frombuffer(bytes(data), np.uint8)
    return b, (b.ctypes.data if b.size else None)


def decode(data, pixels: bool = True, coefs: bool = True) -> Decoded:
    b, ptr = _buf(data)
    info = np.zeros(8, np.uint64)
    msg = C.create_string_buffer(256)
    lib().jd_decode(ptr, b.size, None, None, info.ctypes.data, msg)
    st = int(info[0])
    if st != OK:
        return Decoded(st, msg.value.decode())
    px = np.zeros(max(int(info[7]), 1), np.uint8)
    k = np.zeros((max(int(info[5]), 1), 64), np.int16)
    lib().jd_decode(ptr, b.size, px.ctypes.data if pixels else None, k.ctypes.data if coefs else None,
                    info.ctypes.data, msg)
    stored = int(info[6])
    return Decoded(st, "", int(info[1]), int(info[2]), int(info[3]), px[:int(info[7])] if pixels else None,
                   k[:stored] if coefs else None, stored, int(info[5]))


def idct_block(coef, q) -> np.ndarray:
    c = np.ascontiguousarray(coef, np.int16).reshape(64)
    qq = np.ascontiguousarray(q, np.uint16).reshape(64)
    out = np.zeros(64, np.uint8)
    lib().jd_idct_block(c.ctypes.data, qq.ctypes.data, out.ctypes.data)
    return out


def find_entropy_end(data) -> int:
    b, ptr = _buf(data)
    return int(lib().jd_find_entropy_end(ptr, b.size))
