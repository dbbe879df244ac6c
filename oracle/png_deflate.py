"""ctypes binding of oracle/png_deflate.c, pixo's deflate_zlib_packed at levels 1-9 (test infrastructure), and
pixo's PNG chunk writers in Python: write_chunk (src/png/chunk.rs:10), write_ihdr / write_idat_chunks / write_iend
(src/png/mod.rs:592-630).  The library built here goes to oracle/libpng_deflate.so, as png_quantize's does.

deflate_zlib(data, level) -> bytes            the whole zlib stream
deflate_kind(data, level) -> 0 | 1 | 2        stored, fixed or dynamic
lz77(data, level) -> uint32 array             pixo's packed tokens
histogram(tokens) -> (lit[286], dist[30])     symbol counts, before the EOB and the dist_freqs[0] = 1 rule
code_lengths(freqs, max_len) -> uint8 array   build_codes' lengths
"""
from __future__ import annotations

import ctypes as C
import os
import struct
import subprocess
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libpng_deflate.so")
SIGNATURE = b"\x89PNG\r\n\x1a\n"
IDAT_CHUNK = 256 * 1024


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "png_deflate.c")
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(src):
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-fPIC", "-Wall", "-shared", "-o", SO, src])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        p, z = C.c_void_p, C.c_size_t
        L.pd_lz77.argtypes, L.pd_lz77.restype = [p, z, C.c_int, p], z
        L.pd_code_lengths.argtypes = [p, C.c_int, C.c_int, p]
        L.pd_histogram.argtypes = [p, z, p, p]
        L.pd_high_entropy.argtypes, L.pd_high_entropy.restype = [p, z], C.c_int
        L.pd_deflate_zlib.argtypes, L.pd_deflate_zlib.restype = [p, z, C.c_int, p, z, p], z
        _lib = L
    return _lib


def _u8(data) -> np.ndarray:
    return np.ascontiguousarray(np.frombuffer(bytes(data), np.uint8) if isinstance(data, (bytes, bytearray))
                                else np.asarray(data, np.uint8).reshape(-1))


def _deflate(data, level):
    d = _u8(data)
    n = lib().pd_deflate_zlib(d.ctypes.data, d.size, level, None, 0, None)
    out = np.empty(max(n, 1), np.uint8)
    kind = C.c_int()
    lib().pd_deflate_zlib(d.ctypes.data, d.size, level, out.ctypes.data, n, C.byref(kind))
    return out[:n].tobytes(), kind.value


def deflate_zlib(data, level: int) -> bytes:
    return _deflate(data, level)[0]


def deflate_kind(data, level: int) -> int:
    return _deflate(data, level)[1]


def lz77(data, level: int) -> np.ndarray:
    d = _u8(data)
    t = np.empty(max(d.size, 1), np.uint32)
    n = lib().pd_lz77(d.ctypes.data, d.size, level, t.ctypes.data)
    return t[:n].copy()


def histogram(tokens: np.ndarray):
    t = np.ascontiguousarray(tokens, np.uint32)
    lit, dist = np.zeros(286, np.uint32), np.zeros(30, np.uint32)
    lib().pd_histogram(t.ctypes.data, t.size, lit.ctypes.data, dist.ctypes.data)
    return lit, dist


def code_lengths(freqs, max_len: int) -> np.ndarray:
    f = np.ascontiguousarray(freqs, np.uint32)
    out = np.zeros(f.size, np.uint8)
    lib().pd_code_lengths(f.ctypes.data, f.size, max_len, out.ctypes.data)
    return out


def high_entropy(data) -> bool:
    d = _u8(data)
    return bool(lib().pd_high_entropy(d.ctypes.data, d.size))


def chunk(kind: bytes, payload: bytes) -> bytes:
    """chunk::write_chunk (src/png/chunk.rs:10): length, type, data, CRC-32 of type and data."""
    return struct.pack(">I", len(payload)) + kind + payload + struct.pack(">I", zlib.crc32(kind + payload))


def png_file(width: int, height: int, bit_depth: int, color_type_byte: int, zstream: bytes,
             palette=None, trns: bytes | None = None) -> bytes:
    """encode_into's container (src/png/mod.rs:437-630): signature, IHDR, PLTE and tRNS when given, the zlib stream
    in IDAT chunks of 256 KiB, IEND.  palette: (n, 3 or 4) RGB(A) rows; PLTE takes their RGB."""
    out = SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", width, height, bit_depth, color_type_byte, 0, 0, 0))
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8)[:, :3].tobytes())
    if trns:
        out += chunk(b"tRNS", bytes(trns))
    for i in range(0, len(zstream), IDAT_CHUNK):
        out += chunk(b"IDAT", zstream[i:i + IDAT_CHUNK])
    return out + chunk(b"IEND", b"")


def chunks(png: bytes):
    """[(type, payload)] of a PNG file after its signature."""
    assert png[:8] == SIGNATURE
    out, i = [], 8
    while i < len(png):
        n = struct.unpack(">I", png[i:i + 4])[0]
        out.append((png[i + 4:i + 8], png[i + 8:i + 8 + n]))
        i += 12 + n
    return out
