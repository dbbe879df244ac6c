"""Constructed JPEG files for the decoder tests: seeded, so the CPU and GPU tests see the same bytes.

  constructed(seed)   a baseline file built from random headers and a random scan: sampling factors 1-4 per axis
                      (non-dividing ratios too), sometimes after an earlier SOF0 with factors up to 15 whose maxima
                      pixo keeps, 8- or 16-bit DQT (products that overflow the IDCT's i32), DHT tables
                      with arbitrary counts and values (DC categories up to 255, oversubscribed code spaces), restart
                      intervals with RSTn markers in the scan, stuffed bytes, fill bytes, garbage between markers,
                      and APPn / COM / unknown segments
  truncations(data)   every prefix of a file
  corrupted(data, seed, n)  copies with scan bytes replaced
"""
from __future__ import annotations

import struct

import numpy as np


def seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


def sof0(w: int, h: int, comps: bytes) -> bytes:
    """an 8-bit SOF0 segment; comps: 3 bytes (id, sampling, quantisation table) per component"""
    return seg(0xC0, bytes([8]) + struct.pack(">HH", h, w) + bytes([len(comps) // 3]) + comps)


def _dht(rng, cls: int, tid: int, dc_wild: bool) -> bytes:
    kind = rng.integers(0, 3)
    if kind == 0:    # a small complete code
        bits = [0] * 16
        bits[1], bits[2] = 3, int(rng.integers(1, 6))
    elif kind == 1:  # random counts, possibly oversubscribed
        bits = [int(x) for x in rng.integers(0, 5, 16)]
    else:            # long codes only: the slow path
        bits = [0] * 16
        for i in rng.integers(8, 16, 4):
            bits[int(i)] += 2
    nv = sum(bits)
    if cls == 0:
        vals = rng.integers(0, 256 if dc_wild else 12, nv)
    else:
        vals = rng.integers(0, 256, nv)
        vals[: min(2, nv)] = [0, 0xF0][: min(2, nv)]
    return bytes([cls << 4 | tid]) + bytes(bits) + bytes(int(v) for v in vals)


def _scan(rng, n: int, restart: bool) -> bytes:
    out = bytearray()
    k = 0
    for b in rng.integers(0, 256, n):
        out.append(int(b))
        if b == 0xFF:
            out.append(0x00)
        if restart and rng.random() < 0.02:
            out += bytes([0xFF, 0xD0 + k % 8])
            k += 1
    return bytes(out)


def constructed(seed: int) -> bytes:
    rng = np.random.default_rng(seed)
    ncomp = 1 if rng.random() < 0.3 else 3
    w, h = (int(x) for x in rng.integers(1, 70, 2))
    parts = [b"\xFF\xD8"]
    if rng.random() < 0.5:
        parts.append(seg(0xE0, b"JFIF\x00" + bytes(9)))
    if rng.random() < 0.3:
        parts.append(b"garbage" + b"\xFF" * int(rng.integers(1, 4)))   # skipped by read_marker
    if rng.random() < 0.3:
        parts.append(seg(0xFE, b"comment"))
    if rng.random() < 0.2:
        parts.append(seg(0xF3, b"\x01\x02"))   # an unknown marker with a payload
    for t in range(2):
        if rng.random() < 0.3:
            q = rng.integers(1, 65536, 64)
            parts.append(seg(0xDB, bytes([0x10 | t]) + b"".join(struct.pack(">H", int(x)) for x in q)))
        else:
            parts.append(seg(0xDB, bytes([t]) + bytes(int(x) for x in rng.integers(1, 256, 64))))
    if rng.random() < 0.3:
        # an earlier SOF0 whose sampling maxima pixo keeps: the planes of the real one are then sized by them
        big = bytes(b for c in range(3) for b in (c + 1, int(rng.integers(1, 16)) << 4 | int(rng.integers(1, 16)), 0))
        parts.append(sof0(w, h, big))
    comps = b""
    for c in range(ncomp):
        hs, vs = (int(x) for x in rng.integers(1, 5, 2))
        comps += bytes([c + 1, hs << 4 | vs, min(c, 1)])
    parts.append(sof0(w, h, comps))
    dc_wild = rng.random() < 0.4
    for cls in range(2):
        for t in range(2):
            parts.append(seg(0xC4, _dht(rng, cls, t, dc_wild)))
    restart = rng.random() < 0.4
    if restart:
        parts.append(seg(0xDD, struct.pack(">H", int(rng.integers(1, 6)))))
    sos = bytes([ncomp]) + b"".join(bytes([c + 1, (min(c, 1) << 4) | min(c, 1)]) for c in range(ncomp)) + b"\x00\x3F\x00"
    parts.append(seg(0xDA, sos))
    parts.append(_scan(rng, int(rng.integers(0, 3000)), restart))
    if rng.random() < 0.8:
        parts.append(b"\xFF\xD9")
    return b"".join(parts)


def truncations(data: bytes):
    return [data[:i] for i in range(len(data) + 1)]


def corrupted(data: bytes, seed: int, n: int):
    rng = np.random.default_rng(seed)
    sos = data.rfind(b"\xFF\xDA")
    start = sos + 4 + struct.unpack(">H", data[sos + 2:sos + 4])[0] - 2
    out = []
    for _ in range(n):
        d = bytearray(data)
        for p in rng.integers(start, len(d), 3):
            d[int(p)] = int(rng.integers(0, 256))
        out.append(bytes(d))
    return out
