"""Reference progressive files (test infrastructure), composed from oracles that are pinned on their own:

- the frame headers (SOI, APP0, DQT, DHT, DRI) of the baseline file the C oracle writes for the same
  options (oracle/pyoracle.py, pinned to real pixo by tests/test_golden_reference.py), with SOF0 turned
  into SOF2: pixo writes the same headers and the same tables for both (src/jpeg/mod.rs:379-410; the
  optimised tables come from the plain-rounded statistics, restart interval included, in both);
- the coefficients of compute_all_coefficients: oracle/jpeg_trellis.c with trellis_quant, else
  oracle/pixo_oracle.c;
- the 7 scans of tests/jpeg_progressive_scans.py, coded with the tables read back from that DHT.

tests/test_jpeg_progressive.py checks that this reproduces every real-pixo max-preset file of
tests/golden/trellis/ whole.
"""
from __future__ import annotations

import numpy as np

import jpeg_progressive_scans as ps
from oracle import jpeg_trellis as jt
from oracle import pyoracle as po

SOS = [bytes([0xFF, 0xDA, 0, 8, 1, comp + 1, 0x11 if comp else 0x00, ss, se, 0]) for comp, ss, se in ps.SCRIPT]


def frame_headers(baseline: bytes) -> bytes:
    """SOI .. DRI of a baseline file, with its SOF0 marker turned into SOF2."""
    out = bytearray(baseline[:2])
    i = 2
    while True:
        m = baseline[i + 1]
        n = (baseline[i + 2] << 8) | baseline[i + 3]
        if m == 0xDA:
            return bytes(out)
        seg = bytearray(baseline[i:i + 2 + n])
        if m == 0xC0:
            seg[1] = 0xC2
        out += seg
        i += 2 + n


def coefficients(img, w, h, ct, ss, q, trellis):
    if trellis:
        return jt.jpeg_coefficients(img, w, h, ct, ss, q)
    return po.jpeg_coefficients(img, w, h, ct, ss, q)


def assemble(headers: bytes, segments) -> bytes:
    out = bytearray(headers)
    for sos, seg in zip(SOS, segments):
        out += sos + seg
    return bytes(out + b"\xff\xd9")


def encode(img, w, h, ct=2, ss=1, q=80, restart=0, optimize=True, trellis=True) -> bytes:
    """The file pixo's encode_into writes with progressive = true and these options."""
    base = po.jpeg_encode(img, w, h, ct, q, ss, restart or 0, optimize)
    y, cb, cr = coefficients(img, w, h, ct, ss, q, trellis)
    return assemble(frame_headers(base), ps.encode_scans(y, cb, cr, ps.dht(base)))
