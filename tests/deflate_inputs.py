"""Inputs for the DEFLATE tests: the filtered streams inside the real-pixo PNG goldens, and streams built to reach
each branch of pixo's deflate_zlib_packed (src/compress/deflate.rs:1008-1079, src/compress/lz77.rs:403-812)."""
from __future__ import annotations

import json
import os
import zlib

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PRESET_LEVEL = {0: 2, 1: 6}   # PngOptions::from_preset: fast 2, balanced 6 (max runs optimal_compression)


def golden_pngs():
    """[(path, level)] of every real-pixo PNG golden with preset 0 or 1 (preset 2's optimal_compression is out of
    scope)."""
    out = []
    for sub in ("", "reduce", "quantize"):
        base = os.path.join(GOLDEN, sub)
        for e in json.load(open(os.path.join(base, "manifest.json")))["png"]:
            if e["preset"] in PRESET_LEVEL:
                out.append((os.path.join(base, e["file"]), PRESET_LEVEL[e["preset"]]))
    return out


def idat(png: bytes) -> bytes:
    from oracle import png_deflate as pd
    return b"".join(p for k, p in pd.chunks(png) if k == b"IDAT")


def stored_rule_stream() -> bytes:
    """65 535 bytes whose dynamic block at level 6 is 6 bytes longer than the input: should_use_stored counts
    n / 65535 + 1 = 2 block headers (10 bytes) and keeps the dynamic block, although deflate_stored would write
    only one header."""
    rng = np.random.default_rng(1)
    w = np.ones(256)
    w[:16] += 0.875
    d = rng.choice(256, 65535, p=w / w.sum()).astype(np.uint8)
    d[8:16] = d[0:8]
    return d.tobytes()


def small_cases():
    """{name: bytes}: small streams, each built to take one branch of the parse (asserted through deflate_ref)."""
    rng = np.random.default_rng(7)
    noise = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    low = lambda n: rng.integers(100, 120, n, dtype=np.uint8).tobytes()   # 20 symbols: minimum match 3
    head = noise(512)
    fill = lambda n: rng.integers(0, 16, n, dtype=np.uint8).tobytes()
    # "Q A B C" and "A B ... L" apart, then "Q A B ... L": a 4-byte match at Q, a 12-byte one at A
    lazy = fill(60) + bytes(range(200, 204)) + fill(60) + bytes(range(201, 213)) + fill(60) + bytes(range(200, 213))
    return {
        "empty": b"",
        "one": b"\x07",
        "tiny_fixed": b"abcabcabcabcabc" * 4,                         # few tokens: a fixed block
        "short_noise": noise(600),                                     # literals only, below 8 KiB
        "zeros_2000": bytes(2000),                                     # distance-1 runs, sparse updates, nice exits
        "incompressible_exit": head + noise(2000) + head,              # 512-literal streak, then a probe match
        "gate_8192": b"\x01\x02\x03" + low(9000) + b"\x01\x02\x03" + low(50),   # a 3-byte match 9 003 back
        "tail_match": noise(300) + noise(40) * 2,                     # a match that ends at the data's end
        "sawtooth": bytes(range(256)) * 12,                            # 258-byte matches: nice-length exits
        "text": b"".join(b"row %d: fox %d jumps\n" % (i, i * i % 97) for i in range(300)),
        "lazy": lazy + fill(60),                                       # a short match, a longer one a byte later
        "window_edge": (lambda w: w + low(33000) + w)(noise(300)),    # a repeat beyond the 32 KiB window
    }


def constructed():
    """{name: bytes}: small_cases plus streams that reach the driver's size-dependent branches."""
    rng = np.random.default_rng(8)
    noise = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    window = noise(40000)
    return dict(small_cases(), **{
        "noise_12k": noise(12000),                                     # no match at >= 8 KiB: stored
        "noise_70k": noise(70000),                                     # stored, two 65 535-byte blocks
        "zeros_9000": bytes(9000),
        "window_inside": window[:32000] + window[:4000],              # a repeat just inside the window
        "paletted": rng.integers(0, 4, 30000, dtype=np.uint8).tobytes(),
        "stored_rule_65535": stored_rule_stream(),
    })


def inflate(z: bytes) -> bytes:
    return zlib.decompress(z)
