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


# ---- is_high_entropy_data on both sides of its threshold (deflate.rs:1108-1145) ---------------------------------

def he_hash(v: int) -> int:
    """is_high_entropy_data's 12-bit hash of a little-endian 4-gram."""
    return ((v * 0x1E35A7BD) & 0xFFFFFFFF) >> 20 & 4095


def entropy_stream(n: int, forced: int = 0, seed: int = 0, tail: int = 0):
    """(stream, collisions, tail): n bytes over a 32-symbol alphabet, each byte picked so that its 4-gram lands in an
    unused slot of the 4 096 while one of the 32 allows it; the last `forced` bytes pick a used slot instead.  The
    collisions are those of the whole stream.  `tail` more bytes continue the free-slot rule past the stream over all
    256 byte values, so a sample that reads a few bytes past n sees a lower collision rate than the stream has.  The small alphabet makes the two sides
    of the bail differ: parsed, the literals code at about 5 bits and the block is dynamic; bailed, it is stored."""
    rng = np.random.default_rng(seed)
    d = [int(x) for x in rng.integers(0, 32, 3)]
    seen = bytearray(4096)
    coll = 0
    while len(d) < n + tail:
        base = d[-3] | d[-2] << 8 | d[-1] << 16
        cands = rng.permutation(32 if len(d) < n else 256)
        want = 1 if n - forced <= len(d) < n else 0
        c = int(cands[0])
        for x in cands:
            if seen[he_hash(base | int(x) << 24)] == want:
                c = int(x)
                break
        k = he_hash(base | c << 24)
        if len(d) < n:
            coll += seen[k]
        seen[k] = 1
        d.append(c)
    return bytes(d[:n]), coll, bytes(d[n:])


# The longest stream the construction makes fire: seeds 0-399 without forced collisions, the best prefix of each
LONGEST_BAIL = (4186, 283)


def entropy_cases():
    """{name: (stream, collisions, fires, tail)}: streams at the bail's edges.  At 4 103 bytes 205 collisions are
    exactly 5 % in f32 (no bail), 204 are just under; at 4 096 bytes 204 fire and 205 do not.  206, 207 and 208
    repeats at 4 123, 4 143 and 4 163 bytes are exactly 5 % too, each with another divisor whose reciprocal an
    approximate division would round differently.  A stream of 4 095
    bytes is below the sample pixo takes; LONGEST_BAIL is the longest the construction makes fire.  The tail of a
    stream that fires repeats its first bytes (every 4-gram a collision), the tail of one that does not continues
    with fresh slots, so a sample that reads 8 bytes past the stream flips the decision either way."""
    out = {}
    for name, n, forced, seed, want_coll, fires in (
            ("bail_4103_204", 4103, 17, 0, 204, True), ("bail_4103_205", 4103, 19, 0, 205, False),
            ("bail_4096_204", 4096, 20, 0, 204, True), ("bail_4096_205", 4096, 21, 0, 205, False),
            ("bail_4123_206", 4123, 3, 0, 206, False), ("bail_4143_207", 4143, 10, 8, 207, False),
            ("bail_4163_208", 4163, 6, 15, 208, False), ("bail_4095", 4095, 0, 0, None, False),
            ("bail_longest", LONGEST_BAIL[0], 0, LONGEST_BAIL[1], None, True)):
        s, coll, fresh = entropy_stream(n, forced, seed, tail=512)
        assert want_coll is None or coll == want_coll, (name, coll)
        out[name] = (s, coll, fires, s[:512] if fires else fresh)
    return out


# ---- tails that change the output when a kernel reads past a stream -----------------------------------------------

def read_past_tail(s: bytes, size: int, tail: bytes = b"") -> bytes:
    """`size` bytes to lay after stream s: `tail` if given, else the stream's last 300 bytes (a match, run or 4-byte
    read that runs past the end then finds a longer or a different match).  For streams under 4 096 bytes the byte
    values s lacks follow within the first 4 096 bytes, so a census that counts past the end raises pixo's minimum
    match length.  The rest repeats the stream's end."""
    end = s[-300:] or b"\x00"
    if not tail:
        tail = end
        if len(s) < 4096:
            missing = bytes(sorted(set(range(256)) - set(s)))
            room = 4096 - len(s) - len(missing)
            tail = (end[:max(room, 0)] + missing) if room < len(end) else end + missing
    out = (tail + end * (size // len(end) + 1))[:size]
    assert len(out) == size
    return out


def families(count: int, seed: int = 0):
    """`count` streams of 1-4 KiB in families of about 40 that share content: each family has a 1 KiB prefix, and its
    streams are that prefix followed by copies of it with a few bytes changed, at random offsets.  A warp's hash
    table left from an earlier stream of the same family points at content the next stream also has."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        prefix = rng.integers(0, 48, 1024, dtype=np.uint8)
        for _ in range(min(40, count - len(out))):
            n = int(rng.integers(1024, 4097))
            parts = [prefix]
            while sum(p.size for p in parts) < n:
                v = np.roll(prefix, int(rng.integers(0, 1024)))[:int(rng.integers(64, 1025))].copy()
                v[rng.integers(0, v.size, int(rng.integers(1, 8)))] = rng.integers(0, 256, dtype=np.uint8)
                parts.append(v)
            out.append(np.concatenate(parts)[:n].tobytes())
    order = rng.permutation(len(out))
    return [out[i] for i in order]


def stored_block_noise():
    """{n: noise}: streams at and beside multiples of 65 535 bytes, which pixo stores in ceil(n / 65 535) blocks."""
    rng = np.random.default_rng(12)
    return {n: rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in (65534, 65535, 65536, 131070, 131071, 196605)}


def filtered_frame(w: int, h: int, bpp: int, seed: int, noise_band: bool = False) -> bytes:
    """A filtered frame's stream as test_full_size_frames builds it (filter byte 1 and smooth rows of w * bpp bytes),
    with an optional band of noise over an eighth of it."""
    rows = (np.arange(w * bpp, dtype=np.uint32)[None, :] // 9 + np.arange(h, dtype=np.uint32)[:, None] // 5 + seed) & 0xFF
    out = np.concatenate([np.ones((h, 1), np.uint32), rows], axis=1).astype(np.uint8).reshape(-1)
    if noise_band:
        a = out.size // 3
        out[a:a + out.size // 8] = np.random.default_rng(seed).integers(0, 256, out.size // 8, dtype=np.uint8)
    return out.tobytes()
