"""An independent baseline (sequential DCT, Huffman) scan decoder, written from ITU-T T.81:
Annex B (marker syntax), C (Huffman table specification), F.2.2 (decoding of the DC difference and
the AC coefficients).  Test infrastructure only: it shares no code with the product or the oracle,
so it can check both.

`decode(jpg)` returns the quantised coefficients in natural order, in compute_all_coefficients'
layout (Y: the MCU's blocks in raster order - TL, TR, BL, BR for 4:2:0 -, then one Cb and one Cr
block per MCU), and is strict about everything a conforming baseline encoder must get right:

  * every DHT: at most 256 values, code lengths 1..16, and a code space that is NOT full (C.2: no
    code may consist of 1-bits only, so the Kraft sum stays below 1);
  * the scan: FF 00 is a stuffed 0xFF; any other FF xx must be the expected RSTn (n = 0..7, cycling)
    at the end of a restart interval; no RSTn before EOI; every interval and the scan end on a byte
    boundary padded with 1-bits (F.1.2.3), with no byte left over;
  * DC categories <= 11, AC sizes <= 10, no AC run past coefficient 63.

DC predictors wrap to 16 bits (a DC value is the int16 sum of the differences), reset to 0 at every
restart interval (F.2.1.3.1).
"""
from __future__ import annotations

import dataclasses

import numpy as np

# zig-zag position k -> natural index (Figure A.6)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5,
                   12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                   58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


class ScanError(ValueError):
    pass


@dataclasses.dataclass
class Decoded:
    width: int
    height: int
    comps: list            # [(id, h, v, tq)]
    y: np.ndarray          # [ny, 64] int16, natural order
    cb: np.ndarray         # [nc, 64] (empty for one component)
    cr: np.ndarray
    restart_interval: int
    tables: dict           # (class, id) -> (bits[16], vals)
    block_start: np.ndarray | None   # bit offset of every block (scan order) in `unstuffed`
    interval_end: list     # per restart interval: bit offset in `unstuffed` where its code ends (before padding)
    unstuffed: bytes       # the intervals' entropy-coded bytes, stuffing and markers removed, concatenated


def _huffman_lut(bits, vals):
    """(C.2) canonical codes -> a 16-bit look-up: entry = (length << 8) | symbol, 0 = no code."""
    if len(bits) != 16 or sum(bits) != len(vals) or len(vals) > 256:
        raise ScanError("DHT: counts and values disagree")
    lut = np.zeros(1 << 16, np.int32)
    code, k = 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            if code >= (1 << ln):
                raise ScanError("DHT: more codes than the code space holds")
            if code == (1 << ln) - 1:
                raise ScanError("DHT: an all-ones code (the code space is full)")
            lo = code << (16 - ln)
            lut[lo:lo + (1 << (16 - ln))] = (ln << 8) | vals[k]
            code += 1
            k += 1
        code <<= 1
    return lut.tolist()


def _segments(jpg: bytes):
    """Marker segments up to SOS: yields (marker, payload); then ('scan', index of the first scan byte)."""
    if jpg[:2] != b"\xff\xd8":
        raise ScanError("no SOI")
    i = 2
    while True:
        if jpg[i] != 0xFF:
            raise ScanError(f"expected a marker at {i}")
        m = jpg[i + 1]
        ln = int.from_bytes(jpg[i + 2:i + 4], "big")
        yield m, jpg[i + 4:i + 2 + ln]
        i += 2 + ln
        if m == 0xDA:
            yield "scan", i
            return


def _intervals(jpg: bytes, start: int):
    """Entropy-coded data -> [unstuffed bytes of each restart interval], checking RSTn order; ends at EOI."""
    out, cur = [], bytearray()
    i, n = start, len(jpg)
    expect = 0
    while True:
        if i >= n:
            raise ScanError("scan runs past the end of the file")
        b = jpg[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        m = jpg[i + 1]
        if m == 0x00:
            cur.append(0xFF)
        elif m == 0xD9:
            out.append(bytes(cur))
            if i + 2 != n:
                raise ScanError("bytes after EOI")
            return out
        elif 0xD0 <= m <= 0xD7:
            if m != 0xD0 + expect:
                raise ScanError(f"RST{m - 0xD0} where RST{expect} was expected")
            expect = (expect + 1) & 7
            out.append(bytes(cur))
            cur = bytearray()
        else:
            raise ScanError(f"marker FF {m:02X} inside the scan")
        i += 2


def decode(jpg: bytes, block_starts: bool = False) -> Decoded:
    tables, qt, comps, ri = {}, {}, None, 0
    width = height = 0
    scan_start, scan_comps = None, None
    for m, p in _segments(jpg):
        if m == "scan":
            scan_start = p
            break
        if m == 0xDB:
            k = 0
            while k < len(p):
                if p[k] >> 4:
                    raise ScanError("16-bit quantisation table in a baseline file")
                qt[p[k] & 15] = p[k + 1:k + 65]
                k += 65
        elif m == 0xC0:
            if p[0] != 8:
                raise ScanError("sample precision is not 8")
            height, width, nf = int.from_bytes(p[1:3], "big"), int.from_bytes(p[3:5], "big"), p[5]
            comps = [(p[6 + 3 * c], p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15, p[8 + 3 * c]) for c in range(nf)]
        elif m == 0xC4:
            k = 0
            while k < len(p):
                tc, th = p[k] >> 4, p[k] & 15
                bits = list(p[k + 1:k + 17])
                vals = list(p[k + 17:k + 17 + sum(bits)])
                if tc > 1 or th > 1:
                    raise ScanError("baseline allows two tables per class")
                tables[(tc, th)] = (bits, vals)
                k += 17 + sum(bits)
        elif m == 0xDD:
            ri = int.from_bytes(p[0:2], "big")
        elif m == 0xDA:
            ns = p[0]
            scan_comps = [(p[1 + 2 * c], p[2 + 2 * c] >> 4, p[2 + 2 * c] & 15) for c in range(ns)]
            if tuple(p[1 + 2 * ns:4 + 2 * ns]) != (0, 63, 0):
                raise ScanError("not a sequential baseline scan (Ss, Se, Ah/Al)")
        elif m in (0xC1, 0xC2, 0xC3) or 0xC5 <= m <= 0xCF:
            raise ScanError(f"not a baseline frame (SOF{m - 0xC0})")
    if comps is None or scan_comps is None:
        raise ScanError("no SOF0 / SOS")
    if len(scan_comps) != len(comps):
        raise ScanError("the scan does not hold every component")
    luts = {k: _huffman_lut(*v) for k, v in tables.items()}

    hmax = max(c[1] for c in comps)
    vmax = max(c[2] for c in comps)
    if len(comps) == 1:        # non-interleaved: one block per MCU (A.2.2)
        mcus = ((width + 7) // 8) * ((height + 7) // 8)
        layout = [(0, 1)]
    else:
        mcus = ((width + 8 * hmax - 1) // (8 * hmax)) * ((height + 8 * vmax - 1) // (8 * vmax))
        layout = [(c, comps[c][1] * comps[c][2]) for c in range(len(comps))]
    # block s of an MCU -> (component, Huffman tables)
    plan = []
    for c, nb in layout:
        cid, td, ta = scan_comps[c]
        if cid != comps[c][0]:
            raise ScanError("scan components out of frame order")
        if (0, td) not in luts or (1, ta) not in luts:
            raise ScanError("the scan uses an undefined Huffman table")
        plan += [(c, luts[(0, td)], luts[(1, ta)])] * nb
    blocks = [[] for _ in comps]
    starts = []

    intervals = _intervals(jpg, scan_start)
    per = ri if ri else mcus
    n_int = (mcus + per - 1) // per
    if len(intervals) != n_int:
        raise ScanError(f"{len(intervals)} restart intervals, expected {n_int} (an RSTn before EOI?)")
    base = 0
    ends = []
    for it, data in enumerate(intervals):
        d = data + b"\x00\x00\x00\x00"
        nbits = 8 * len(data)
        pos = 0
        pred = [0] * len(comps)

        def bits16(p):
            return (int.from_bytes(d[p >> 3:(p >> 3) + 3], "big") >> (8 - (p & 7))) & 0xFFFF

        def symbol(lut):
            nonlocal pos
            e = lut[bits16(pos)]
            if not e:
                raise ScanError(f"no Huffman code at bit {pos} of interval {it}")
            pos += e >> 8
            return e & 0xFF

        def receive_extend(s):
            nonlocal pos
            if s == 0:
                return 0
            v = bits16(pos) >> (16 - s)
            pos += s
            return v - (1 << s) + 1 if v < (1 << (s - 1)) else v

        for _ in range(min(per, mcus - it * per)):
            for c, dc_lut, ac_lut in plan:
                if block_starts:
                    starts.append(base + pos)
                blk = np.zeros(64, np.int32)
                t = symbol(dc_lut)
                if t > 11:
                    raise ScanError(f"DC category {t}")
                pred[c] = ((pred[c] + receive_extend(t) + 32768) & 0xFFFF) - 32768
                blk[0] = pred[c]
                k = 1
                while k < 64:
                    rs = symbol(ac_lut)
                    r, s = rs >> 4, rs & 15
                    if s == 0:
                        if r != 15:
                            break       # EOB
                        k += 16          # ZRL
                        if k > 63:
                            raise ScanError("ZRL past coefficient 63")
                        continue
                    if s > 10:
                        raise ScanError(f"AC size {s}")
                    k += r
                    if k > 63:
                        raise ScanError("AC run past coefficient 63")
                    blk[ZIGZAG[k]] = receive_extend(s)
                    k += 1
                blocks[c].append(blk)
                if pos > nbits:
                    raise ScanError(f"interval {it} ends inside a code")
        pad = -pos % 8
        if pos + pad != nbits:
            raise ScanError(f"interval {it}: {nbits - pos - pad} bits left over")
        if pad and (bits16(pos) >> (16 - pad)) != (1 << pad) - 1:
            raise ScanError(f"interval {it}: padding is not all 1-bits")
        ends.append(base + pos)
        base += nbits
    arr = [np.array(b, np.int16).reshape(-1, 64) for b in blocks]
    empty = np.zeros((0, 64), np.int16)
    return Decoded(width, height, comps, arr[0], arr[1] if len(arr) > 1 else empty,
                   arr[2] if len(arr) > 2 else empty, ri, tables,
                   np.array(starts, np.int64) if block_starts else None, ends, b"".join(intervals))


def scan_bytes(jpg: bytes) -> bytes:
    """The entropy-coded segment: after the SOS header, before EOI."""
    for m, p in _segments(jpg):
        if m == "scan":
            return jpg[p:-2]
