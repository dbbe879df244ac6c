"""Test-side restatement of pixo's progressive scan writer, as its max preset runs it
(src/jpeg/mod.rs encode_progressive :872-927, encode_dc_scan / encode_ac_first_scan :1248-1370;
src/jpeg/progressive.rs simple_progressive_script :98-110, encode_ac_first :141-210, flush_eob_run
:313-345, get_code_from_table :363-380 with its (0, 4) fallback; BitWriterMsb src/bits.rs:195-278).

It depends only on coefficient arrays: the Huffman tables are read from the file's DHT, so a max-preset
file is reproduced scan by scan from the coefficients that made it.  Blocks go in array order (the order
compute_all_coefficients returns them) in every scan, as pixo writes them.

scans(jpeg_bytes) -> [(component ids, ss, se, ah, al, entropy-coded bytes)] per SOS
dht(jpeg_bytes) -> {(class, id): (bits[16], vals)}
encode_scans(y, cb, cr, tables) -> [entropy-coded bytes] for the 7 scans of simple_progressive_script
"""
from __future__ import annotations

import numpy as np

ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
          7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
          39, 46, 53, 60, 61, 54, 47, 55, 62, 63]
# (component, ss, se) of simple_progressive_script; ah = al = 0 throughout
SCRIPT = [(0, 0, 0), (1, 0, 0), (2, 0, 0), (0, 1, 10), (0, 11, 63), (1, 1, 63), (2, 1, 63)]


def _segments(data: bytes):
    """(marker, payload, end offset) of every marker segment up to EOI."""
    assert data[:2] == b"\xff\xd8"
    i = 2
    while i < len(data):
        assert data[i] == 0xFF, f"marker expected at {i}"
        m = data[i + 1]
        if m == 0xD9:
            return
        n = (data[i + 2] << 8) | data[i + 3]
        yield m, data[i + 4:i + 2 + n], i + 2 + n
        i += 2 + n
        if m == 0xDA:   # skip the entropy-coded data to the next marker
            while not (data[i] == 0xFF and data[i + 1] not in (0x00,) and not 0xD0 <= data[i + 1] <= 0xD7):
                i += 1


def dht(data: bytes) -> dict:
    out = {}
    for m, p, _ in _segments(data):
        if m != 0xC4:
            continue
        j = 0
        while j < len(p):
            tc_th = p[j]
            bits = list(p[j + 1:j + 17])
            n = sum(bits)
            out[(tc_th >> 4, tc_th & 15)] = (bits, list(p[j + 17:j + 17 + n]))
            j += 17 + n
    return out


def scans(data: bytes):
    res = []
    for m, p, end in _segments(data):
        if m != 0xDA:
            continue
        ns = p[0]
        comps = [p[1 + 2 * k] - 1 for k in range(ns)]
        ss, se, ahal = p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns]
        k = end
        while not (data[k] == 0xFF and data[k + 1] != 0x00 and not 0xD0 <= data[k + 1] <= 0xD7):
            k += 1
        res.append((comps, ss, se, ahal >> 4, ahal & 15, data[end:k]))
    return res


def code_from_table(bits, vals, symbol):
    """get_code_from_table: canonical code of `symbol`, or pixo's fallback (0, 4) when it is absent."""
    code, idx = 0, 0
    for length, count in enumerate(bits):
        for _ in range(count):
            if idx < len(vals) and vals[idx] == symbol:
                return code, length + 1
            idx += 1
            code += 1
        code <<= 1
    return 0, 4


class BitWriterMsb:
    def __init__(self):
        self.buf = bytearray()
        self.cur = 0
        self.pos = 8

    def write(self, value: int, n: int):
        while n > 0:
            t = min(n, self.pos)
            bits = (value >> (n - t)) & ((1 << t) - 1)
            self.pos -= t
            self.cur |= bits << self.pos
            n -= t
            if self.pos == 0:
                self._flush_byte()

    def _flush_byte(self):
        self.buf.append(self.cur)
        if self.cur == 0xFF:
            self.buf.append(0)
        self.cur, self.pos = 0, 8

    def finish(self) -> bytes:
        if self.pos < 8:
            self.cur |= (1 << self.pos) - 1
            self._flush_byte()
        return bytes(self.buf)


def _category(v: int) -> int:
    return abs(int(v)).bit_length()


def _value_bits(v: int):
    cat = _category(v)
    return ((v - 1) if v < 0 else v) & ((1 << cat) - 1), cat


def _i16(v: int) -> int:
    return (v + 0x8000) % 0x10000 - 0x8000


def encode_scans(y, cb, cr, tables) -> list[bytes]:
    comps = [np.asarray(y, np.int16).reshape(-1, 64), np.asarray(cb, np.int16).reshape(-1, 64),
             np.asarray(cr, np.int16).reshape(-1, 64)]
    out = []
    for comp, ss, se in SCRIPT:
        w = BitWriterMsb()
        blocks = comps[comp]
        lum = comp == 0
        dc_tab = tables.get((0, 0 if lum else 1), ([0] * 16, []))
        ac_tab = tables.get((1, 0 if lum else 1), ([0] * 16, []))
        if len(blocks) and ss == 0:
            prev = 0
            for b in blocks:
                diff = _i16(int(b[0]) - prev)
                cat = _category(diff)
                w.write(*code_from_table(dc_tab[0], dc_tab[1], cat))
                if cat:
                    w.write(*_value_bits(diff))
                prev = int(b[0])
        elif len(blocks):
            eob_run = 0

            def flush_eob():
                nonlocal eob_run
                if eob_run == 0:
                    return
                nbits = max(eob_run.bit_length() - 1, 0)
                w.write(*code_from_table(ac_tab[0], ac_tab[1], nbits << 4))
                if nbits:
                    w.write(eob_run - (1 << nbits), nbits)
                eob_run = 0

            for b in blocks:
                zz = [int(b[ZIGZAG[k]]) for k in range(64)]
                k = se
                while k >= ss and zz[k] == 0:
                    if k == ss:
                        break
                    k -= 1
                last = k
                if last == ss and zz[ss] == 0:
                    eob_run += 1
                    if eob_run == 0x7FFF:
                        flush_eob()
                    continue
                if eob_run > 0:
                    flush_eob()
                run = 0
                for k in range(ss, last + 1):
                    c = zz[k]
                    if c == 0:
                        run += 1
                        continue
                    while run >= 16:
                        w.write(*code_from_table(ac_tab[0], ac_tab[1], 0xF0))
                        run -= 16
                    w.write(*code_from_table(ac_tab[0], ac_tab[1], (run << 4) | _category(c)))
                    w.write(*_value_bits(c))
                    run = 0
                if last < se:
                    eob_run = 1
            flush_eob()
        out.append(w.finish())
    return out
