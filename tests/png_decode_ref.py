"""An independent pure-Python restatement of pixo::decode::decode_png (src/decode/png.rs:101-626) with its inflate
(src/decode/inflate.rs:46-513) and LSB bit reader (src/decode/bit_reader.rs:10-135), table quirks included, written
from pixo's source without reference to oracle/png_decode.c.  Slow; for small constructed files only.

decode(data) -> (kind, message, width, height, color_type, pixels: bytes)   kind as oracle.png_decode
"""
from __future__ import annotations

import struct
import zlib

OK, INVALID, UNSUPPORTED, DIMENSIONS, TOO_LARGE = 0, 1, 2, 3, 4


class Refused(Exception):
    def __init__(self, kind, msg):
        super().__init__(msg)
        self.kind, self.msg = kind, msg


def invalid(msg):
    return Refused(INVALID, "Decode error: " + msg)


class Reader:
    """bit_reader.rs: a position in bits over the data; pixo's byte-at-a-time buffer holds exactly the bits between
    this position and the next whole byte it loaded, so only the count of bits left matters."""

    def __init__(self, data: bytes):
        self.data, self.bit = data, 0

    def left(self):
        return 8 * len(self.data) - self.bit

    def peek(self, n):
        v = 0
        for k in range(n):
            b = self.bit + k
            v |= ((self.data[b >> 3] >> (b & 7)) & 1) << k
        return v

    def read(self, n):
        if self.left() < n:
            raise invalid("unexpected end of stream")
        v = self.peek(n)
        self.bit += n
        return v

    def align(self):
        self.bit = (self.bit + 7) & ~7


class Table:
    """HuffmanTable::from_lengths: the 9-bit lookup with later symbols overwriting earlier ones, and the canonical
    codes decode_slow compares, in symbol order."""

    def __init__(self, lengths):
        self.lengths = list(lengths)
        self.max_len = max(self.lengths, default=0)
        self.lookup = [None] * 512
        self.codes = {}
        if not self.max_len:
            return
        count = [0] * 16
        for L in self.lengths:
            if L:
                count[L] += 1
        nxt, code = [0] * 16, 0
        for bits in range(1, 16):
            code = (code + count[bits - 1]) << 1
            nxt[bits] = code
        for s, L in enumerate(self.lengths):
            if L:
                self.codes[s] = nxt[L]
                nxt[L] += 1
        for s, L in enumerate(self.lengths):
            if 0 < L <= 9:
                c = self.codes[s] & 0xFFFF
                rev = int(format(c & ((1 << L) - 1), f"0{L}b")[::-1], 2)
                for i in range(1 << (9 - L)):
                    self.lookup[rev | (i << L)] = (s, L)

    def decode(self, r: Reader):
        if not self.max_len:
            raise invalid("empty Huffman table")
        avail = min(9, r.left())
        if avail > 0:
            e = self.lookup[r.peek(avail)]
            if e and e[1] <= avail:
                r.bit += e[1]
                return e[0]
        code = 0
        for L in range(1, self.max_len + 1):
            code = (code << 1) | r.read(1)
            for s, sl in enumerate(self.lengths):
                if sl == L and self.codes[s] == code:
                    return s
        raise invalid("invalid Huffman code")


LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]
ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = Table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
FIXED_DIST = Table([5] * 32)


def _block(r, out, lit, dist):
    while True:
        s = lit.decode(r)
        if s < 256:
            out.append(s)
        elif s == 256:
            return
        elif s <= 285:
            length = LEN_BASE[s - 257] + r.read(LEN_EXTRA[s - 257])
            d = dist.decode(r)
            if d >= 30:
                raise invalid("invalid distance code")
            distance = DIST_BASE[d] + r.read(DIST_EXTRA[d])
            if distance > len(out):
                raise invalid("distance too far back")
            start = len(out) - distance
            for i in range(length):
                out.append(out[start + i % distance])
        else:
            raise invalid(f"invalid literal/length code: {s}")


def inflate_raw(data: bytes) -> bytearray:
    r, out = Reader(data), bytearray()
    while True:
        final, btype = r.read(1), r.read(2)
        if btype == 0:
            r.align()
            n, nn = r.read(16), r.read(16)
            if n != (~nn & 0xFFFF):
                raise invalid("stored block LEN/NLEN mismatch")
            if r.left() < 8 * n:
                raise invalid("unexpected end of stream")
            out += data[r.bit >> 3:(r.bit >> 3) + n]
            r.bit += 8 * n
        elif btype == 1:
            _block(r, out, FIXED_LIT, FIXED_DIST)
        elif btype == 2:
            hlit, hdist, hclen = r.read(5) + 257, r.read(5) + 1, r.read(4) + 4
            cl = [0] * 19
            for k in range(hclen):
                cl[ORDER[k]] = r.read(3)
            clt = Table(cl)
            lens = []
            while len(lens) < hlit + hdist:
                s = clt.decode(r)
                if s < 16:
                    lens.append(s)
                    continue
                if s == 16:
                    if not lens:
                        raise invalid("repeat code at start")
                    rep, val = r.read(2) + 3, lens[-1]
                else:
                    rep, val = (r.read(3) + 3 if s == 17 else r.read(7) + 11), 0
                for _ in range(rep):
                    if len(lens) >= hlit + hdist:
                        raise invalid("too many code lengths")
                    lens.append(val)
            _block(r, out, Table(lens[:hlit]), Table(lens[hlit:]))
        else:
            raise invalid("reserved block type")
        if final:
            return out


def inflate_zlib(data: bytes, expected: int) -> bytes:
    if len(data) < 6:
        raise invalid("zlib stream too short")
    if data[0] & 15 != 8:
        raise invalid("invalid zlib compression method")
    if (data[0] << 8 | data[1]) % 31:
        raise invalid("invalid zlib header checksum")
    if data[1] & 0x20:
        raise Refused(UNSUPPORTED, "Unsupported: preset dictionary not supported")
    out = bytes(inflate_raw(data[2:-4]))
    stored, got = struct.unpack(">I", data[-4:])[0], zlib.adler32(out)
    if stored != got:
        raise invalid(f"Adler32 mismatch: expected {stored:08X}, got {got:08X}")
    if len(out) != expected:
        raise invalid(f"decompressed size mismatch: expected {expected}, got {len(out)}")
    return out


NAMES = {0: "Grayscale", 2: "Rgb", 3: "Indexed", 4: "GrayscaleAlpha", 6: "Rgba"}
LEGAL = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
SAMPLES = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def _decode(data: bytes):
    if len(data) < 8 or data[:8] != b"\x89PNG\r\n\x1a\n":
        raise invalid("not a PNG file")
    pos, hdr, idat, plte, trns, iend = 8, None, bytearray(), None, None, False
    while pos + 12 <= len(data):
        n = int.from_bytes(data[pos:pos + 4], "big")
        kind = data[pos + 4:pos + 8]
        if pos + 12 + n > len(data):
            raise invalid("truncated PNG chunk")
        body = data[pos + 8:pos + 8 + n]
        if int.from_bytes(data[pos + 8 + n:pos + 12 + n], "big") != zlib.crc32(kind + body):
            raise invalid(f"CRC mismatch in {kind.decode('utf-8', 'replace')} chunk")
        if kind == b"IHDR":
            if n != 13:
                raise invalid("invalid IHDR length")
            if body[9] not in NAMES:
                raise invalid(f"invalid PNG color type: {body[9]}")
            hdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"PLTE":
            if n % 3:
                raise invalid("invalid PLTE length")
            plte = [body[i:i + 3] for i in range(0, n, 3)]
        elif kind == b"tRNS":
            trns = body
        elif kind == b"IDAT":
            idat += body
        elif kind == b"IEND":
            iend = True
            break
        pos += 12 + n
    if not iend:
        raise invalid("missing IEND chunk")
    if hdr is None:
        raise invalid("missing IHDR chunk")
    w, h, depth, ct, comp, filt, lace = hdr
    if w == 0 or h == 0:
        raise Refused(DIMENSIONS, f"Invalid image dimensions: {w}x{h}")
    if w > 1 << 24 or h > 1 << 24:
        raise Refused(TOO_LARGE, f"Image {w}x{h} exceeds maximum dimension {1 << 24}")
    if comp:
        raise invalid("unsupported compression method")
    if filt:
        raise invalid("unsupported filter method")
    if lace:
        raise Refused(UNSUPPORTED, "Unsupported: Adam7 interlaced images not supported")
    if depth not in LEGAL[ct]:
        raise invalid(f"invalid bit depth {depth} for color type {NAMES[ct]}")
    if not idat:
        raise invalid("no IDAT data")
    bits = depth * SAMPLES[ct]
    sb = (w * bits + 7) // 8
    bpp = 1 if ct in (0, 3) and depth < 8 or ct == 3 else bits // 8
    raw = bytearray(inflate_zlib(bytes(idat), h * (1 + sb)))
    prev = bytearray(sb)
    rows = []
    for y in range(h):
        f = raw[y * (sb + 1)]
        cur = raw[y * (sb + 1) + 1:(y + 1) * (sb + 1)]
        if f > 4:
            raise invalid(f"invalid filter type: {f}")
        for i in range(sb):
            a = cur[i - bpp] if i >= bpp else 0
            c = prev[i - bpp] if i >= bpp else 0
            cur[i] = (cur[i] + (0, a, prev[i], (a + prev[i]) >> 1, _paeth(a, prev[i], c))[f]) & 255
        rows.append(cur)
        prev = cur
    alpha = trns is not None and any(v != 255 for v in trns)
    out = bytearray()
    if ct == 3 and plte is None:
        raise invalid("missing PLTE chunk")
    for row in rows:
        if depth == 16:
            out += row[::2]
            continue
        if depth == 8 and ct != 3:
            out += row
            continue
        samples = [(row[(x * depth) >> 3] >> (8 - depth - (x * depth) % 8)) & ((1 << depth) - 1) for x in range(w)]
        if ct == 0:
            out += bytes(s * 255 // ((1 << depth) - 1) for s in samples)
            continue
        for s in samples:
            rgb = bytes(plte[s]) if s < len(plte) else b"\0\0\0"
            a = (trns[s] if trns is not None and s < len(trns) else 255) if s < len(plte) else 255
            out += rgb + (bytes([a]) if alpha else b"")
    oct = {0: 0, 4: 1, 2: 2, 6: 3}.get(ct, 3 if alpha else 2)
    return w, h, oct, bytes(out)


def decode(data: bytes):
    try:
        w, h, ct, px = _decode(bytes(data))
        return OK, "", w, h, ct, px
    except Refused as e:
        return e.kind, e.msg, 0, 0, 0, b""
