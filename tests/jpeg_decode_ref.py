"""An independent pure-Python restatement of pixo::decode::decode_jpeg (src/decode/jpeg.rs, bit_reader.rs, idct.rs),
for checking the C oracle (oracle/jpeg_decode.c) on small constructed files.  Slow; shares no code with the oracle
or the product.

pixo's release-build arithmetic is written out: u8 bits_in_buf wraps, u32 / i32 arithmetic wraps, shift counts are
masked, `as` casts truncate.

decode(data) -> ("ok", width, height, color_type, pixels bytes) | (kind, message)   kind: "invalid" | "unsupported"
| "panic"
"""
from __future__ import annotations

M32 = 0xFFFFFFFF


def i32(x: int) -> int:
    x &= M32
    return x - (1 << 32) if x & 0x80000000 else x


def i16(x: int) -> int:
    x &= 0xFFFF
    return x - 0x10000 if x & 0x8000 else x


class Fail(Exception):
    def __init__(self, kind, msg):
        super().__init__(msg)
        self.kind, self.msg = kind, msg


class Table:
    """HuffmanTable::build"""

    def __init__(self, bits=None, values=b""):
        self.lookup = [0] * 256
        self.values = bytes(values)
        self.maxcode = [-1] * 17
        self.valoff = [0] * 17
        if bits is None:
            return
        sizes = [i + 1 for i in range(16) for _ in range(bits[i])]
        codes, code, si = [], 0, (sizes[0] if sizes else 0)
        for s in sizes:
            while s > si:
                code = (code << 1) & M32
                si += 1
            codes.append(code & 0xFFFF)
            code += 1
        vi = 0
        for i in range(1, 17):
            if bits[i - 1]:
                self.valoff[i] = vi - codes[vi]
                vi += bits[i - 1]
                self.maxcode[i] = codes[vi - 1]
        for idx, s in enumerate(sizes):
            if s <= 8:
                base = codes[idx] << (8 - s)
                for j in range(1 << (8 - s)):
                    if base | j < 256:
                        self.lookup[base | j] = values[idx] | (s << 8)


class Bits:
    """MsbBitReader"""

    class End(Exception):
        pass

    def __init__(self, data):
        self.d, self.pos, self.buf, self.n = data, 0, 0, 0

    def byte(self):
        while True:
            if self.pos >= len(self.d):
                raise Bits.End
            b = self.d[self.pos]
            self.pos += 1
            if b != 0xFF:
                return b
            if self.pos >= len(self.d):
                raise Bits.End
            nx = self.d[self.pos]
            if nx == 0:
                self.pos += 1
                return b
            if 0xD0 <= nx <= 0xD7:
                self.pos += 1
                self.buf = self.n = 0
                continue
            self.pos -= 1
            raise Bits.End

    def peek(self, n):
        while self.n < n:
            b = self.byte()
            self.buf = ((self.buf << 8) | b) & M32
            self.n = (self.n + 8) & 0xFF
        return (self.buf >> ((self.n - n) & 31)) & (((1 << (n & 31)) - 1) & M32)

    def consume(self, n):
        self.n = (self.n - n) & 0xFF
        self.buf &= ((1 << self.n) - 1) if self.n < 32 else M32

    def read(self, n):
        v = self.peek(n)
        self.consume(n)
        return v


def huff(t: Table, r: Bits) -> int:
    try:
        e = t.lookup[r.peek(8)]
        if 0 < e >> 8 <= 8:
            r.consume(e >> 8)
            return e & 0xFF
    except Bits.End:
        pass
    code = 0
    for ln in range(1, 17):
        code = (code << 1) | r.read(1)
        if code <= t.maxcode[ln]:
            idx = code + t.valoff[ln]
            if 0 <= idx < len(t.values):
                return t.values[idx]
            raise Bits.End
    raise Bits.End


def amplitude(r: Bits, size: int) -> int:
    bits = i32(r.read(size))
    thr = i32(1 << ((size - 1) & 31))
    return i32(bits - i32(2 * thr - 1)) if bits < thr else bits


def entropy_end(d: bytes) -> int:
    if len(d) < 2:
        return len(d)
    i = 0
    while i < len(d) - 1:
        if d[i] == 0xFF and d[i + 1] not in (0, 0xFF):
            if 0xD0 <= d[i + 1] <= 0xD7:
                i += 2
                continue
            return i
        i += 1
    return len(d)


UNZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27,
            20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
            58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]


def fm(a, b):
    return i32((a * b) >> 13)


def butterfly(d):
    t0, t1, t2, t3 = (i32(d[k] << 13) for k in (0, 2, 4, 6))
    a10, a11 = i32(t0 + t2), i32(t0 - t2)
    z1 = fm(i32(t1 + t3), 4433)
    a12, a13 = i32(z1 - fm(t3, 15137)), i32(z1 + fm(t1, 6270))
    e0, e3, e1, e2 = i32(a10 + a13), i32(a10 - a13), i32(a11 + a12), i32(a11 - a12)
    z1, z2, z3, z4 = d[1], d[3], d[5], d[7]
    z5 = fm(i32(z1 + z3), 9633)
    b10, b11, b12, b13 = fm(z1, 2446), fm(z2, 16819), fm(z3, 25172), fm(z4, 12299)
    y1, y2 = fm(i32(z1 + z4), -7373), fm(i32(z2 + z3), -20995)
    y3, y4 = i32(fm(i32(z3 + z4), -16069) + z5), i32(fm(i32(d[1] + d[3]), -3196) + z5)
    b10, b11 = i32(b10 + y1 + y3), i32(b11 + y2 + y4)
    b12, b13 = i32(b12 + y2 + y3), i32(b13 + y1 + y4)
    return [i32(e0 + b13), i32(e1 + b12), i32(e2 + b11), i32(e3 + b10),
            i32(e3 - b10), i32(e2 - b11), i32(e1 - b12), i32(e0 - b13)]


def idct(coefs, q):
    nat = [0] * 64
    for i in range(64):
        nat[UNZIGZAG[i]] = coefs[i] * q[i]
    ws = [0] * 64
    for c in range(8):
        o = butterfly([nat[c + 8 * k] for k in range(8)])
        for k in range(8):
            ws[c + 8 * k] = i32(o[k] + 1024) >> 11
    out = [0] * 64
    for r in range(8):
        o = butterfly(ws[8 * r:8 * r + 8])
        for k in range(8):
            out[8 * r + k] = min(max((i32(o[k] + (1 << 17)) >> 18) + 128, 0), 255)
    return out


def decode(data: bytes):
    try:
        return _decode(bytes(data))
    except Fail as f:
        return (f.kind, f.msg)


def _decode(d: bytes):
    if len(d) < 2 or d[0] != 0xFF or d[1] != 0xD8:
        raise Fail("invalid", "not a JPEG file")
    pos = 2
    W = H = 0
    comps = []   # [h, v, q, dc, ac]
    quant = [[0] * 64 for _ in range(4)]
    dct, act = [Table() for _ in range(4)], [Table() for _ in range(4)]
    restart, mh, mv = 0, 1, 1
    while True:
        while pos < len(d) and d[pos] != 0xFF:
            pos += 1
        while pos < len(d) and d[pos] == 0xFF:
            pos += 1
        if pos >= len(d):
            raise Fail("invalid", "unexpected end of file")
        m = d[pos]
        pos += 1
        s = b""
        if not (m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7):
            if pos + 2 > len(d):
                raise Fail("invalid", "truncated marker")
            ln = d[pos] << 8 | d[pos + 1]
            pos += 2
            if ln < 2 or pos + ln - 2 > len(d):
                raise Fail("invalid", "invalid marker length")
            s = d[pos:pos + ln - 2]
            pos += ln - 2
        if m == 0xC0:
            if len(s) < 8:
                raise Fail("invalid", "invalid SOF0 length")
            if s[0] != 8:
                raise Fail("unsupported", f"{s[0]}-bit precision not supported")
            H, W = s[1] << 8 | s[2], s[3] << 8 | s[4]
            nc = s[5]
            if nc not in (1, 3):
                raise Fail("unsupported", f"{nc} components not supported")
            if len(s) < 6 + nc * 3:
                raise Fail("invalid", "truncated SOF0 components")
            comps = []
            for i in range(nc):
                cid, samp, qid = s[6 + 3 * i:9 + 3 * i]
                h, v = samp >> 4, samp & 15
                if h == 0 or v == 0:
                    raise Fail("invalid", f"invalid sampling factors {h}x{v} for component {cid}")
                if qid > 3:
                    raise Fail("invalid", f"invalid quantization table ID {qid} for component {cid}")
                mh, mv = max(mh, h), max(mv, v)
                comps.append([h, v, qid, 0, 0])
        elif m == 0xC2:
            raise Fail("unsupported", "progressive JPEG not supported")
        elif m == 0xC4:
            o = 0
            while o < len(s):
                cls, tid = s[o] >> 4, s[o] & 15
                if tid > 3:
                    raise Fail("invalid", "invalid Huffman table ID")
                o += 1
                if o + 16 > len(s):
                    raise Fail("invalid", "truncated DHT")
                bits = list(s[o:o + 16])
                o += 16
                nv = sum(bits)
                if o + nv > len(s):
                    raise Fail("invalid", "truncated DHT values")
                (dct if cls == 0 else act)[tid] = Table(bits, s[o:o + nv])
                o += nv
        elif m == 0xDB:
            o = 0
            while o < len(s):
                prec, tid = s[o] >> 4, s[o] & 15
                if tid > 3:
                    raise Fail("invalid", "invalid quantization table ID")
                o += 1
                if prec == 0:
                    if o + 64 > len(s):
                        raise Fail("invalid", "truncated DQT")
                    quant[tid] = list(s[o:o + 64])
                    o += 64
                else:
                    if o + 128 > len(s):
                        raise Fail("invalid", "truncated DQT")
                    quant[tid] = [s[o + 2 * i] << 8 | s[o + 2 * i + 1] for i in range(64)]
                    o += 128
        elif m == 0xDD:
            if len(s) != 2:
                raise Fail("invalid", "invalid DRI length")
            restart = s[0] << 8 | s[1]
        elif m == 0xDA:
            if not s:
                raise Fail("invalid", "empty SOS segment")
            if s[0] != len(comps):
                raise Fail("invalid", "SOS component count mismatch")
            for i in range(len(comps)):
                o = 1 + 2 * i
                if o + 1 >= len(s):
                    raise Fail("invalid", "truncated SOS segment")
                dc, ac = s[o + 1] >> 4, s[o + 1] & 15
                if dc > 3:
                    raise Fail("invalid", f"invalid DC Huffman table ID {dc} for component {s[o]}")
                if ac > 3:
                    raise Fail("invalid", f"invalid AC Huffman table ID {ac} for component {s[o]}")
                comps[i][3], comps[i][4] = dc, ac
            if not comps:
                raise Fail("panic", "SOS with no frame components")
            break
        elif m == 0xD9:
            raise Fail("invalid", "no image data found")
    mw, mhh = -(-W // (mh * 8)), -(-H // (mv * 8))
    pw = [mw * c[0] * 8 for c in comps]
    planes = [bytearray(pw[i] * mhh * c[1] * 8) for i, c in enumerate(comps)]
    r = Bits(d[pos:pos + entropy_end(d[pos:])])
    pred = [0, 0, 0]
    count = 0
    try:
        for my in range(mhh):
            for mx in range(mw):
                if restart and count and count % restart == 0:
                    pred = [0, 0, 0]
                for ci, (h, v, qid, dc, ac) in enumerate(comps):
                    for by in range(v):
                        for bx in range(h):
                            k64 = [0] * 64
                            cat = huff(dct[dc], r)
                            diff = amplitude(r, cat) if cat else 0
                            pred[ci] = i32(pred[ci] + diff)
                            k64[0] = i16(pred[ci])
                            k = 1
                            while k < 64:
                                sym = huff(act[ac], r)
                                if sym == 0:
                                    break
                                if sym == 0xF0:
                                    k += 16
                                    continue
                                k += sym >> 4
                                if k >= 64:
                                    break
                                if sym & 15:
                                    k64[k] = i16(amplitude(r, sym & 15))
                                k += 1
                            px = idct(k64, quant[qid])
                            x0, y0 = (mx * h + bx) * 8, (my * v + by) * 8
                            for yy in range(8):
                                planes[ci][(y0 + yy) * pw[ci] + x0:(y0 + yy) * pw[ci] + x0 + 8] = bytes(
                                    px[8 * yy:8 * yy + 8])
                count += 1
    except Bits.End:
        pass
    out = bytearray()
    if len(comps) == 1:
        for y in range(H):
            for x in range(W):
                i = y * pw[0] + x
                out.append(planes[0][i] if i < len(planes[0]) else 0)
        return ("ok", W, H, 0, bytes(out))
    yw = mw * mh * 8
    hb, vb = mh // comps[1][0], mv // comps[1][1]
    hr, vr = mh // comps[2][0], mv // comps[2][1]
    for y in range(H):
        for x in range(W):
            yi, bi, ri = y * yw + x, (y // vb) * pw[1] + x // hb, (y // vr) * pw[2] + x // hr
            Y = planes[0][yi] if yi < len(planes[0]) else 0
            cb = (planes[1][bi] if bi < len(planes[1]) else 128) - 128
            cr = (planes[2][ri] if ri < len(planes[2]) else 128) - 128
            for val in (Y + ((cr * 359) >> 8), Y - ((cb * 88 + cr * 183) >> 8), Y + ((cb * 454) >> 8)):
                out.append(min(max(val, 0), 255))
    return ("ok", W, H, 2, bytes(out))
