"""Constructed PNG files for the decoder tests: every colour type and legal bit depth, all five filters (row 0 too),
palettes with and without tRNS, chunk layouts, every zlib level and strategy, and hand-built DEFLATE streams that
reach pixo's table quirks and each of its inflate errors.  Deterministic; numpy and zlib only."""
from __future__ import annotations

import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(t: bytes, data: bytes, crc: int | None = None) -> bytes:
    c = zlib.crc32(t + data) if crc is None else crc
    return struct.pack(">I", len(data)) + t + data + struct.pack(">I", c & 0xFFFFFFFF)


def ihdr(w, h, depth, ct, comp=0, filt=0, interlace=0) -> bytes:
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ct, comp, filt, interlace))


def png(w, h, depth, ct, stream: bytes, pre=(), post=(), idat_split=None) -> bytes:
    """A file: IHDR, the chunks in pre, the stream in IDAT chunks (cut at idat_split offsets), post, IEND."""
    cuts = [0] + list(idat_split or []) + [len(stream)]
    idats = b"".join(chunk(b"IDAT", stream[a:b]) for a, b in zip(cuts, cuts[1:]))
    return SIG + ihdr(w, h, depth, ct) + b"".join(pre) + idats + b"".join(post) + chunk(b"IEND", b"")


def row_bytes(w, depth, ct):
    return (w * depth * CHANNELS[ct] + 7) // 8


def filter_bpp(depth, ct):
    return max(1, depth * CHANNELS[ct] // 8) if ct != 3 else 1


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def filter_rows(raw: np.ndarray, filters, bpp: int) -> bytes:
    """raw [h, sb] unfiltered rows -> the filtered stream with the given filter type per row."""
    out = bytearray()
    h, sb = raw.shape
    for y in range(h):
        f = filters[y % len(filters)]
        r = [int(v) for v in raw[y]]
        p = [int(v) for v in raw[y - 1]] if y else [0] * sb
        out.append(f)
        for i in range(sb):
            a = r[i - bpp] if i >= bpp else 0
            c = p[i - bpp] if i >= bpp else 0
            pred = (0, a, p[i], (a + p[i]) // 2, _paeth(a, p[i], c))[f] if f <= 4 else 0
            out.append((r[i] - pred) & 255)
    return bytes(out)


def image(w, h, depth, ct, seed, filters=(0, 1, 2, 3, 4), level=6, strategy=zlib.Z_DEFAULT_STRATEGY, pre=(),
          post=(), idat_split=None):
    rng = np.random.default_rng(seed)
    sb = row_bytes(w, depth, ct)
    raw = rng.integers(0, 256, (h, sb), dtype=np.uint8)
    data = filter_rows(raw, filters, filter_bpp(depth, ct))
    co = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    return png(w, h, depth, ct, co.compress(data) + co.flush(), pre, post, idat_split)


# ---- hand-built DEFLATE ------------------------------------------------------------------------------------

class Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, n):   # LSB first
        self.v |= (value & ((1 << n) - 1)) << self.n
        self.n += n

    def code(self, code, n):   # a Huffman code, MSB first
        for k in range(n - 1, -1, -1):
            self.put((code >> k) & 1, 1)

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical(lengths):
    """pixo's codes for a list of code lengths (no completeness check)."""
    bl = [0] * 16
    for L in lengths:
        if L:
            bl[L] += 1
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for L in lengths:
        if L:
            out.append(nxt[L])
            nxt[L] += 1
        else:
            out.append(None)
    return out


def zwrap(deflate: bytes, payload_adler: bytes | None = None, cmf=0x78, flg=0x01) -> bytes:
    return bytes([cmf, flg]) + deflate + (payload_adler if payload_adler is not None else b"\0\0\0\0")


def zlib_of(deflate: bytes, produced: bytes) -> bytes:
    return zwrap(deflate, struct.pack(">I", zlib.adler32(produced)))


CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def dynamic_block(bits: Bits, lit_lens, dist_lens, final=True, cl_lens=None, length_syms=None):
    """A dynamic block header: code lengths sent literally through a code length code of 5-bit codes (or the given
    cl_lens and symbol sequence)."""
    bits.put(1 if final else 0, 1)
    bits.put(2, 2)
    bits.put(len(lit_lens) - 257, 5)
    bits.put(len(dist_lens) - 1, 5)
    if cl_lens is None:
        cl_lens = [5] * 19
    bits.put(15, 4)
    for k in range(19):
        bits.put(cl_lens[CL_ORDER[k]], 3)
    clc = canonical(cl_lens)
    seq = length_syms if length_syms is not None else [(L, None) for L in list(lit_lens) + list(dist_lens)]
    for sym, extra in seq:
        bits.code(clc[sym], cl_lens[sym])
        if extra is not None:
            bits.put(*extra)
    return canonical(list(lit_lens)), canonical(list(dist_lens))


def gray8_file(stream: bytes, w: int, h: int) -> bytes:
    return png(w, h, 8, 0, stream)


def hand_built():
    """(name, file) pairs of 8-bit gray files around hand-built streams."""
    out = []
    # a payload of w x h gray, filter None rows
    w, h = 7, 3
    rows = bytes(b for y in range(h) for b in [0] + [(y * 31 + x * 7) & 255 for x in range(w)])

    def lit_stream(lit_lens, dist_lens, payload, final=True, tail=None):
        b = Bits()
        lc, dc = dynamic_block(b, lit_lens, dist_lens, final)
        for ch in payload:
            b.code(lc[ch], lit_lens[ch])
        if tail:
            tail(b, lc, dc)
        b.code(lc[256], lit_lens[256])
        return b.bytes()

    # complete 9-bit code over 257 symbols + some 10-bit ones: the slow path
    L = [9] * 256 + [9] + [0] * 29
    L[250:256] = [10] * 6
    L[256] = 10
    D = [1]
    out.append(("slow_path_codes", gray8_file(zlib_of(lit_stream(L, D, rows), rows), w, h)))
    # 15-bit codes
    L2 = [8] * 256 + [15] + [0] * 29
    L2[0] = 15
    out.append(("fifteen_bit_codes", gray8_file(zlib_of(lit_stream(L2, D, rows), rows), w, h)))
    # oversubscribed: every symbol 1 bit (later symbols win the lookup; decode_slow takes the first)
    L3 = [1] * 257 + [0] * 29
    out.append(("oversubscribed", gray8_file(zlib_of(lit_stream(L3, D, b""), b""), w, h)))
    L3b = [2] * 257 + [0] * 29
    out.append(("oversubscribed_2bit", gray8_file(zlib_of(lit_stream(L3b, D, b"\x00\x01"), b""), w, h)))
    # incomplete table: a code no symbol has
    L4 = [0] * 286
    L4[0], L4[256] = 2, 2
    b = Bits()
    lc, dc = dynamic_block(b, L4, D)
    b.code(3, 2)
    out.append(("incomplete_table", gray8_file(zlib_of(b.bytes(), b""), w, h)))
    # a single-code table: only the end-of-block symbol
    L5 = [0] * 256 + [1] + [0] * 29
    out.append(("single_code_eob", gray8_file(zlib_of(lit_stream(L5, D, b""), b""), w, h)))
    # single code + a one-code distance table: a match of 258 from a literal
    L6 = [0] * 286
    L6[0], L6[256], L6[285] = 2, 2, 1
    b = Bits()
    lc, dc = dynamic_block(b, L6, [1])
    b.code(lc[0], 2)
    payload = b"\0"
    for _ in range(4):
        b.code(lc[285], 1)
        b.code(dc[0], 1)
        payload += b"\0" * 258
    b.code(lc[256], 2)
    out.append(("matches_258", png(1, 1, 8, 0, zlib_of(b.bytes(), payload))))   # too long for a 1x1 frame
    # empty distance table used by a match
    L7 = [0] * 286
    L7[0], L7[256], L7[257] = 2, 2, 1
    b = Bits()
    lc, dc = dynamic_block(b, L7, [0])
    b.code(lc[0], 2)
    b.code(lc[257], 1)
    out.append(("empty_distance_table", gray8_file(zlib_of(b.bytes(), b""), w, h)))
    # distance too far back
    L8 = [0] * 286
    L8[0], L8[256], L8[257] = 2, 2, 1
    Dd = [0] * 30
    Dd[5] = 1
    b = Bits()
    lc, dc = dynamic_block(b, L8, Dd)
    b.code(lc[0], 2)
    b.code(lc[257], 1)
    b.code(dc[5], 1)
    b.put(0, 1)
    out.append(("distance_too_far", gray8_file(zlib_of(b.bytes(), b""), w, h)))
    # symbols 286/287 and distances 30/31 in a dynamic block (hlit 288, hdist 32)
    for sym in (286, 287):
        Lx = [0] * 288
        Lx[sym], Lx[256] = 1, 1
        b = Bits()
        lc, dc = dynamic_block(b, Lx, [1] * 1 + [0] * 31)
        b.code(lc[sym], 1)
        out.append((f"dynamic_litlen_{sym}", gray8_file(zlib_of(b.bytes() + b"\0", b""), w, h)))
    for dsym in (30, 31):
        Lx = [0] * 286
        Lx[0], Lx[256], Lx[257] = 2, 2, 1
        Dx = [0] * 32
        Dx[dsym] = 1
        b = Bits()
        lc, dc = dynamic_block(b, Lx, Dx)
        b.code(lc[0], 2)
        b.code(lc[257], 1)
        b.code(dc[dsym], 1)
        out.append((f"dynamic_dist_{dsym}", gray8_file(zlib_of(b.bytes() + b"\0", b""), w, h)))
    # fixed table: 286 / 287 and distance 30 / 31
    for sym, code in ((286, 0b11000110), (287, 0b11000111)):
        b = Bits()
        b.put(1, 1)
        b.put(1, 2)
        b.code(code, 8)
        out.append((f"fixed_litlen_{sym}", gray8_file(zlib_of(b.bytes() + b"\0\0", b""), w, h)))
    for dsym in (30, 31):
        b = Bits()
        b.put(1, 1)
        b.put(1, 2)
        b.code(0b00110000, 8)            # literal 0
        b.code(0b0000001, 7)             # length 3 (257)
        b.code(dsym, 5)
        out.append((f"fixed_dist_{dsym}", gray8_file(zlib_of(b.bytes() + b"\0\0", b""), w, h)))
    # repeat code at start; too many code lengths (16, 17 and 18)
    b = Bits()
    dynamic_block(b, [8] * 257, [1], length_syms=[(16, (0, 2))])
    out.append(("repeat_at_start", gray8_file(zlib_of(b.bytes() + b"\0" * 4, b""), w, h)))
    for sym, extra in ((16, (3, 2)), (17, (7, 3)), (18, (127, 7))):
        seq = [(8, None)] * 256 + [(8, None)] + [(sym, extra)]
        b = Bits()
        dynamic_block(b, [8] * 257, [1], length_syms=seq)
        out.append((f"too_many_lengths_{sym}", gray8_file(zlib_of(b.bytes() + b"\0" * 8, b""), w, h)))
    # all-zero code length code: an empty table
    b = Bits()
    dynamic_block(b, [8] * 257, [1], cl_lens=[0] * 19, length_syms=[])
    out.append(("empty_cl_table", gray8_file(zlib_of(b.bytes() + b"\0" * 4, b""), w, h)))
    # stored blocks: LEN/NLEN mismatch, block type 3, a stored block past the data, stored then fixed
    b = Bits()
    b.put(1, 1); b.put(0, 2); b.put(0, 5)
    st = b.bytes() + struct.pack("<HH", 5, 0x1234) + b"abcde"
    out.append(("len_nlen_mismatch", gray8_file(zlib_of(st, b""), w, h)))
    b = Bits()
    b.put(1, 1); b.put(3, 2)
    out.append(("block_type_3", gray8_file(zlib_of(b.bytes() + b"\0", b""), w, h)))
    b = Bits()
    b.put(1, 1); b.put(0, 2); b.put(0, 5)
    st = b.bytes() + struct.pack("<HH", 100, 0xFFFF ^ 100) + b"x" * 10
    out.append(("stored_past_end", gray8_file(zlib_of(st, b""), w, h)))
    b = Bits()
    b.put(0, 1); b.put(0, 2); b.put(0, 5)
    st = b.bytes() + struct.pack("<HH", len(rows) - 2, 0xFFFF ^ (len(rows) - 2)) + rows[:-2]
    b2 = Bits()
    b2.put(1, 1); b2.put(1, 2)
    for ch in rows[-2:]:
        b2.code(0b00110000 + ch, 8) if ch < 144 else b2.code(0b110010000 + ch - 144, 9)
    b2.code(0, 7)
    out.append(("stored_then_fixed", gray8_file(zlib_of(st + b2.bytes(), rows), w, h)))
    # the final symbol inside the last 9 bits (try_peek_bits takes a short code that fits)
    b = Bits()
    b.put(1, 1); b.put(1, 2)
    for ch in rows:
        b.code(0b00110000 + ch, 8) if ch < 144 else b.code(0b110010000 + ch - 144, 9)
    b.code(0, 7)
    out.append(("final_symbol_near_end", gray8_file(zlib_of(b.bytes(), rows), w, h)))
    # end of data inside a symbol
    out.append(("eos_in_symbol", gray8_file(zlib_of(b.bytes()[:-3], rows), w, h)))
    # output shorter / longer than expected, a ~1000x expansion past it, a bad Adler, trailing bytes, FDICT
    short = zlib.compress(rows[:-1])
    out.append(("output_short", gray8_file(short, w, h)))
    longer = zlib.compress(rows + b"\0\0\0")
    out.append(("output_long", gray8_file(longer, w, h)))
    big = zlib.compress(rows + bytes(1000 * len(rows)), 9)
    out.append(("expansion_1000x", gray8_file(big, w, h)))
    bomb = zlib.compress(bytes(200000), 9)
    out.append(("huge_claim_small_idat", png(100000, 100000, 8, 0, bomb)))
    good = zlib.compress(rows)
    out.append(("bad_adler", gray8_file(good[:-1] + bytes([good[-1] ^ 1]), w, h)))
    out.append(("trailing_after_final", gray8_file(good[:-4] + b"\xAA\xBB\xCC" + good[-4:], w, h)))
    out.append(("fdict", gray8_file(bytes([0x78, 0x20 | (31 - (0x7820 % 31))]) + good[2:], w, h)))
    out.append(("cinfo_unchecked", gray8_file(bytes([0xF8, 31 - (0xF800 % 31)]) + good[2:], w, h)))
    out.append(("zlib_too_short", gray8_file(good[:5], w, h)))
    out.append(("zlib_bad_cm", gray8_file(bytes([0x79, 0x01]) + good[2:], w, h)))
    out.append(("zlib_bad_fcheck", gray8_file(bytes([0x78, 0x02]) + good[2:], w, h)))
    return out


def structural():
    """(name, file) pairs of chunk layouts and the errors decided around the chunk walk, in pixo's order."""
    out = []
    rows = bytes([0, 1, 2, 3, 0, 4, 5, 6])
    z = zlib.compress(rows)
    base = png(3, 2, 8, 0, z)
    out.append(("plain", base))
    out.append(("not_png", b"\x89PNX" + base[4:]))
    out.append(("short", base[:7]))
    out.append(("trailing_bytes_ignored", base + b"junk!"))
    out.append(("bytes_after_iend_chunk", base + chunk(b"zzZz", b"x")))
    out.append(("truncated_chunk", SIG + ihdr(3, 2, 8, 0) + b"\0\0\3\xe8IDAT" + z + b"\0" * 8))
    out.append(("no_iend", base[:-12]))
    out.append(("no_iend_short_tail", base[:-12] + b"\0" * 11))
    out.append(("no_ihdr", SIG + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("crc_unknown_chunk", SIG + ihdr(3, 2, 8, 0) + chunk(b"abCd", b"xyz", 1) + chunk(b"IDAT", z) +
                chunk(b"IEND", b"")))
    out.append(("crc_non_utf8_type", SIG + ihdr(3, 2, 8, 0) + chunk(b"\xff\xc3\x28A", b"", 7) + chunk(b"IDAT", z) +
                chunk(b"IEND", b"")))
    out.append(("crc_utf8_type", SIG + ihdr(3, 2, 8, 0) + chunk("é€".encode()[:4], b"", 7) + chunk(b"IDAT", z) +
                chunk(b"IEND", b"")))
    out.append(("crc_ihdr", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 3, 2, 8, 0, 0, 0, 0), 5) +
                chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("ihdr_length", SIG + chunk(b"IHDR", b"\0" * 12) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("ihdr_color_type", SIG + ihdr(3, 2, 8, 5) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("plte_length", SIG + ihdr(3, 2, 8, 3) + chunk(b"PLTE", b"\0" * 4) + chunk(b"IDAT", z) +
                chunk(b"IEND", b"")))
    out.append(("zero_width", png(0, 2, 8, 0, z)))
    out.append(("zero_height", png(3, 0, 8, 0, z)))
    out.append(("too_wide", png((1 << 24) + 1, 2, 8, 0, z)))
    out.append(("too_tall_limit_ok", png(3, 1 << 24, 8, 0, z)))
    out.append(("compression_method", SIG + ihdr(3, 2, 8, 0, comp=1) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("filter_method", SIG + ihdr(3, 2, 8, 0, filt=1) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("adam7", SIG + ihdr(3, 2, 8, 0, interlace=1) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("bit_depth", png(3, 2, 4, 2, z)))
    out.append(("bit_depth_indexed_16", png(3, 2, 16, 3, z)))
    out.append(("no_idat", SIG + ihdr(3, 2, 8, 0) + chunk(b"IEND", b"")))
    out.append(("empty_idats", SIG + ihdr(3, 2, 8, 0) + chunk(b"IDAT", b"") + chunk(b"IEND", b"")))
    # precedence: the order the checks run in
    out.append(("iend_before_ihdr_missing", SIG + chunk(b"IEND", b"") + ihdr(3, 2, 8, 0)))
    out.append(("zero_dims_and_adam7", SIG + ihdr(0, 0, 8, 0, interlace=1) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("adam7_and_bad_depth", SIG + ihdr(3, 2, 3, 0, interlace=1) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("bad_depth_and_no_idat", SIG + ihdr(3, 2, 3, 0) + chunk(b"IEND", b"")))
    out.append(("no_iend_and_no_ihdr", SIG + chunk(b"IDAT", z)))
    badcrc_idat = SIG + ihdr(3, 2, 8, 0) + chunk(b"IDAT", z, 0x1234)
    out.append(("idat_crc", badcrc_idat + chunk(b"IEND", b"")))
    out.append(("idat_crc_before_truncation", badcrc_idat + b"\0\0\0\x20tEXt"))
    out.append(("idat_crc_before_bad_plte", badcrc_idat + chunk(b"PLTE", b"\0\0") + chunk(b"IEND", b"")))
    out.append(("idat_crc_before_missing_iend", badcrc_idat))
    out.append(("idat_crc_beats_zlib_header", SIG + ihdr(3, 2, 8, 0) + chunk(b"IDAT", b"\0\0" + z[2:], 9) +
                chunk(b"IEND", b"")))
    out.append(("idat_crc_second_chunk", SIG + ihdr(3, 2, 8, 0) + chunk(b"IDAT", z[:3]) + chunk(b"IDAT", z[3:], 9) +
                chunk(b"IEND", b"")))
    out.append(("bad_plte_before_idat_crc", SIG + ihdr(3, 2, 8, 0) + chunk(b"PLTE", b"\0\0") +
                chunk(b"IDAT", z, 9) + chunk(b"IEND", b"")))
    # repeated chunks: the last IHDR / PLTE / tRNS wins, IDATs concatenate, the walk stops at the first IEND
    out.append(("two_ihdr", SIG + ihdr(9, 9, 16, 6) + ihdr(3, 2, 8, 0) + chunk(b"IDAT", z) + chunk(b"IEND", b"")))
    out.append(("idat_after_iend_ignored", SIG + ihdr(3, 2, 8, 0) + chunk(b"IDAT", z) + chunk(b"IEND", b"") +
                chunk(b"IDAT", b"garbage")))
    out.append(("split_idat", png(3, 2, 8, 0, z, idat_split=[1, 1, 2, 5])))
    out.append(("zero_length_idats", png(3, 2, 8, 0, z, idat_split=[0, 0, 4, 4])))
    out.append(("unknown_chunks", png(3, 2, 8, 0, z, pre=[chunk(b"tEXt", b"k\0v"), chunk(b"abCD", b"")],
                                      post=[chunk(b"zzzz", b"123")])))
    out.append(("idat_before_ihdr", SIG + chunk(b"IDAT", z) + ihdr(3, 2, 8, 0) + chunk(b"IEND", b"")))
    # filters: an invalid filter type (first bad row reported), and one that beats a missing PLTE
    bad = bytes([0, 1, 2, 3, 7, 4, 5, 6])
    out.append(("bad_filter_row1", png(3, 2, 8, 0, zlib.compress(bad))))
    bad2 = bytes([9, 1, 2, 3, 5, 4, 5, 6])
    out.append(("bad_filter_row0", png(3, 2, 8, 0, zlib.compress(bad2))))
    out.append(("bad_filter_beats_missing_plte", png(3, 2, 8, 3, zlib.compress(bad))))
    out.append(("missing_plte", png(3, 2, 8, 3, z)))
    out.append(("size_beats_bad_filter", png(3, 2, 8, 0, zlib.compress(bad + b"\0"))))
    out.append(("adler_beats_size", png(3, 2, 8, 0, zlib.compress(rows + b"\0")[:-1] + b"\0")))
    return out


def palettes():
    out = []
    rng = np.random.default_rng(7)
    for depth in (1, 2, 4, 8):
        n = 1 << depth
        w, h = 13, 5
        raw = rng.integers(0, 256, (h, row_bytes(w, depth, 3)), dtype=np.uint8)
        z = zlib.compress(filter_rows(raw, (0, 1, 2, 3, 4), 1))
        full = bytes(rng.integers(0, 256, 3 * n, dtype=np.uint8))
        short = full[:3 * max(1, n // 2)]
        out.append((f"pal{depth}", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", full)])))
        out.append((f"pal{depth}_short_plte", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", short)])))
        out.append((f"pal{depth}_empty_plte", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", b"")])))
        out.append((f"pal{depth}_trns", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", full),
                                                                    chunk(b"tRNS", bytes(range(0, 256, 3))[:n])])))
        out.append((f"pal{depth}_short_trns", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", full),
                                                                          chunk(b"tRNS", b"\x10")])))
        out.append((f"pal{depth}_opaque_trns", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", full),
                                                                           chunk(b"tRNS", b"\xff" * n)])))
        out.append((f"pal{depth}_long_trns", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", short),
                                                                         chunk(b"tRNS", b"\xff" * 300 + b"\x01")])))
        out.append((f"pal{depth}_two_plte", png(w, h, depth, 3, z, pre=[chunk(b"PLTE", full), chunk(b"PLTE", short)])))
    # tRNS on gray and RGB is ignored
    out.append(("gray_trns", image(5, 4, 8, 0, 1, pre=[chunk(b"tRNS", b"\0\1")])))
    out.append(("rgb_trns", image(5, 4, 8, 2, 2, pre=[chunk(b"tRNS", b"\0\1\0\2\0\3")])))
    return out


def colour_types():
    out = []
    k = 0
    for ct, depths in DEPTHS.items():
        for d in depths:
            for (w, h) in ((1, 1), (9, 7), (33, 5)):
                pre = [chunk(b"PLTE", bytes(np.random.default_rng(k).integers(0, 256, 768, dtype=np.uint8)))] \
                    if ct == 3 else []
                out.append((f"ct{ct}_d{d}_{w}x{h}", image(w, h, d, ct, k, pre=pre)))
                k += 1
    return out


def zlib_settings():
    out = []
    for level in range(10):
        out.append((f"level{level}", image(40, 9, 8, 6, 100 + level, level=level)))
    for name, s in (("fixed", zlib.Z_FIXED), ("huffman_only", zlib.Z_HUFFMAN_ONLY), ("rle", zlib.Z_RLE)):
        out.append((name, image(40, 9, 8, 2, 200, strategy=s)))
    # a smooth image, so that matches (and overlapping short-distance matches) are common
    w, h = 64, 16
    raw = (np.arange(h)[:, None] * 3 + (np.arange(w * 3)[None, :] // 7)).astype(np.uint8)
    for level in (1, 9):
        out.append((f"smooth_level{level}", png(w, h, 8, 2, zlib.compress(filter_rows(raw, (0, 1, 2, 3, 4), 3), level))))
    return out


def corpus():
    """Every constructed file, as (name, bytes)."""
    return structural() + hand_built() + palettes() + colour_types() + zlib_settings()


def truncations(data: bytes, step: int = 0):
    step = step or max(1, len(data) // 23)
    return [data[:n] for n in range(0, len(data), step)]


def bit_flips(data: bytes, count: int, seed: int):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        b = bytearray(data)
        i = int(rng.integers(8, len(b)))
        b[i] ^= 1 << int(rng.integers(0, 8))
        out.append(bytes(b))
    return out
