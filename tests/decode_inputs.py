"""Large, well-formed inputs for the decoder tests, built fast enough to make full-size files in a test.

  filter_rows_np(raw, filters, bpp)   filter_rows (png_decode_corpus) vectorised: one filter type per row
  png_image(...)                      a PNG of seeded noise or a smooth image, with the filters, zlib level and
                                      strategy, and IDAT chunk lengths given; returns the file and its source rows
  jfif(w, h, comps, coefs, ...)       a baseline JPEG written from quantised coefficients in pixo's decode order:
                                      sampling factors 1-4 per axis, 8- or 16-bit DQT, the standard tables or tables
                                      built per file from the symbol counts, restart intervals with RSTn markers and
                                      1-bit padding, 0xFF stuffing
  sparse_coefs / dense_coefs          coefficients for jfif; safe_tails makes them decode exactly under pixo's reader

Coefficients travel as Coefs(dc, blk, k, val): one DC per block and the non-zero AC coefficients as (block, zig-zag
position, value), sorted by block then position, so a file of millions of blocks is written without a [n, 64] array.
Deterministic; numpy and zlib only.
"""
from __future__ import annotations

import dataclasses
import struct
import zlib

import numpy as np

from coef_corpus import (AC_CHR_BITS, AC_CHR_VALS, AC_LUM_BITS, AC_LUM_VALS, DC_CHR_BITS, DC_LUM_BITS)
from png_decode_corpus import CHANNELS, chunk, filter_bpp, png, row_bytes

# ---- PNG -----------------------------------------------------------------------------------------------------


def filter_rows_np(raw: np.ndarray, filters, bpp: int) -> bytes:
    """raw [h, sb] unfiltered rows -> the filtered stream; filters[y % len(filters)] is row y's type (types above 4
    predict 0, as filter_rows writes them)."""
    raw = np.ascontiguousarray(raw, np.uint8)
    h, sb = raw.shape
    f = np.resize(np.asarray(filters, np.uint8), h)
    out = np.empty((h, sb + 1), np.uint8)
    out[:, 0] = f
    step = max(1, (1 << 22) // max(sb, 1))   # rows per slice: bounded temporaries on 4K frames
    for y0 in range(0, h, step):
        y1 = min(h, y0 + step)
        r = raw[y0:y1].astype(np.int16)
        b = np.zeros_like(r)
        b[1:] = r[:-1]
        if y0:
            b[0] = raw[y0 - 1]
        a = np.zeros_like(r)
        a[:, bpp:] = r[:, :-bpp]
        c = np.zeros_like(r)
        c[:, bpp:] = b[:, :-bpp]
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        ft = f[y0:y1, None]
        pred = np.select([ft == 1, ft == 2, ft == 3, ft == 4], [a, b, (a + b) >> 1, paeth], 0)
        out[y0:y1, 1:] = (r - pred) & 255
    return out.tobytes()


def source_rows(w: int, h: int, depth: int, ct: int, seed: int, kind: str = "noise") -> np.ndarray:
    """[h, row bytes] unfiltered rows: seeded noise, or a smooth image of long runs and short-distance repeats."""
    sb = row_bytes(w, depth, ct)
    if kind == "noise":
        return np.random.default_rng(seed).integers(0, 256, (h, sb), dtype=np.uint8)
    y, x = np.arange(h)[:, None], np.arange(sb)[None, :]
    return ((y * 3 + x // 7 + seed) & 255).astype(np.uint8)


def png_image(w: int, h: int, depth: int, ct: int, seed: int, filters=(0, 1, 2, 3, 4), level: int = 6,
              strategy: int = zlib.Z_DEFAULT_STRATEGY, idat_chunks=None, kind: str = "noise", raw=None):
    """(file, raw rows).  filters: per-row types, cycled, or "random" for seeded per-row types; idat_chunks: IDAT
    payload lengths, cycled (the last chunk takes the rest); an indexed file gets a 256-entry PLTE."""
    if raw is None:
        raw = source_rows(w, h, depth, ct, seed, kind)
    if isinstance(filters, str):
        assert filters == "random"
        filters = np.random.default_rng(seed + 1).integers(0, 5, h)
    co = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    stream = co.compress(filter_rows_np(raw, filters, filter_bpp(depth, ct))) + co.flush()
    pre = [chunk(b"PLTE", palette(seed))] if ct == 3 else []
    return png(w, h, depth, ct, stream, pre=pre, idat_split=idat_split(len(stream), idat_chunks)), raw


def idat_split(n: int, chunks):
    """png()'s cut offsets for IDAT payloads of the given lengths, cycled, over a stream of n bytes"""
    if not chunks:
        return None
    split, o, k = [], 0, 0
    while o + chunks[k % len(chunks)] < n:
        o += chunks[k % len(chunks)]
        split.append(o)
        k += 1
    return split


def palette(seed: int) -> bytes:
    return bytes(np.random.default_rng(seed + 2).integers(0, 256, 768, dtype=np.uint8))


def expand_source(raw: np.ndarray, w: int, depth: int, ct: int, seed: int) -> np.ndarray:
    """The frame decode_png returns for the rows of png_image(..., seed): the high byte of 16-bit samples, bit
    replication of sub-8-bit gray, the PLTE lookup of indices; 8-bit rows as they are."""
    h = raw.shape[0]
    ch = CHANNELS[ct]
    if depth == 16:
        return np.ascontiguousarray(raw[:, :w * ch * 2:2]).reshape(-1)
    if depth == 8:
        v = raw[:, :w * ch]
    else:
        bits = np.unpackbits(raw, axis=1)[:, :w * depth].reshape(h, w, depth)
        v = (bits * (1 << np.arange(depth - 1, -1, -1, dtype=np.uint8))).sum(axis=2).astype(np.uint8)
    if ct == 3:
        return np.frombuffer(palette(seed), np.uint8).reshape(256, 3)[v].reshape(-1)
    if depth < 8:
        v = (v * {1: 255, 2: 0x55, 4: 0x11}[depth]).astype(np.uint8)
    return np.ascontiguousarray(v).reshape(-1)


# ---- baseline JPEG -------------------------------------------------------------------------------------------

STD = {"dc0": (DC_LUM_BITS, list(range(12))), "dc1": (DC_CHR_BITS, list(range(12))),
       "ac0": (AC_LUM_BITS, list(AC_LUM_VALS)), "ac1": (AC_CHR_BITS, list(AC_CHR_VALS))}


@dataclasses.dataclass
class Coefs:
    """Quantised coefficients of a file in decode order: dc[n]; the non-zero AC ones as blk / k (zig-zag position
    1-63) / val, sorted by (blk, k)."""
    dc: np.ndarray
    blk: np.ndarray
    k: np.ndarray
    val: np.ndarray

    @property
    def n(self) -> int:
        return len(self.dc)

    @classmethod
    def from_dense(cls, zz: np.ndarray) -> "Coefs":
        zz = np.asarray(zz, np.int16).reshape(-1, 64)
        b, k = np.nonzero(zz[:, 1:])
        return cls(zz[:, 0].astype(np.int64), b.astype(np.int64), k.astype(np.int64) + 1,
                   zz[b, k + 1].astype(np.int64))

    def dense(self) -> np.ndarray:
        out = np.zeros((self.n, 64), np.int16)
        out[:, 0] = self.dc
        out[self.blk, self.k] = self.val
        return out


def geometry(w: int, h: int, comps):
    """(mcu_w, mcu_h, blocks per MCU) as pixo sizes a frame: MCUs of 8 max_h x 8 max_v pixels."""
    mh = max(c[0] for c in comps)
    mv = max(c[1] for c in comps)
    return -(-w // (8 * mh)), -(-h // (8 * mv)), sum(c[0] * c[1] for c in comps)


def category(v: np.ndarray) -> np.ndarray:
    a = np.abs(np.asarray(v, np.int64))
    out = np.zeros(a.shape, np.int64)
    while (a >> out).any():
        out += (a >> out) > 0
    return out


def huffman_bits(counts) -> tuple:
    """(BITS, HUFFVAL) of an optimal table of codes of at most 16 bits for the symbol counts, by the procedure of
    ITU-T T.81 Annex K.2 (a reserved symbol keeps any code from being all ones)."""
    freq = [int(c) for c in counts] + [1]
    n = len(freq)
    codesize, others = [0] * n, [-1] * n
    live = {i for i in range(n) if freq[i]}
    while len(live) > 1:
        c1 = min(live, key=lambda i: (freq[i], -i))
        live.discard(c1)
        c2 = min(live, key=lambda i: (freq[i], -i))
        live.add(c1)
        live.discard(c2)
        freq[c1] += freq[c2]
        for c in (c1, c2):
            j = c
            codesize[j] += 1
            while others[j] >= 0:
                j = others[j]
                codesize[j] += 1
        j = c1
        while others[j] >= 0:
            j = others[j]
        others[j] = c2
    top = max(32, max(codesize))
    bits = [0] * (top + 1)
    for i in range(n):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(top, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1   # the reserved symbol
    vals = [s for L in range(1, top + 1) for s in range(n - 1) if codesize[s] == L]
    return bits[1:17], vals


def _codes(bits, vals):
    """code and length arrays over the 256 symbols of a (BITS, HUFFVAL) table (length 0: not in it)"""
    code, ln = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c, k = 0, 0
    for L in range(1, 17):
        for _ in range(bits[L - 1]):
            code[vals[k]], ln[vals[k]] = c, L
            c += 1
            k += 1
        c <<= 1
    return code, ln


def _symbols(C: Coefs, comp_of: np.ndarray, first_in_interval: np.ndarray):
    """Every block's symbols in scan order as (block, order key, table class, symbol, amplitude, category)."""
    n = C.n
    # DC differences, per component, predictors reset at each restart interval
    diff = np.empty(n, np.int64)
    for c in np.unique(comp_of):
        idx = np.nonzero(comp_of == c)[0]
        d = C.dc[idx].astype(np.int64)
        prev = np.concatenate([[0], d[:-1]])
        prev[first_in_interval[idx]] = 0
        diff[idx] = d - prev
    dcat = category(diff)
    blocks = np.arange(n, dtype=np.int64)
    # AC: a ZRL for every 16 zeros before a coefficient, then (run, size)
    prevk = np.zeros(len(C.k), np.int64)
    prevk[1:] = np.where(C.blk[1:] == C.blk[:-1], C.k[:-1], 0)
    run = C.k - prevk - 1
    acat = category(C.val)
    nzrl = run // 16
    zb = np.repeat(C.blk, nzrl)
    zk = np.repeat(C.k, nzrl)
    zj = np.arange(len(zb)) - np.repeat(np.cumsum(nzrl) - nzrl, nzrl)
    last = np.zeros(n, np.int64)
    np.maximum.at(last, C.blk, C.k)
    eob = np.nonzero(last < 63)[0]
    blk = np.concatenate([blocks, zb, C.blk, eob])
    key = np.concatenate([blocks * 4096, zb * 4096 + zk * 8 + zj, C.blk * 4096 + C.k * 8 + 4, eob * 4096 + 64 * 8])
    cls = np.concatenate([np.zeros(n, np.int64), np.ones(len(zb) + len(C.blk) + len(eob), np.int64)])
    sym = np.concatenate([dcat, np.full(len(zb), 0xF0), (run % 16) * 16 + acat, np.zeros(len(eob), np.int64)])
    amp = np.concatenate([diff, np.zeros(len(zb), np.int64), C.val, np.zeros(len(eob), np.int64)])
    cat = np.concatenate([dcat, np.zeros(len(zb), np.int64), acat, np.zeros(len(eob), np.int64)])
    o = np.argsort(key, kind="stable")
    return blk[o], cls[o], sym[o], amp[o], cat[o]


def _bits_to_bytes(vals: np.ndarray, lens: np.ndarray) -> np.ndarray:
    """MSB-first concatenation of vals[i] in lens[i] bits (a multiple of 8 in total)."""
    starts = np.cumsum(lens) - lens
    total = int(lens.sum())
    assert total % 8 == 0
    bits = np.empty(total, np.uint8)
    step = 1 << 18
    for s in range(0, len(lens), step):
        L, V, S = lens[s:s + step], vals[s:s + step], starts[s:s + step]
        if not len(L) or not L.sum():
            continue
        rl = np.repeat(L, L)
        off = np.arange(int(L.sum()), dtype=np.int64) - np.repeat(S - S[0], L)
        bits[S[0]:S[0] + int(L.sum())] = (np.repeat(V, L) >> (rl - 1 - off)) & 1
    return np.packbits(bits)


def seg(marker: int, payload: bytes) -> bytes:
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


class RestartTail(ValueError):
    """pixo's reader clears its bit buffer when it fetches an RSTn marker, so an interval whose last Huffman code,
    its amplitude and the padding after them are fewer than 8 bits loses those bits to the 8-bit peek."""


def jfif(w: int, h: int, comps, coefs, restart: int = 0, tables: str = "standard", dqt16=None) -> bytes:
    """A baseline JPEG of the coefficients (Coefs, or int16 [blocks, 64] in zig-zag order), in pixo's decode order:
    MCU by MCU, each component's v x h blocks in rows.  comps: (h, v, q) per component, q 64 values in zig-zag order;
    component c uses quantisation table c.  tables: "standard" (T.81 K.3: luma tables for component 0, chroma for
    the others) or "optimal" (per-component tables from the file's symbol counts).  dqt16: 16-bit DQT (default: when
    a value exceeds 255).  restart: the DRI interval in MCUs (0: none)."""
    C = coefs if isinstance(coefs, Coefs) else Coefs.from_dense(coefs)
    mw, mh, bpm = geometry(w, h, comps)
    nmcu = mw * mh
    if C.n != nmcu * bpm:
        raise ValueError(f"{C.n} blocks for {nmcu} MCUs of {bpm}")
    pattern = np.concatenate([np.full(hh * vv, c) for c, (hh, vv, _) in enumerate(comps)])
    comp_of = np.tile(pattern, nmcu)
    mcu = np.arange(C.n, dtype=np.int64) // bpm
    interval = mcu // restart if restart else np.zeros(C.n, np.int64)
    first = np.zeros(C.n, bool)
    for c in range(len(comps)):
        idx = np.nonzero(comp_of == c)[0]
        iv = interval[idx]
        first[idx[np.concatenate([[True], iv[1:] != iv[:-1]])]] = True
    blk, cls, sym, amp, cat = _symbols(C, comp_of, first)
    tid = np.where(comp_of[blk] == 0, 0, 1) if tables == "standard" else comp_of[blk]
    tabs = {}
    for t in np.unique(tid):
        for k in (0, 1):
            sel = (tid == t) & (cls == k)
            if tables == "standard":
                tabs[(k, t)] = STD[("dc" if k == 0 else "ac") + str(t)]
            else:
                tabs[(k, t)] = huffman_bits(np.bincount(sym[sel], minlength=256))
    code = np.zeros(len(sym), np.int64)
    ln = np.zeros(len(sym), np.int64)
    for (k, t), (bits, vals) in tabs.items():
        sel = (tid == t) & (cls == k)
        cd, cl = _codes(bits, vals)
        code[sel], ln[sel] = cd[sym[sel]], cl[sym[sel]]
    if (ln == 0).any():
        bad = sym[ln == 0][0]
        raise ValueError(f"symbol {bad:#04x} is not in its table")
    if (cat > 16).any():
        raise ValueError("a coefficient needs more than 16 amplitude bits")
    ampbits = np.where(amp < 0, amp - 1, amp) & ((1 << cat) - 1)
    vals = (code << cat) | ampbits
    lens = ln + cat
    # padding: 1 bits to the byte boundary at the end of each interval and of the scan
    iv = interval[blk]
    nint = int(iv[-1]) + 1 if len(iv) else 1
    tot = np.bincount(iv, weights=lens, minlength=nint).astype(np.int64)
    pad = (-tot) % 8
    ends = np.searchsorted(iv, np.arange(nint), "right")
    if nint > 1 and ((lens[ends[:-1] - 1] + pad[:-1]) < 8).any():
        raise RestartTail("an interval's last code, amplitude and padding are fewer than 8 bits: see safe_tails")
    vals = np.insert(vals, ends, (1 << pad) - 1)
    lens = np.insert(lens, ends, pad)
    data = _bits_to_bytes(vals, lens)
    # stuffing after every 0xFF, RSTn between intervals
    byte_ends = np.cumsum((tot + pad) // 8)[:-1]
    ff = np.nonzero(data == 0xFF)[0] + 1
    pos = np.concatenate([ff, np.repeat(byte_ends, 2)])
    order = np.concatenate([np.zeros(len(ff)), np.tile([1, 2], len(byte_ends))])
    ins = np.concatenate([np.zeros(len(ff), np.uint8),
                          np.stack([np.full(len(byte_ends), 0xFF), 0xD0 + np.arange(len(byte_ends)) % 8], 1).reshape(-1)
                          ]).astype(np.uint8)
    o = np.lexsort((order, pos))
    scan = np.insert(data, pos[o], ins[o]).tobytes()
    # headers
    ncomp = len(comps)
    big = dqt16 if dqt16 is not None else any(max(q) > 255 for _, _, q in comps)
    dqt = b"".join(bytes([(0x10 if big else 0) | c]) + (b"".join(struct.pack(">H", int(x)) for x in q) if big
                                                            else bytes(int(x) for x in q))
                   for c, (_, _, q) in enumerate(comps))
    sof = bytes([8]) + struct.pack(">HHB", h, w, ncomp) + b"".join(
        bytes([c + 1, hh << 4 | vv, c]) for c, (hh, vv, _) in enumerate(comps))
    dht = b"".join(bytes([k << 4 | t]) + bytes(bits) + bytes(vals) for (k, t), (bits, vals) in sorted(tabs.items()))
    tid_of = [0 if (tables == "standard" and c == 0) else (1 if tables == "standard" else c) for c in range(ncomp)]
    sos = bytes([ncomp]) + b"".join(bytes([c + 1, tid_of[c] << 4 | tid_of[c]]) for c in range(ncomp)) + b"\x00\x3F\x00"
    return (b"\xFF\xD8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00") + seg(0xDB, dqt) +
            seg(0xC0, sof) + seg(0xC4, dht) + (seg(0xDD, struct.pack(">H", restart)) if restart else b"") +
            seg(0xDA, sos) + scan + b"\xFF\xD9")


def _amplitudes(rng, n: int, cat_max: int) -> np.ndarray:
    cat = rng.integers(1, cat_max + 1, n)
    lo = 1 << (cat - 1)
    v = lo + (rng.random(n) * lo).astype(np.int64)
    v = np.minimum(v, (1 << cat) - 1)
    return np.where(rng.random(n) < 0.5, -v, v).astype(np.int64)


def _dc_walk(rng, n: int, cat_max: int, lim: int) -> np.ndarray:
    """DC values whose differences take every category up to cat_max (clipped to +-lim)."""
    d = np.where(rng.random(n) < 0.1, 0, _amplitudes(rng, n, cat_max))
    return np.clip(np.cumsum(d), -lim, lim)


def sparse_coefs(n: int, seed: int, nac: int = 3, dc_lim: int = 1023, ac_cat: int = 10) -> Coefs:
    """DC plus up to nac AC coefficients per block, at random zig-zag positions (long zero runs: ZRLs)."""
    rng = np.random.default_rng(seed)
    dc = _dc_walk(rng, n, 10, dc_lim)
    blk = np.repeat(np.arange(n, dtype=np.int64), nac)
    k = rng.integers(1, 64, n * nac)
    keep = rng.random(n * nac) < 0.7
    blk, k = blk[keep], k[keep]
    o = np.lexsort((k, blk))
    blk, k = blk[o], k[o]
    u = np.concatenate([[True], (blk[1:] != blk[:-1]) | (k[1:] != k[:-1])])[:len(blk)]
    blk, k = blk[u], k[u]
    return Coefs(dc, blk, k, _amplitudes(rng, len(blk), ac_cat))


def dense_coefs(n: int, seed: int, ac_cat: int = 10, dc_cat: int = 11, density: float = 0.6) -> Coefs:
    """Blocks of random AC coefficients over every category up to ac_cat, DC differences up to dc_cat; ac_cat 15
    and dc_cat 16 need the optimal tables."""
    rng = np.random.default_rng(seed)
    z = np.zeros((n, 64), np.int64)
    mask = rng.random((n, 63)) < density
    z[:, 1:][mask] = _amplitudes(rng, int(mask.sum()), ac_cat)
    lim = (1 << (dc_cat - 1)) - 1 if dc_cat <= 11 else 32767
    z[:, 0] = _dc_walk(rng, n, min(dc_cat, 15), lim)
    if dc_cat == 16:
        z[rng.random(n) < 0.05, 0] = -32768 + rng.integers(0, 2)   # differences of 16 bits
    return Coefs.from_dense(z.astype(np.int16))


def safe_tails(C: Coefs, bpm: int, restart: int, nmcu: int, seed: int = 0) -> Coefs:
    """The coefficients with the last block of every restart interval but the last ending on a coefficient at
    zig-zag position 63 of 7 amplitude bits, so that the interval's last code, amplitude and padding are at least 8
    bits and pixo's reader decodes it exactly (see RestartTail)."""
    if not restart or restart >= nmcu:
        return C
    tails = np.arange(restart, nmcu, restart, dtype=np.int64) * bpm - 1
    rng = np.random.default_rng(seed)
    keep = ~(np.isin(C.blk, tails) & (C.k == 63))
    tv = rng.integers(64, 128, len(tails)) * np.where(rng.random(len(tails)) < 0.5, -1, 1)
    blk = np.concatenate([C.blk[keep], tails])
    k = np.concatenate([C.k[keep], np.full(len(tails), 63)])
    val = np.concatenate([C.val[keep], tv])
    o = np.lexsort((k, blk))
    return Coefs(C.dc, blk[o], k[o], val[o])


def qtable(seed: int, hi: int = 255) -> list:
    return [int(x) for x in np.random.default_rng(seed).integers(1, hi + 1, 64)]
