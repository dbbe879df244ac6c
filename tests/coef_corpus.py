"""Constructed quantised-coefficient arrays that drive the entropy coders to their edges - symbols,
block lengths, 0xFF stuffing and DC chains that no 8-bit image reaches.  numpy + the CPU oracle.

Every generator returns (y, cb, cr, w, h, ct, ss) in compute_all_coefficients' layout (natural
order int16 [n, 64]; 4:2:0 Y blocks TL, TR, BL, BR per MCU).  The edge each case names is asserted
by the tests that use it (the standard tables of ITU-T T.81 Annex K, the oracle's histograms, or
the block boundaries the independent decoder in jpeg_scan_decode.py reports).
"""
from __future__ import annotations

import heapq

import numpy as np

from jpeg_scan_decode import ZIGZAG

GRAY, RGB = 0, 2
S444, S420 = 0, 1

# ---- ITU-T T.81 Annex K.3 (typical Huffman tables) ----------------------------------------------
DC_LUM_BITS = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
DC_CHR_BITS = [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]
AC_LUM_BITS = [0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D]
AC_CHR_BITS = [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]
AC_LUM_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a"
    "3435363738393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a9293949596"
    "9798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2"
    "f3f4f5f6f7f8f9fa")
AC_CHR_VALS = bytes.fromhex(
    "00010203110405213106124151076171132232810814429 1a1b1c109233352f0156272d10a162434e125f11718191a26272829"
    "2a35363738393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495"
    "969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3"
    "f4f5f6f7f8f9fa".replace(" ", ""))


def code_lengths(bits, vals) -> dict:
    """symbol -> code length of a (BITS, HUFFVAL) table"""
    out, k = {}, 0
    for ln, n in enumerate(bits, 1):
        for _ in range(n):
            out[vals[k]] = ln
            k += 1
    return out


DC_LUM = code_lengths(DC_LUM_BITS, list(range(12)))
DC_CHR = code_lengths(DC_CHR_BITS, list(range(12)))
AC_LUM = code_lengths(AC_LUM_BITS, AC_LUM_VALS)
AC_CHR = code_lengths(AC_CHR_BITS, AC_CHR_VALS)
assert len(AC_LUM) == len(AC_CHR) == 162


def category(v: int) -> int:
    return abs(int(v)).bit_length()


def huffman_depth(counts) -> int:
    """Depth of an unconstrained Huffman tree over the non-zero counts (heapq build)."""
    heap = [(int(c), i, 0) for i, c in enumerate(counts) if c]
    heapq.heapify(heap)
    n = len(heap)
    while len(heap) > 1:
        a, b = heapq.heappop(heap), heapq.heappop(heap)
        heapq.heappush(heap, (a[0] + b[0], n, max(a[2], b[2]) + 1))
        n += 1
    return heap[0][2]


# ---- building blocks -----------------------------------------------------------------------------

def block(zz: dict, dc: int = 0) -> np.ndarray:
    """A natural-order block from {zig-zag position: value}."""
    b = np.zeros(64, np.int16)
    b[0] = dc
    for k, v in zz.items():
        b[ZIGZAG[k]] = v
    return b


def pack(symbols) -> list:
    """(run, value) AC symbols -> as few blocks as hold them in order (a symbol that does not fit
    starts the next block)."""
    out, cur, pos = [], {}, 1
    for run, v in symbols:
        if pos + run > 63:
            out.append(block(cur))
            cur, pos = {}, 1
        cur[pos + run] = v
        pos += run + 1
    out.append(block(cur))
    return out


def exact_block(bits: int) -> np.ndarray:
    """A block of exactly `bits` bits on the standard LUMA tables when its DC difference is 0 (2 bits):
    (0, s) symbols with all-ones amplitudes, then EOB."""
    cost = {s: AC_LUM[s] + s for s in range(1, 11)}          # (0, s) + amplitude
    target = bits - DC_LUM[0] - AC_LUM[0x00]
    n26 = max(0, (target - 40) // cost[10])
    for combo in _small_sums(target - n26 * cost[10], cost):
        sizes = [10] * n26 + list(combo)
        if len(sizes) <= 62:
            return block({k + 1: (1 << s) - 1 for k, s in enumerate(sizes)})
    raise ValueError(bits)


def _small_sums(rem, cost):
    """size lists of at most four (0, s) symbols whose costs sum to rem"""
    out = []
    sizes = list(cost)
    for a in [None] + sizes:
        for b in [None] + sizes:
            for c in [None] + sizes:
                for d in [None] + sizes:
                    combo = [x for x in (a, b, c, d) if x]
                    if sum(cost[x] for x in combo) == rem:
                        out.append(tuple(combo))
    return out


def heavy_block(sign: int = 1) -> np.ndarray:
    """All 63 AC = +-1023: 63 x (0, 10) + ten amplitude bits, no EOB."""
    return block({k: sign * 1023 for k in range(1, 64)})


def with_dc_chain(blocks, diffs) -> list:
    """Copies of `blocks` whose DC values follow the difference sequence (int16 wrapping)."""
    out, dc = [], 0
    for i, b in enumerate(blocks):
        dc = ((dc + int(diffs[i % len(diffs)]) + 32768) & 0xFFFF) - 32768
        c = b.copy()
        c[0] = dc
        out.append(c)
    return out


def frame(y_blocks, c_blocks, ct, ss, mcus_x=16):
    """Arrays of a frame of ct / ss big enough for the lists (cycled to fill it): y_blocks fill the Y
    array in index order, c_blocks the Cb array and (rotated) the Cr array."""
    ypm = 4 if (ct == RGB and ss == S420) else 1
    need = max((len(y_blocks) + ypm - 1) // ypm, len(c_blocks) if ct == RGB else 0, 1)
    mx = min(need, mcus_x)
    my = (need + mx - 1) // mx
    n = mx * my
    mcu = 16 if ypm == 4 else 8
    y = np.stack([y_blocks[i % len(y_blocks)] for i in range(n * ypm)])
    if ct == GRAY:
        z = np.zeros((0, 64), np.int16)
        return y, z, z, mx * mcu, my * mcu, ct, ss
    cb = np.stack([c_blocks[i % len(c_blocks)] for i in range(n)])
    cr = np.stack([c_blocks[(i + 5) % len(c_blocks)] for i in range(n)])
    return y, cb, cr, mx * mcu, my * mcu, ct, ss


def _dc_sweep():
    """DC differences of every category 0..11, both signs: +-2^(c-1), +-(2^c - 1), incl. 1024 / 2047"""
    d = [0]
    for c in range(1, 12):
        for m in (1 << (c - 1), (1 << c) - 1):
            d += [m, -m]
    return d


# ---- the corpus -----------------------------------------------------------------------------------

def symbol_sweep(ct=RGB, ss=S444):
    """Every AC (run 0-15, size 1-10) at the extremes of its size, both signs, ZRL, EOB, and every DC
    category 0-11 in both signs - in Y and in both chroma arrays."""
    syms = []
    for run in range(16):
        for s in range(1, 11):
            for v in ((1 << (s - 1)), (1 << s) - 1):
                syms += [(run, v), (run, -v)]
    syms += [(16, 1), (20, -1023), (33, 512)]          # ZRL, then (4, s) / (1, s)
    blocks = with_dc_chain(pack(syms), _dc_sweep())
    return frame(blocks, blocks[::-1], ct, ss)


def zero_runs(ct=RGB, ss=S444):
    """Runs of 15, 16, 17, 31, 32, 47, 48 and 62 zeros before a coefficient; zig-zag 63 set with no
    EOB; only zig-zag 63 set (three ZRLs, then (14, s)); DC only; all zero."""
    bl = []
    for i, run in enumerate((15, 16, 17, 31, 32, 47, 48, 62)):
        bl.append(block({1 + run: (1, -1023, 512, -3)[i % 4]}, dc=i * 3))
        bl.append(block({1 + run: 7, min(63, 2 + run): -1}))
    bl.append(block({k: (k % 5) - 2 or 1 for k in range(1, 64)}, dc=-40))
    bl.append(block({63: -700}, dc=5))
    bl.append(block({}, dc=100))
    bl.append(block({}))
    bl.append(block({62: 1, 63: 1}))
    return frame(bl * 4, bl[3:] + bl[:3], ct, ss)


BLOCK_BITS = (511, 512, 513, 543, 544, 545)
MAX_BLOCK_BITS = 1658


def block_lengths():
    """Gray frame, standard tables: blocks of exactly 511, 512, 513, 543, 544 and 545 bits (around the
    512-bit shared slot and its first spill word) and the 1658-bit maximum (DC category 11 + 63 AC of
    +-1023), at lanes 0, 15 and 31 of 32-block chunks, between short filler blocks.  Returns the case
    and {block index: expected bits}."""
    specials = [exact_block(b) for b in BLOCK_BITS]
    fill = block({1: 3, 5: -1})
    blocks, want = [], {}
    dcs = []
    for chunk in range(len(BLOCK_BITS) + 1):
        for lane in range(32):
            i = chunk * 32 + lane
            if lane in (0, 15, 31):
                if chunk < len(BLOCK_BITS):
                    blocks.append(specials[(chunk + lane) % len(specials)])
                    want[i] = BLOCK_BITS[(chunk + lane) % len(specials)]
                    dcs.append(dcs[-1] if dcs else 0)
                else:
                    blocks.append(heavy_block(1 if lane != 15 else -1))
                    want[i] = MAX_BLOCK_BITS
                    dcs.append(2047 if (not dcs or dcs[-1] == 0) else 0)
            else:
                blocks.append(fill)
                dcs.append(dcs[-1] if dcs else 0)
    blocks = [b.copy() for b in blocks]
    for b, d in zip(blocks, dcs):
        b[0] = d
    z = np.zeros((0, 64), np.int16)
    n = len(blocks)
    return (np.stack(blocks), z, z, 8 * 32, 8 * (n // 32), GRAY, S444), want


def stuffing_gray(nblocks=256):
    """Every block (0, 10) + 1023 63 times (16-bit code, ten 1-bits) with DC differences
    alternating +-2047: a scan of mostly 0xFF bytes."""
    bl = [heavy_block(1)] * nblocks
    z = np.zeros((0, 64), np.int16)
    y = np.stack(with_dc_chain(bl, [2047, -2047]))
    return y, z, z, 8 * 16, 8 * (nblocks // 16), GRAY, S444


def straddle(nblocks: int, border: int, phase: int, mcus_x: int = 8):
    """Gray frame: block border-1 ends in ten 1-bits (63 AC = +1023), block `border` starts with eight
    (DC difference +2047), and a tuner block before them (600 + phase bits) moves the border through
    the bit positions of a byte.  The tests pick the phase whose border byte is 0xFF."""
    fill = block({1: 2, 3: -1})
    bl = [fill] * nblocks
    bl[border - 2] = exact_block(600 + phase)
    bl[border - 1] = heavy_block(1)
    dcs = [0] * border + [2047] * (nblocks - border)
    bl = [b.copy() for b in bl]
    for b, d in zip(bl, dcs):
        b[0] = d
    bl[border][0] = 2047
    z = np.zeros((0, 64), np.int16)
    return np.stack(bl), z, z, 8 * mcus_x, 8 * (nblocks // mcus_x), GRAY, S444


def restart_padding():
    """Gray frame, restart interval 2 MCUs: every interval is a tuner block (600 + j bits) and a
    block that ends in ten 1-bits, so the interval's 1-padding of 8 - j bits completes a 0xFF byte
    (j = 1..7) - and j = 0, no padding.  Returns the case and its restart interval."""
    bl = []
    for j in (1, 2, 3, 4, 5, 6, 7, 0):
        bl += [exact_block(600 + j), heavy_block(1)]
    z = np.zeros((0, 64), np.int16)
    return (np.stack(bl), z, z, 8 * 16, 8, GRAY, S444), 2


def dc_chains(ct=RGB, ss=S444, nmcus=96):
    """DC differences of +-2047 at every block (so across every chunk, segment and band border), Cb
    and Cr chains of opposite sign (a predictor taken from the wrong array is off by 4094)."""
    ypm = 4 if (ct == RGB and ss == S420) else 1
    fill = [block({1: 1}), block({2: -5, 9: 3}), block({})]
    y = with_dc_chain(fill * (nmcus * ypm), [2047, -2047])[:nmcus * ypm]
    cb = with_dc_chain(fill * nmcus, [-2047, 2047])[:nmcus]
    crs = with_dc_chain(fill * nmcus, [2047, -2047])[:nmcus]
    out = list(frame(y, cb, ct, ss, mcus_x=8))
    if ct == RGB:
        out[2] = np.stack(crs)
    return tuple(out)


def dc_climb(ct=RGB, ss=S444, nmcus=64):
    """DC values that climb through the int16 range: every difference is +2047 (or -2047 in Cb),
    the values wrap at +-32768 several times.  Valid only without restart intervals."""
    ypm = 4 if (ct == RGB and ss == S420) else 1
    y = with_dc_chain([block({1: 1, 4: -2})] * (nmcus * ypm), [2047])
    c = with_dc_chain([block({2: 3})] * nmcus, [-2047])
    out = list(frame(y, c, ct, ss, mcus_x=8))
    if ct == RGB:
        out[2] = np.stack(with_dc_chain([block({3: -3})] * nmcus, [2047]))
    return tuple(out)


def fibonacci(nsym: int, ct=GRAY, ss=S444):
    """Luma AC symbol counts in Fibonacci proportion (nsym symbols (run 0-2, size 1..10)): with
    22 symbols the unconstrained Huffman tree is deeper than 16 (the standard tables are used); with 19
    the optimised table has
    16-bit codes.  DC differences are all 0."""
    fib = [1, 1]
    while len(fib) < nsym:
        fib.append(fib[-1] + fib[-2])
    kinds = [(r, s) for r in (0, 1, 2) for s in range(1, 11)][:nsym]
    rng = np.random.default_rng(nsym)
    seq = []
    for (r, s), n in zip(kinds, fib):
        seq += [(r, (1 << s) - 1)] * n
    order = rng.permutation(len(seq))
    syms = [(seq[i][0], seq[i][1] * (1 if i % 2 else -1)) for i in order]
    blocks = pack(syms)
    # one row of MCUs: a gray frame holds exactly these blocks (repeating some would skew the counts)
    return frame(blocks, blocks, ct, ss, mcus_x=len(blocks))


def dense(ct=RGB, ss=S420, w_mcus=32, h_mcus=24):
    """Every block near the 1658-bit maximum: 63 AC of +-1023 (signs varying by block) and DC
    differences of +-2047.  The scan is about 2x (4:2:0) to 4x (gray) the raw pixel bytes."""
    bl = [heavy_block(1), heavy_block(-1), block({k: (1023 if k % 3 else -1023) for k in range(1, 64)})]
    ypm = 4 if (ct == RGB and ss == S420) else 1
    n = w_mcus * h_mcus
    y = with_dc_chain(bl * (n * ypm // 3 + 1), [2047, -2047])[:n * ypm]
    c = with_dc_chain(bl * (n // 3 + 1), [-2047, 2047])[:n]
    return frame(y, c, ct, ss, mcus_x=w_mcus)


def geometries():
    return [(RGB, S420), (RGB, S444), (GRAY, S444)]


# cases every coder must code byte-identically (name -> generator taking (ct, ss))
MATRIX = {
    "symbol_sweep": symbol_sweep,
    "zero_runs": zero_runs,
    "dc_chains": dc_chains,
    "dc_climb": dc_climb,
    "fib_deep": lambda ct, ss: fibonacci(22, ct, ss),
    "fib_16bit": lambda ct, ss: fibonacci(19, ct, ss),
}
NO_RESTART = {"dc_climb"}    # differences are in range only while nothing resets the predictors
