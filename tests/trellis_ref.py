"""Pure-Python restatement of pixo's trellis_quantize (src/jpeg/trellis.rs:67-244), independent of the C
oracle: every arithmetic step is one numpy float32 operation, so each rounds once as binary32 does in the
reference.  Slow (a block takes milliseconds); used to cross-check the C oracle on constructed blocks."""
from __future__ import annotations

import math

import numpy as np

ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
          7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
          39, 46, 53, 60, 61, 54, 47, 55, 62, 63]
F = np.float32


def _i16(x: float) -> int:
    if math.isnan(x):
        return 0
    return int(max(-32768, min(32767, math.trunc(x))))


def _round_half_away(x: float) -> float:
    return math.copysign(math.floor(abs(x) + 0.5), x) if abs(x) < 2 ** 23 else x


def candidates(fq) -> list[int]:
    fq = float(fq)
    r, fl, ce = _i16(_round_half_away(fq)), _i16(math.floor(fq)), _i16(math.ceil(fq))
    c = [0]
    for v in (fl, r, ce):
        if v != 0 and v not in c:
            c.append(v)
    if abs(fq) > 1.5:
        e = ce + 1 if fq >= 0.0 else fl - 1
        if e not in c:
            c.append(e)
    return c


def category(v: int) -> int:
    return abs(int(v)).bit_length()


def huffman_length(rs: int):
    table = {0x00: 4.0, 0x01: 2.0, 0x02: 2.5, 0x03: 3.0, 0x04: 4.0, 0x11: 3.0, 0x12: 4.0, 0x21: 4.0, 0xF0: 10.0}
    if rs in table:
        return F(table[rs])
    return F(F(F(3.0) + F(rs >> 4) * F(0.5)) + F(rs & 15) * F(0.3))


def ac_rate(value: int, run: int):
    cat = category(value)
    return F(huffman_length((run << 4) | cat) + F(cat))


def trellis_quantize(dct, q, lam=None) -> np.ndarray:
    dct = np.asarray(dct, np.float32).reshape(64)
    q = np.asarray(q, np.float32).reshape(64)
    lam = F(1.0 if lam is None else lam)
    out = np.zeros(64, np.int16)
    out[0] = _i16(_round_half_away(float(F(dct[0] / q[0]))))
    cur = [(F(0.0), 0, 0, 0)]          # (cost, zero_run, parent, value)
    steps = [cur]
    for zz in range(1, 64):
        nat = ZIGZAG[zz]
        coef, qq = F(dct[nat]), F(q[nat])
        cands = candidates(F(coef / qq))
        nxt: list = []
        for pi, (pc, prun, _, _) in enumerate(cur):
            for c in cands:
                d = F(coef - F(F(c) * qq))
                dist = F(d * d)
                if c == 0:
                    nr = prun + 1
                    rate, nr = (F(10.0), 0) if nr >= 16 else (F(0.0), nr)
                else:
                    rate, nr = ac_rate(c, prun), 0
                cost = F(F(pc + rate) + F(lam * dist))
                for i, s in enumerate(nxt):
                    if s[3] == c and s[1] == nr:
                        if cost < s[0]:
                            nxt[i] = (cost, nr, pi, c)
                        break
                else:
                    nxt.append((cost, nr, pi, c))
        nxt.sort(key=lambda s: s[0])   # stable
        cur = nxt[:8]
        steps.append(cur)
    final = [F(s[0] + F(4.0)) if s[1] > 0 else s[0] for s in cur]
    best = min(range(len(cur)), key=lambda i: (final[i], i))
    for zz in range(63, 0, -1):
        s = steps[zz][best]
        out[ZIGZAG[zz]] = s[3]
        best = s[2]
    return out


def adaptive_lambda(quality: int):
    if quality >= 80:
        return F(F(0.5) + F(100 - quality) * F(0.025))
    if quality >= 50:
        return F(F(1.0) + F(80 - quality) * F(0.033))
    return F(F(2.0) + F(50 - quality) * F(0.04))


def constructed_blocks(seed: int = 1, n_random: int = 200):
    """Constructed (dct [n,64] f32, q [n,64] f32) covering the trellis's corners: all zero, exact .5
    quotients (equal-distortion ties), |dct/q| either side of 1.5, zero runs of 15/16/17/31/32 before a
    non-zero coefficient (ZRL states), 63 non-zeros, q = 1 with large magnitudes, and random blocks."""
    rng = np.random.default_rng(seed)
    d, qs = [], []

    def add(block, q):
        d.append(np.asarray(block, np.float32).reshape(64))
        qs.append(np.broadcast_to(np.asarray(q, np.float32), (64,)).copy())

    add(np.zeros(64), 16.0)
    for q in (2.0, 10.0, 16.0, 99.0):                      # exact .5 quotients
        k = rng.integers(-6, 6, 64)
        add((k + 0.5) * q, q)
        b = np.zeros(64); b[ZIGZAG[1:20]] = 0.5 * q
        add(b, q)
    for eps in (-1e-3, 0.0, 1e-3):                        # |fq| around 1.5
        for sgn in (1, -1):
            add(np.full(64, sgn * (1.5 + eps) * 16.0), 16.0)
    for run in (15, 16, 17, 31, 32):                       # zero runs before a non-zero
        b = np.zeros(64); b[0] = 300.0
        zz = 1
        while zz < 64:
            b[ZIGZAG[zz]] = rng.choice([-1, 1]) * rng.uniform(10.0, 60.0)
            zz += run + 1
        add(b, 8.0)
        b2 = np.zeros(64); b2[ZIGZAG[min(run + 1, 63)]] = 40.0
        add(b2, 4.0)
    add(rng.uniform(20.0, 200.0, 64) * rng.choice([-1, 1], 64), 4.0)   # 63 non-zeros
    add(rng.uniform(-2000.0, 2000.0, 64), 1.0)                         # q = 1, large magnitudes
    add(np.full(64, 8.0), 16.0)
    add(np.full(64, 10.0), 16.0)
    for _ in range(n_random):
        q = rng.integers(1, 256, 64).astype(np.float32) if rng.random() < 0.5 else \
            np.full(64, float(rng.integers(1, 100)), np.float32)
        scale = rng.choice([2.0, 20.0, 200.0])
        b = rng.laplace(0.0, scale, 64) * (rng.random(64) < rng.uniform(0.1, 1.0))
        if rng.random() < 0.3:
            b = np.round(b)
        add(b, q)
    return np.stack(d), np.stack(qs)


LAMBDAS = (0.1, 0.5, 1.0, 2.0, 10.0)
