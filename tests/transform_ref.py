"""A plain restatement of the JPEG transform stage (k_jpeg_420, k_jpeg_444, k_jpeg_gray in csrc/jpeg_transform.cu),
written from pixo's semantics, not from the kernels:
  * rgb_to_ycbcr              src/color.rs:60-77, vectorised in integers;
  * dct_2d / aan_dct_1d       src/jpeg/dct.rs:591-700, in numpy float32 op for op (numpy rounds once per float32
                              op and never contracts);
  * quantize_block            src/jpeg/quantize.rs:99-105: (dct / q).round(), the quotient in float32, the
                              half-away rounding done exactly in float64;
  * the 4:2:0 chroma block    src/jpeg/mod.rs:1608-1656: quad sums in f32, then * 0.25 - 128.
It also restates the kernels' own quantiser sequence (DESIGN.md section 3) with every directed rounding emulated
exactly through fractions.Fraction, the single faults of that sequence the tests are built to catch, and the unit
walk of the persistent kernels' advance()."""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

F32 = np.float32
A1, A2, A3, A4, A5 = F32(0.70710678118654752440), F32(0.5411961), F32(0.70710678118654752440), F32(1.3065629), \
    F32(0.38268343)
S = np.array([0.3535534, 0.2548978, 0.2705981, 0.3006724, 0.3535534, 0.4499881, 0.6532815, 1.2814578], F32)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


# ---- colour -------------------------------------------------------------------------------------------
def rgb_to_ycbcr(rgb):
    """[..., 3] integers 0..255 -> [..., 3] uint8 (Y, Cb, Cr), color.rs:60-77"""
    a = np.asarray(rgb).astype(np.int32)
    r, g, b = a[..., 0], a[..., 1], a[..., 2]
    y = (77 * r + 150 * g + 29 * b + 128) >> 8
    cb = ((-43 * r - 85 * g + 128 * b + 128) >> 8) + 128
    cr = ((128 * r - 107 * g - 21 * b + 128) >> 8) + 128
    return np.clip(np.stack([y, cb, cr], -1), 0, 255).astype(np.uint8)


def all_colours_ycbcr():
    """(Y, Cb, Cr) of colour c = r << 16 | g << 8 | b for all 2^24 colours: [2^24, 3] uint8"""
    c = np.arange(1 << 24, dtype=np.int32)
    return rgb_to_ycbcr(np.stack([c >> 16, (c >> 8) & 255, c & 255], -1))


# ---- DCT ----------------------------------------------------------------------------------------------
def aan_1d(d):
    """aan_dct_1d (dct.rs:648-700) on a list of eight float32 arrays, before the S[k] post-scale"""
    tmp0, tmp7 = d[0] + d[7], d[0] - d[7]
    tmp1, tmp6 = d[1] + d[6], d[1] - d[6]
    tmp2, tmp5 = d[2] + d[5], d[2] - d[5]
    tmp3, tmp4 = d[3] + d[4], d[3] - d[4]
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    o = [None] * 8
    o[0], o[4] = tmp10 + tmp11, tmp10 - tmp11
    z1 = (tmp12 + tmp13) * A1
    o[2], o[6] = tmp13 + z1, tmp13 - z1
    u10, u11, u12 = tmp4 + tmp5, tmp5 + tmp6, tmp6 + tmp7
    z5 = (u10 - u12) * A5
    z2 = u10 * A2 + z5
    z4 = u12 * A4 + z5
    z3 = u11 * A3
    z11, z13 = tmp7 + z3, tmp7 - z3
    o[5], o[3] = z13 + z2, z13 - z2
    o[1], o[7] = z11 + z4, z11 - z4
    return o


def dct_2d(blocks):
    """dct_2d (dct.rs:614-646): [..., 64] float32 (natural order) -> [..., 64] float32; rows, then columns"""
    b = np.asarray(blocks, F32).reshape(-1, 8, 8)
    rows = aan_1d([b[:, :, k] for k in range(8)])
    t = np.stack([rows[k] * S[k] for k in range(8)], -1)          # t[:, r, c]
    cols = aan_1d([t[:, k, :] for k in range(8)])
    out = np.stack([cols[k] * S[k] for k in range(8)], 1)          # out[:, r, c]
    return out.reshape(np.asarray(blocks).shape[:-1] + (64,))


def round_half_away(q):
    """f32 quotients -> int16, f32::round then `as i16` (saturating); exact in float64"""
    q = np.asarray(q, np.float64)
    return np.clip(np.copysign(np.floor(np.abs(q) + 0.5), q), -32768, 32767).astype(np.int16)


def quantize(dct, q):
    """quantize_block (quantize.rs:99-105): [..., 64] float32 DCT, 64 divisors -> int16"""
    return round_half_away(np.asarray(dct, F32) / np.asarray(q, F32))


def gray_block(v):
    """pixel values (any shape ending in 64) -> the f32 block extract_block hands the DCT"""
    return np.asarray(v, F32) - F32(128)


def chroma_420_block(quad_sums):
    """[..., 64] quad sums of one chroma component (0..1020) -> s * 0.25 - 128 in f32 (mod.rs:1642-1653)"""
    return np.asarray(quad_sums, F32) * F32(0.25) - F32(128)


def flat_dc(v):
    """DC of a flat block of value v - 128 (v may be a quarter-integer: the 4:2:0 quad average) quantised by 1"""
    b = np.repeat(np.asarray(v, F32).reshape(-1, 1) - F32(128), 64, axis=1)
    return quantize(dct_2d(b), np.ones(64, F32))[:, 0]


# ---- the kernels' quantiser, exactly --------------------------------------------------------------------
def _f32_neighbours(x: Fraction):
    """(lo, hi): the largest float32 <= x and the smallest >= x, as Fractions"""
    c = np.float32(float(x))
    while Fraction(float(c)) > x:
        c = np.nextafter(c, F32(-np.inf))
    lo = c
    while Fraction(float(c)) < x:
        c = np.nextafter(c, F32(np.inf))
    return Fraction(float(lo)), Fraction(float(c)), lo


def f32_round(x: Fraction, mode: str) -> Fraction:
    """x rounded to float32: 'rn' (nearest, ties to even), 'rz' (toward zero), 'rd' (toward -inf)"""
    lo, hi, lo32 = _f32_neighbours(x)
    if lo == hi:
        return lo
    if mode == "rd":
        return lo
    if mode == "rz":
        return lo if x > 0 else hi
    dl, dh = x - lo, hi - x
    if dl != dh:
        return lo if dl < dh else hi
    return lo if int(np.asarray(lo32).view(np.uint32)) % 2 == 0 else hi


def rn(x):
    return f32_round(Fraction(x), "rn")


def pixo_quant(x, d) -> int:
    """pixo on one coefficient: RN(x / d), then round half away from zero"""
    q = rn(Fraction(float(x)) / d)
    a = int(abs(q) + Fraction(1, 2))
    return -a if q < 0 else a


# Single faults of the kernel's sequence, each a way the kernel could be subtly wrong:
#   rz_to_rn     w = RN(q + 0.5) instead of RZ (add2_rz -> add2)
#   no_residual  q = q0 = RN(x * RN(1/d)): the fma residual correction dropped
#   half_even    the rounding done by __float2int_rn (half to even)
#   half_up_neg  negative quotients rounded half toward +inf: floor(q + 0.5)
#   no_fold      4:2:0 chroma: r = RN(1/d), not RN(1/d) / 4 (the x0.25 fold dropped from the reciprocal)
MUTANTS = ("rz_to_rn", "no_residual", "half_even", "half_up_neg", "no_fold")
MAGIC = Fraction(12582912)   # 1.5 * 2^23


def kernel_parts(x, d, sc=1, mut=()):
    """The kernel's division for a (scaled) coefficient x and divisor d: (q0, q), Fractions holding float32 values.
    sc: the chroma fold (4 for 4:2:0 chroma, whose block reaches the DCT as 4x pixo's)."""
    xf = Fraction(float(x)) * sc                       # the kernel's block is sc x pixo's: exact
    r0 = rn(Fraction(1, d))
    r = r0 if "no_fold" in mut else r0 / sc          # sc is a power of two: exact
    q0 = rn(xf * r)
    if "no_residual" in mut:
        return q0, q0
    e = rn(q0 * (-d * sc) + xf)                        # fma(q0, -d, x)
    return q0, rn(e * r + q0)                          # fma(e, r, q0)


def kernel_quant(x, d, sc=1, mut=()) -> int:
    """The kernel's quantiser (dct_cols_quant_store_x2) on one coefficient: the int16 it stores"""
    _, q = kernel_parts(x, d, sc, mut)
    if "half_even" in mut:
        return round(q)                                 # Fraction.__round__ is half to even
    neg = q < 0
    if neg and "half_up_neg" in mut:
        return math.floor(q + Fraction(1, 2))
    w = f32_round(q + Fraction(1, 2), "rn" if "rz_to_rn" in mut else "rz")
    tt = f32_round(w * (-1 if neg else 1) + MAGIC, "rd")   # fma.rm(w, copysign(1, q), 1.5 * 2^23)
    m = int(tt - MAGIC)
    return ~m if neg else m


# ---- the persistent kernels' unit walk ------------------------------------------------------------------
def walk(units_x, mcus_y, n, stride):
    """advance() of k_jpeg_420 / k_jpeg_444 for every warp of a grid of `stride` warps.
    Returns (units, branches): units[u] = (img, my, ux) of unit u as the walk reached it (all units are reached
    exactly once), and the set of branch tuples the steps took: (ux carried, my wrapped, ux landed exactly on
    units_x, my landed exactly on mcus_y)."""
    per_img = units_x * mcus_y
    nunits = per_img * n
    d_ux, d_t = stride % units_x, stride // units_x
    d_my, d_img = d_t % mcus_y, d_t // mcus_y
    u0 = np.arange(min(stride, nunits), dtype=np.int64)
    img, rem = u0 // per_img, u0 % per_img
    my, ux = rem // units_x, rem % units_x
    u = u0.copy()
    units = np.full((nunits, 3), -1, np.int64)
    branches = set()
    live = u < nunits
    while live.any():
        units[u[live]] = np.stack([img[live], my[live], ux[live]], -1)
        ux = ux + d_ux
        cx, ex = ux >= units_x, ux == units_x
        ux = np.where(cx, ux - units_x, ux)
        my = my + cx + d_my
        cm, em = my >= mcus_y, my == mcus_y
        my = np.where(cm, my - mcus_y, my)
        img = img + cm + d_img
        u = u + stride
        step = live & (u < nunits)
        for t in set(zip(cx[step].tolist(), cm[step].tolist(), ex[step].tolist(), em[step].tolist())):
            branches.add(t)
        live = step
    return units, branches
