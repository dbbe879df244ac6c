"""pixo's Nearest and Bilinear resizers (src/resize.rs:299-389) restated in numpy float32, independent of
oracle/resize.c, and the Lanczos3 work planner of csrc/resize.cu (`lanczos_bands` and the frame passes)
restated in Python, so that a test can say which path a case takes.

Every float operation is one numpy float32 operation, rounded once (numpy does not fuse a multiply and an
add).  `half` selects the rounding of f32::round: "away" (roundf, pixo's) or "even" (rintf, a fault the
exact-half inputs must tell apart)."""
from __future__ import annotations

import numpy as np

F = np.float32
SCRATCH = 256 << 20   # kResizeScratch: the intermediate's cap when PIXO_B200_RESIZE_SCRATCH is unset


def round_f32(v, half="away"):
    """f32::round (half away from zero), or round-half-even; v - trunc(v) is exact in float32."""
    v = np.asarray(v, F)
    if half == "even":
        return np.rint(v).astype(F)
    t = np.trunc(v)
    return (t + np.where(np.abs(v - t) >= F(0.5), np.sign(v), F(0))).astype(F)


def to_u8(v, half="away"):
    return np.clip(round_f32(v, half), 0, 255).astype(np.uint8)


def nearest_index(d, ratio, src, half="away"):
    """((d as f32 + 0.5) * ratio - 0.5).round().max(0.0).min((src - 1) as f32) as usize"""
    f = (np.asarray(d, F) + F(0.5)) * F(ratio) - F(0.5)
    return np.minimum(np.maximum(round_f32(f, half), F(0)), F(src - 1)).astype(np.int64)


def bilinear_taps(dst, ratio, src):
    """(i0, i1, frac) per destination index: floor(d * ratio) clamped to src - 1, as csrc/resize.cu does"""
    f = np.arange(dst, dtype=F) * F(ratio)
    i0 = np.minimum(np.floor(f).astype(np.int64), src - 1)
    return i0, np.minimum(i0 + 1, src - 1), (f - i0.astype(F)).astype(F)


def nearest(img, sw, sh, dw, dh, bpp, half="away"):
    a = np.asarray(img, np.uint8).reshape(sh, sw, bpp)
    ys = nearest_index(np.arange(dh), F(sh) / F(dh), sh, half)
    xs = nearest_index(np.arange(dw), F(sw) / F(dw), sw, half)
    return a[ys][:, xs].reshape(-1)


def bilinear(img, sw, sh, dw, dh, bpp, half="away"):
    a = np.asarray(img, np.uint8).reshape(sh, sw, bpp).astype(F)
    xr = F(sw - 1) / F(dw - 1) if dw > 1 else F(0)
    yr = F(sh - 1) / F(dh - 1) if dh > 1 else F(0)
    x0, x1, xf = bilinear_taps(dw, xr, sw)
    y0, y1, yf = bilinear_taps(dh, yr, sh)
    xf, xf1 = xf[None, :, None], (F(1) - xf)[None, :, None]
    yf, yf1 = yf[:, None, None], (F(1) - yf)[:, None, None]
    top = a[y0][:, x0] * xf1 + a[y0][:, x1] * xf
    bot = a[y1][:, x0] * xf1 + a[y1][:, x1] * xf
    return to_u8(top * yf1 + bot * yf, half).reshape(-1)


def resize(img, sw, sh, dw, dh, bpp, alg, half="away"):
    """Nearest (alg 0) or Bilinear (alg 1)."""
    return (nearest, bilinear)[alg](img, sw, sh, dw, dh, bpp, half)


# ---- Lanczos3's work plan -----------------------------------------------------------------------------
def lanczos_bands(start, count, sh, dw, dh, bpp, cap):
    """csrc/resize.cu's lanczos_bands: [(y0, y1, rs, re, x0, cw)], destination rows y0..y1-1 and columns
    x0..x0+cw-1 from source rows rs..re-1 of the intermediate.  start / count: the vertical axis's tables."""
    start, count = [int(s) for s in start], [int(c) for c in count]
    row = dw * bpp
    if sh * row <= cap:
        return [(0, dh, 0, sh, 0, dw)]
    bands, y0 = [], 0
    while y0 < dh:
        rs, re = (start[y0], start[y0] + count[y0]) if count[y0] else (1 << 32, 0)
        y1 = y0 + 1
        rows1 = max(re - rs, 0)
        if rows1 * row > cap:   # one destination row's taps alone: its columns in chunks
            cw = max(1, cap // (rows1 * bpp))
            bands += [(y0, y1, rs, re, x0, min(cw, dw - x0)) for x0 in range(0, dw, cw)]
            y0 = y1
            continue
        while y1 < dh:
            if count[y1]:
                nrs, nre = min(rs, start[y1]), max(re, start[y1] + count[y1])
                if (nre - nrs) * row > cap:
                    break
                rs, re = nrs, nre
            y1 += 1
        if re <= rs:
            rs = re = 0
        bands.append((y0, y1, rs, re, 0, dw))
        y0 = y1
    return bands


def frames_per_pass(bands, n, bpp, cap):
    """Frames that go through the kernels together: as many whole intermediates as the cap holds, only when
    one band covers the frame."""
    if len(bands) != 1:
        return 1
    most = max(1, max((re - rs) * cw * bpp for _, _, rs, re, _, cw in bands))
    return min(n, 65535, max(1, cap // most))


def lanczos_launches(bands, n, per_pass):
    """Kernel launches of one call: per pass, each band's horizontal pass (if it reads rows) and vertical pass."""
    passes = -(-n // per_pass)
    return passes * sum(1 + (re > rs) for _, _, rs, re, _, _ in bands)
