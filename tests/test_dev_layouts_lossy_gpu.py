"""The device-pointer entry points of the lossy and size-reducing paths at the layouts their callers pass:
pixo_b200_png_reduce_filter_dev, pixo_b200_png_quantize_filter_dev, PIXO_B200_COEF_TRELLIS through
pixo_b200_jpeg_coefficients_dev, and pixo_b200_jpeg_trellis_quantize_dev.  Frames sit at offsets that are
not 4- or 16-byte aligned and at strides that make a batch alternate between the kernels' word and byte
loads; batches mix frames that reduce or quantise differently, so the per-run filter launches and the
reduced-row offsets are exercised; batches cross the 65 535-frames-per-launch split.

The harness is test_dev_layouts_gpu.py's.  Around PNG frames lies a poison that flips a decision if it
is read (a non-gray, translucent colour no frame holds, so a stray read adds a palette entry, a histogram
colour or a non-gray pixel); around JPEG pixels lie 0/255 stripes; every output region sits inside guard
values that must survive the call.  Every frame checked is compared byte for byte with the oracle and
every Adler-32 with zlib."""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle import jpeg_trellis as jt
from oracle import png_quantize as pq
from oracle import png_reduce as pr
from quantize_inputs import make_quantize_input
from reduce_inputs import make_reduce_input
import trellis_ref as tr
from test_dev_layouts_gpu import (GUARD8, GUARD16, GUARD32, OPTIMIZE_ALPHA, Buf, assert_guard, guarded, placed,
                                  run, stripes)

pytestmark = pytest.mark.gpu

RCT, RPAL = 0x200, 0x400
QAUTO, QFORCE, DITHER = 0x800, 0x1000, 0x2000
COEF_ZIGZAG, COEF_TRELLIS = 1, 2
ZZ = np.array(tr.ZIGZAG)


@pytest.fixture(autouse=True)
def _no_host_fallback(gpu_ctx):
    """No frame of this file is finished by host code."""
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was finished by the host"


def flip_poison(n):
    """Seven distinct bytes, none 255, repeated: any 3 or 4 of them read as a pixel are a non-gray,
    translucent colour no test frame holds."""
    return np.resize(np.array([1, 250, 3, 7, 128, 60, 200], np.uint8), n)


# (input offset, input stride padding, output offset, output stride padding).  With frames whose size
# is a multiple of 16, padding 12 alternates 16-byte and 4-byte aligned frames, 13 and 4099 walk every
# phase (byte loads on most frames), 4 keeps every frame word- but not 16-byte aligned.  (0, 13) puts a
# 16-byte aligned frame 0 ahead of frames that only byte loads can read, so a kernel that chose its loads
# from the batch's first frame instead of each frame's own base would issue misaligned loads.
PNG_LAYOUTS = [(0, 0, 0, 0), (4, 4, 5, 3), (0, 12, 0, 0), (0, 13, 5, 3), (1, 13, 5, 0), (7, 4099, 0, 3)]


def png_dev(ctx, fn, frames, w, h, ct, word, layout, *extra):
    """One reduce / quantise _dev call on `frames` laid out as `layout`: checks the guards around every
    frame's output and Adler-32 and returns (descriptions, filtered streams, Adler-32s)."""
    from pixo_b200 import png
    in_off, in_pad, out_off, out_pad = layout
    n, bpp = len(frames), ct + 1
    in_stride = w * h * bpp + in_pad
    out_stride = h * (w * bpp + 1) + out_pad
    src = placed(frames, in_off, in_stride, flip_poison)
    o0 = 64 + out_off
    dst = guarded((n - 1) * out_stride + h * (w * bpp + 1), np.uint8, GUARD8, base=o0)
    ad = guarded(n, np.int32, GUARD32, base=4, tail=4)
    infos = (png._Reduced * n)()
    args = (word,) + extra + (infos, dst.ptr(o0), out_stride, ad.ptr(4))
    run(ctx, fn, src.ptr(in_off), in_stride, n, w, h, ct, *args)
    reds = [png.ReducedImage._from_c(infos[i]) for i in range(n)]
    out, ads = dst.get(), ad.get()
    lens = [h * (r.row_bytes + 1) for r in reds]
    assert_guard(out, [(o0 + i * out_stride, lens[i]) for i in range(n)], GUARD8, f"filtered output {layout}")
    assert_guard(ads, [(4, n)], GUARD32, f"d_adler {layout}")
    return reds, [out[o0 + i * out_stride:][:lens[i]] for i in range(n)], ads[4:4 + n].view(np.uint32)


def reduce_ref(po, img, w, h, ct, word, red=None):
    """pixo: maybe_reduce_color_type -> maybe_optimize_alpha -> apply_filters_with_row_bytes"""
    red = red or pr.reduce(img, w, h, ct, bool(word & RCT), bool(word & RPAL))
    f = po.apply_filters(pr.filter_input(red, bool(word & OPTIMIZE_ALPHA)), w, h, red.bytes_per_pixel, word & 0xFF,
                         row_bytes=red.row_bytes)
    return red, f


def same_lossless(got, want, f, wf, ad, what):
    assert (got.color_type_byte, got.bit_depth, got.bytes_per_pixel, got.row_bytes, int(got.effective_color_type)) == \
        (want.color_type_byte, want.bit_depth, want.bytes_per_pixel, want.row_bytes, want.effective_color_type), what
    if want.palette is None:
        assert got.palette is None, what
    else:
        assert np.array_equal(got.palette, want.palette) and got.trns == want.trns, what
    assert np.array_equal(f, wf), (what, np.flatnonzero(f != wf)[:5])
    assert int(ad) == zlib.adler32(wf.tobytes()), what


# ---- PNG reduce ---------------------------------------------------------------------------------------
# (make_reduce_input kind, colours): ordered so that consecutive frames differ in row_bytes (1- vs 4- vs
# 2-bit), bytes_per_pixel (8-bit palette, RGB, GrayAlpha) or whether they are reduced at all
REDUCE_BATCHES = {
    (3, RCT | RPAL): [("pal", 2), ("pal", 16), ("pal", 4), ("palo", 3), ("pal", 200), ("opaque", 0),
                      ("grayalpha", 0), ("noise", 0), ("graypal", 5), ("pal", 2)],
    (3, RCT): [("graypal", 2), ("graypal", 16), ("graypal", 4), ("graypal", 200), ("opaque", 0), ("grayalpha", 0),
               ("noise", 0), ("graypal", 3)],
    (2, RCT | RPAL): [("pal", 2), ("pal", 16), ("pal", 4), ("pal", 200), ("noise", 0), ("pal", 5)],
    (2, RCT): [("graypal", 2), ("graypal", 16), ("graypal", 4), ("graypal", 256), ("noise", 0), ("graypal", 3)],
}
# w = 2: 1-, 2- and 4-bit rows all 1 byte (one run); w = 5: 1, 2 and 3 bytes.  Areas <= 4096 take pixo's
# Sub rule; 300 x 20 is sticky AdaptiveFast; 131 x 70 spans 16-row bands; 2, 5, 131 and 300 pad 1-bit rows.
REDUCE_GEOMETRIES = [(2, 200), (5, 150), (37, 31), (131, 70), (300, 20)]


@pytest.mark.parametrize("ct,flags", list(REDUCE_BATCHES), ids=["rgba-pal", "rgba-ct", "rgb-pal", "rgb-ct"])
@pytest.mark.parametrize("w,h", REDUCE_GEOMETRIES)
def test_reduce_filter_dev_mixed_batches(po, gpu_ctx, w, h, ct, flags):
    """Frames that become 1/2/4/8-bit palettes or gray, GrayAlpha, RGB or stay unchanged, side by side,
    under all nine strategies (OPTIMIZE_ALPHA on every other one) at every layout."""
    from pixo_b200 import _lib
    fn = _lib.load().pixo_b200_png_reduce_filter_dev
    frames = [make_reduce_input(k, w, h, ct + 1, 100 * i + w, n) for i, (k, n) in enumerate(REDUCE_BATCHES[ct, flags])]
    reds = [pr.reduce(f, w, h, ct, True, bool(flags & RPAL)) for f in frames]
    outcomes = {(r.color_type_byte, r.bit_depth) for r in reds}
    if flags & RPAL:
        assert {(3, 1), (3, 2), (3, 4), (3, 8)} <= outcomes, outcomes
    else:
        assert {(0, 1), (0, 2), (0, 4), (0, 8)} <= outcomes, outcomes
    if ct == 3:
        assert {(2, 8), (4, 8), (6, 8)} <= outcomes, outcomes
    for s in range(9):
        word = s | flags | (OPTIMIZE_ALPHA if s % 2 else 0)
        refs = [reduce_ref(po, f, w, h, ct, word, r) for f, r in zip(frames, reds)]
        if s == 7 and (w, h) == (300, 20):     # sticky AdaptiveFast: each frame keeps its own row-0 winner
            assert len({int(f[0]) for _, f in refs}) >= 2
        for layout in PNG_LAYOUTS:
            got, outs, ads = png_dev(gpu_ctx, fn, frames, w, h, ct, word, layout)
            for i, ((want, wf), g, f, a) in enumerate(zip(refs, got, outs, ads)):
                same_lossless(g, want, f, wf, a, (layout, hex(word), i))


def test_reduce_filter_dev_rows_beyond_the_staging_segment(po, gpu_ctx):
    """1- and 2-bit rows of 37 500 and 75 000 bytes (over the filter's 32 KiB segment) next to an
    unchanged RGB frame, every strategy."""
    from pixo_b200 import _lib
    fn = _lib.load().pixo_b200_png_reduce_filter_dev
    w, h, ct = 300001, 3, 2
    frames = [make_reduce_input("pal", w, h, 3, 1, 2), make_reduce_input("palblk", w, h, 3, 2, 4),
              make_reduce_input("noise", w, h, 3, 3)]
    reds = [pr.reduce(f, w, h, ct, True, True) for f in frames]
    assert [(r.bit_depth, r.row_bytes) for r in reds] == [(1, 37501), (2, 75001), (8, 3 * w)]
    for s in range(9):
        word = s | RCT | RPAL
        refs = [reduce_ref(po, f, w, h, ct, word, r) for f, r in zip(frames, reds)]
        got, outs, ads = png_dev(gpu_ctx, fn, frames, w, h, ct, word, PNG_LAYOUTS[(s % 4) + 1])
        for i, ((want, wf), g, f, a) in enumerate(zip(refs, got, outs, ads)):
            same_lossless(g, want, f, wf, a, (s, i))


def tiny_palette_frames(n, w, h, seed):
    """n frames of w x h RGBA pixels, each with 1..w*h colours drawn from its own random colours."""
    rng = np.random.default_rng(seed)
    npx = w * h
    k = rng.integers(1, npx + 1, n)
    cols = rng.integers(0, 256, (n, npx, 4), dtype=np.uint8)
    cols[rng.random((n, npx)) < 0.5, 3] = 255
    idx = np.arange(npx)[None, :] % k[:, None]
    idx = np.take_along_axis(idx, rng.permuted(np.tile(np.arange(npx), (n, 1)), axis=1), axis=1)
    return np.take_along_axis(cols, idx[..., None], axis=1).reshape(n, -1)


def sampled(n):
    return sorted({0, 1, 65533, 65534, 65535, 65536, n - 1} | set(range(7, n, 331)))


def test_reduce_filter_dev_across_the_launch_split(po, gpu_ctx):
    """65 537 frames of 3 x 2 pixels with 1 to 6 colours (1-, 2- and 4-bit palettes: row_bytes 1 and 2)
    at an odd stride from a 16-byte aligned frame 0: the analyse, index and pack launches split at
    65 535 frames, and each frame picks word or byte loads from its own base."""
    from pixo_b200 import _lib, png
    n, w, h, ct = 65537, 3, 2, 3
    frames = tiny_palette_frames(n, w, h, 4)
    raw = w * h * 4
    word = 4 | RCT | RPAL | OPTIMIZE_ALPHA
    stride = raw + 1                                          # frame i at 25 i
    host = flip_poison(n * stride + 64)
    for i in range(n):
        host[i * stride:i * stride + raw] = frames[i]
    src = Buf(host)
    out_stride = h * (w * 4 + 1)
    dst = guarded(n * out_stride, np.uint8, GUARD8)
    ad = guarded(n, np.int32, GUARD32, base=4, tail=4)
    infos = (png._Reduced * n)()
    run(gpu_ctx, _lib.load().pixo_b200_png_reduce_filter_dev, src.ptr(), stride, n, w, h, ct, word, infos,
        dst.ptr(64), out_stride, ad.ptr(4))
    out, ads = dst.get(), ad.get()
    rbs = np.array([infos[i].row_bytes for i in range(n)])
    assert set(rbs.tolist()) == {1, 2}
    assert_guard(out, [(64 + i * out_stride, h * (int(rbs[i]) + 1)) for i in range(n)], GUARD8, "filtered output")
    assert_guard(ads, [(4, n)], GUARD32, "d_adler")
    for i in sampled(n):
        want, wf = reduce_ref(po, frames[i], w, h, ct, word)
        f = out[64 + i * out_stride:][:h * (int(rbs[i]) + 1)]
        same_lossless(png.ReducedImage._from_c(infos[i]), want, f, wf, ads[4 + i], i)


def test_reduce_filter_dev_rejects_overlapping_frames(gpu_ctx):
    """With more than one frame, an in_stride below a frame or an out_stride below a filtered frame is
    refused before any launch."""
    import torch
    from pixo_b200 import _lib, png
    lib = _lib.load()
    w, h, ct = 20, 6, 3
    raw, need = w * h * 4, h * (w * 4 + 1)
    frames = [make_reduce_input("pal", w, h, 4, s, 3) for s in (1, 2)]
    src = placed(frames, 0, raw, flip_poison)
    dst = guarded(2 * need, np.uint8, GUARD8)
    infos = (png._Reduced * 2)()
    torch.cuda.synchronize()
    l0 = gpu_ctx.launch_count
    for in_stride, out_stride, code in ((raw - 1, need, _lib.ERR_INVALID_DATA_LENGTH),
                                        (raw, need - 1, _lib.ERR_OUTPUT_TOO_SMALL)):
        rc = lib.pixo_b200_png_reduce_filter_dev(gpu_ctx.handle, src.ptr(), in_stride, 2, w, h, ct, 6 | RCT | RPAL,
                                                 infos, dst.ptr(64), out_stride, None)
        assert rc == code, (in_stride, out_stride, rc)
    assert gpu_ctx.launch_count == l0
    gpu_ctx.sync()
    assert_guard(dst.get(), [], GUARD8, "output of a refused call")


# ---- PNG quantise -------------------------------------------------------------------------------------
def quantize_ref(po, img, w, h, ct, word, max_colors, palette=None):
    """(quantised?, description, filtered stream) as encode_into hands them to DEFLATE"""
    mode = "force" if word & QFORCE else "auto"
    if not pq.should_quantize(img, ct, mode, min(max_colors, 256)):
        return (False,) + reduce_ref(po, img, w, h, ct, word & ~(QAUTO | QFORCE | DITHER))
    pal, idx = pq.quantize(img, w, h, ct, max_colors, bool(word & DITHER), palette)
    return True, pal, po.apply_filters(idx, w, h, 1, pq.indexed_strategy(word & 0xFF))


def same_quantized(got, want, f, ad, what):
    quantised, wp, wf = want
    if quantised:
        assert (got.color_type_byte, got.bit_depth, got.bytes_per_pixel, int(got.effective_color_type)) == (3, 8, 1, 2), what
        assert np.array_equal(got.palette, wp), what
        assert got.trns == pq.trimmed_trns(wp), what
        assert np.array_equal(f, wf), (what, np.flatnonzero(f != wf)[:5])
        assert int(ad) == zlib.adler32(wf.tobytes()), what
    else:
        same_lossless(got, wp, f, wf, ad, what)


def quantize_frames(w, h, ct, m, seed):
    """(frame, caller palette or None): median cut and LUT (translucent gradient, noise, 3m colours),
    the early out under Force (m opaque colours), frames Auto leaves lossless, a caller palette"""
    ch = ct + 1
    pal = make_quantize_input("pal", 9, 1, 4, seed, 9).reshape(-1, 4)
    return [(make_quantize_input("grad", w, h, ch, seed), None),
            (make_quantize_input("palo", w, h, ch, seed + 1, m), None),
            (make_quantize_input("noise", w, h, ch, seed + 2), None),
            (make_quantize_input("pal", w, h, ch, seed + 3, 3 * m), None),
            (make_quantize_input("grad", w, h, ch, seed + 4), pal),
            (make_quantize_input("palblk", w, h, ch, seed + 5, 20), None)]


QUANT_CASES = [(mode, dither, m) for mode in (QAUTO, QFORCE) for dither in (0, DITHER) for m in (2, 16, 256)]
# dither heights around the 32-row groups
QUANT_GEOMETRIES = [(45, 31), (33, 32), (29, 33), (21, 65)]


@pytest.mark.parametrize("k", range(len(QUANT_CASES)),
                         ids=[f"{'auto' if a == QAUTO else 'force'}-{'dither' if d else 'plain'}-{m}"
                              for a, d, m in QUANT_CASES])
def test_quantize_filter_dev_mixed_batches(po, gpu_ctx, k):
    """Auto and Force, dithering on and off, 2 / 16 / 256 colours: frames through median cut and the
    LUT, the early out, the lossless path and a caller palette, side by side, at every layout."""
    from pixo_b200 import _lib
    fn = _lib.load().pixo_b200_png_quantize_filter_dev
    mode, dither, m = QUANT_CASES[k]
    w, h = QUANT_GEOMETRIES[k % len(QUANT_GEOMETRIES)]
    ct = 2 if k % 3 == 2 else 3
    word = (k % 9) | mode | dither | (RCT | RPAL | OPTIMIZE_ALPHA if k % 2 else 0)
    fp = quantize_frames(w, h, ct, m, 10 * k)
    frames = [f for f, _ in fp]
    pals = np.zeros((len(fp), 256, 4), np.uint8)
    lens = np.zeros(len(fp), np.uint32)
    for i, (_, p) in enumerate(fp):
        if p is not None:
            pals[i, :len(p)], lens[i] = p, len(p)
    refs = [quantize_ref(po, f, w, h, ct, word, m, p) for f, p in fp]
    if mode == QAUTO:                                 # m opaque colours stay lossless, 3m colours quantise
        assert not refs[1][0] and refs[3][0] and (m == 256 or not refs[2][0])
    else:
        assert all(r[0] for r in refs)
    for layout in PNG_LAYOUTS:
        got, outs, ads = png_dev(gpu_ctx, fn, frames, w, h, ct, word, layout, m, pals.ctypes.data, lens.ctypes.data)
        for i, (r, g, f, a) in enumerate(zip(refs, got, outs, ads)):
            same_quantized(g, r, f, a, (layout, hex(word), m, i))


@pytest.mark.parametrize("dither", [0, DITHER])
def test_quantize_filter_dev_beyond_65535_frames(po, gpu_ctx, dither):
    """65 537 quantised frames of 3 x 2 pixels in one Force call with 2 colours: frames of 1 or 2 colours
    take the early out, the others median cut, k-means and the LUT (dithered when asked).  The
    quantised frames are processed in passes, so no launch exceeds 65 535 frames.  Frame 0 is 16-byte
    aligned and the stride is odd, so k_quant_map's 16-byte, word and byte loads all run."""
    from pixo_b200 import _lib, png
    n, w, h, ct, m = 65537, 3, 2, 3, 2
    frames = tiny_palette_frames(n, w, h, 8 + dither)
    raw = w * h * 4
    stride = raw + 5
    host = flip_poison(n * stride + 64)
    for i in range(n):
        host[i * stride:i * stride + raw] = frames[i]
    src = Buf(host)
    word = 2 | QFORCE | dither
    out_stride = h * (w * 4 + 1)
    dst = guarded(n * out_stride, np.uint8, GUARD8)
    ad = guarded(n, np.int32, GUARD32, base=4, tail=4)
    infos = (png._Reduced * n)()
    run(gpu_ctx, _lib.load().pixo_b200_png_quantize_filter_dev, src.ptr(), stride, n, w, h, ct, word, m, None, None,
        infos, dst.ptr(64), out_stride, ad.ptr(4))
    out, ads = dst.get(), ad.get()
    assert all(infos[i].row_bytes == w and infos[i].color_type_byte == 3 for i in range(n))
    assert_guard(out, [(64 + i * out_stride, h * (w + 1)) for i in range(n)], GUARD8, "filtered output")
    assert_guard(ads, [(4, n)], GUARD32, "d_adler")
    kinds = set()
    for i in sampled(n):
        r = quantize_ref(po, frames[i], w, h, ct, word, m)
        kinds.add(len(np.unique(frames[i].view(np.uint32))) <= m)
        same_quantized(png.ReducedImage._from_c(infos[i]), r, out[64 + i * out_stride:][:h * (w + 1)], ads[4 + i], i)
    assert kinds == {True, False}


# ---- JPEG trellis -------------------------------------------------------------------------------------
def trellis_frames(w, h, ct, n, seed):
    rng = np.random.default_rng(seed)
    ch = 1 if ct == 0 else 3
    y, x = np.mgrid[0:h, 0:w]
    smooth = np.stack([(x * 3 + y * 5 + 40 * c) % 256 for c in range(ch)], -1).astype(np.uint8)
    out = [rng.integers(0, 256, (h, w, ch), dtype=np.uint8), smooth,
           np.where(((x // 8 + y // 8) % 2 == 0)[..., None], rng.integers(0, 256, ch, dtype=np.uint8), 17)]
    return [np.ascontiguousarray(out[i % 3], np.uint8).reshape(-1) for i in range(n)]


def coef_dev(ctx, frames, w, h, ct, ss, q, px_off, px_pad, c_pad, flags):
    """COEF_TRELLIS through jpeg_coefficients_dev at the given layout; checks the guards around every
    frame's coefficient slots and returns each frame's (y, cb, cr) in natural order."""
    from pixo_b200 import _lib, jpeg
    n, flen = len(frames), frames[0].size
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    pixel_stride = flen + px_pad
    src = placed(frames, px_off, pixel_stride, stripes)
    y_stride, c_stride = ny * 64 + c_pad, max(nc, 1) * 64 + c_pad
    dy = guarded((n - 1) * y_stride + ny * 64, np.int16, GUARD16)
    dcb = guarded((n - 1) * c_stride + nc * 64, np.int16, GUARD16)
    dcr = guarded((n - 1) * c_stride + nc * 64, np.int16, GUARD16)
    _, _, lq, cq = jpeg.quant_tables(q)
    run(ctx, _lib.load().pixo_b200_jpeg_coefficients_dev, src.ptr(px_off), pixel_stride, n, w, h, ct, ss,
        lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p), dy.ptr(64), y_stride, dcb.ptr(64), dcr.ptr(64),
        c_stride, COEF_TRELLIS | flags, None)
    layout = (px_off, px_pad, c_pad, flags)
    y, cb, cr = dy.get(), dcb.get(), dcr.get()
    assert_guard(y, [(64 + i * y_stride, ny * 64) for i in range(n)], GUARD16, f"Y {layout}")
    for a, name in ((cb, "Cb"), (cr, "Cr")):
        assert_guard(a, [(64 + i * c_stride, nc * 64) for i in range(n)], GUARD16, f"{name} {layout}")
    inv = np.argsort(ZZ)
    got = []
    for i in range(n):
        arrs = [y[64 + i * y_stride:][:ny * 64], cb[64 + i * c_stride:][:nc * 64], cr[64 + i * c_stride:][:nc * 64]]
        arrs = [a.reshape(-1, 64) for a in arrs]
        if flags & COEF_ZIGZAG:
            arrs = [a[:, inv] for a in arrs]
        got.append(arrs)
    return got


def same_coefficients(got, want, what):
    for g, w_, name in zip(got, want, ("Y", "Cb", "Cr")):
        assert g.shape == w_.shape, (what, name)
        bad = np.flatnonzero((g != w_).any(1))
        assert bad.size == 0, f"{what} {name}: {bad.size} blocks differ, first {bad[:4].tolist()}"


# (pixel offset, pixel stride padding, coefficient stride padding in elements, flags)
TRELLIS_LAYOUTS = [(1, 1, 8, 0), (15, 4099, 72, COEF_ZIGZAG), (3, 0, 0, COEF_ZIGZAG), (8, 7, 8, 0), (5, 2, 16, 0),
                   (13, 0, 8, COEF_ZIGZAG), (2, 3, 0, 0), (11, 5, 64, COEF_ZIGZAG), (4, 9, 8, 0),
                   (6, 1, 72, COEF_ZIGZAG), (7, 0, 0, 0), (9, 11, 8, COEF_ZIGZAG), (10, 1, 16, 0),
                   (12, 3, 8, COEF_ZIGZAG), (14, 0, 0, 0)]


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
@pytest.mark.parametrize("w,h,q", [(1297, 35, 90), (2063, 19, 80), (1100, 48, 95)])
def test_coef_trellis_dev_layouts(gpu_ctx, w, h, q, ct, ss):
    """Three differing frames per call at pixel offsets 1-15, odd pixel strides and padded coefficient
    strides, natural and zig-zag order; every coefficient slot guarded."""
    frames = trellis_frames(w, h, ct, 3, w + q)
    wants = [jt.jpeg_coefficients(f, w, h, ct, ss, q) for f in frames]
    case = [(1297, 35), (2063, 19), (1100, 48)].index((w, h)) * 3 + [(2, 1), (2, 0), (0, 0)].index((ct, ss))
    for layout in (TRELLIS_LAYOUTS[case % 15], TRELLIS_LAYOUTS[(case + 9) % 15]):
        got = coef_dev(gpu_ctx, frames, w, h, ct, ss, q, *layout)
        for i in range(3):
            same_coefficients(got[i], wants[i], (layout, i))


@pytest.mark.parametrize("w,h,ct,ss", [(1, 1, 0, 0), (9, 9, 2, 1)], ids=["gray-1x1", "420-9x9"])
def test_coef_trellis_dev_beyond_65535_frames(gpu_ctx, w, h, ct, ss):
    """70 000 tiny frames in one trellis group (the transform launches split at 65 535), at an odd
    offset and stride, zig-zag order; sampled frames against the oracle."""
    from pixo_b200 import jpeg
    n, ch, q = 70000, 1 if ct == 0 else 3, 75
    rng = np.random.default_rng(w)
    px = rng.integers(0, 256, (n, h * w * ch), dtype=np.uint8)
    px[::3] = px[::3] // 64 * 64
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    got = coef_dev_batch(gpu_ctx, px, w, h, ct, ss, q)
    for i in sampled(n):
        want = jt.jpeg_coefficients(px[i], w, h, ct, ss, q)
        same_coefficients([got[0][i], got[1][i], got[2][i]], want[:3], i)
    assert got[0].shape == (n, ny, 64) and got[1].shape == (n, nc, 64)


def coef_dev_batch(ctx, px, w, h, ct, ss, q):
    """px (n, frame bytes) at offset 5, stride frame + 1; zig-zag order, coefficient strides padded by
    8; returns (y, cb, cr) as (n, blocks, 64) arrays in natural order after checking the guards."""
    from pixo_b200 import _lib, jpeg
    n, flen = px.shape
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    stride = flen + 1
    host = stripes(5 + n * stride + 64)
    host[5:5 + n * stride].reshape(n, stride)[:, :flen] = px
    src = Buf(host)
    ys, cs = ny * 64 + 8, max(nc, 1) * 64 + 8
    dy = guarded(n * ys, np.int16, GUARD16)
    dcb = guarded(n * cs, np.int16, GUARD16)
    dcr = guarded(n * cs, np.int16, GUARD16)
    _, _, lq, cq = jpeg.quant_tables(q)
    run(ctx, _lib.load().pixo_b200_jpeg_coefficients_dev, src.ptr(5), stride, n, w, h, ct, ss,
        lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p), dy.ptr(64), ys, dcb.ptr(64), dcr.ptr(64), cs,
        COEF_TRELLIS | COEF_ZIGZAG, None)
    inv = np.argsort(ZZ)
    out = []
    for buf, st, nb in ((dy, ys, ny), (dcb, cs, nc), (dcr, cs, nc)):
        a = buf.get()
        assert_guard(a, [(64 + i * st, nb * 64) for i in range(n)], GUARD16, "coefficients")
        a = a[64:64 + n * st].reshape(n, st)[:, :nb * 64].reshape(n, nb, 64)
        out.append(a[..., inv])
    return out


def test_coef_trellis_dev_bands_at_a_ragged_width(gpu_ctx, lib):
    """A 12 345 x 11 995 4:2:0 frame (about 890 MB of f32 DCT, bands of 226 MCU rows) at pixel offset 3:
    the pitch 37 035 is odd, so every band's first pixel is unaligned, and the last MCU row is 11 pixel
    rows, so the last band replicates edge rows.  Crops of whole MCU rows around each band border and at
    the bottom edge against the oracle; guards before and after every array."""
    import torch
    from pixo_b200 import _lib, jpeg
    w, h, ct, ss, q, mcu, off = 12345, 11995, 2, 1, 80, 16, 3
    g = torch.Generator(device="cuda").manual_seed(12)
    base = torch.randint(0, 256, ((h + 7) // 8, (w + 7) // 8, 3), dtype=torch.uint8, device="cuda", generator=g)
    img = base.repeat_interleave(8, 0).repeat_interleave(8, 1)[:h, :w]
    buf = torch.full((w * h * 3 + 64,), 255, dtype=torch.uint8, device="cuda")
    buf[off:off + w * h * 3] = img.reshape(-1)
    buf[off:off + w * h * 3].view(h, w, 3)[::3] ^= torch.randint(0, 16, ((h + 2) // 3, w, 3), dtype=torch.uint8,
                                                                   device="cuda", generator=g)
    del base, img
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    arrs = [torch.full((n * 64 + 128,), GUARD16, dtype=torch.int16, device="cuda") for n in (ny, nc, nc)]
    _, _, lq, cq = jpeg.quant_tables(q)
    run(gpu_ctx, lib.pixo_b200_jpeg_coefficients_dev, buf.data_ptr() + off, w * h * 3, 1, w, h, ct, ss,
        lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p), arrs[0].data_ptr() + 128, ny * 64,
        arrs[1].data_ptr() + 128, arrs[2].data_ptr() + 128, nc * 64, COEF_TRELLIS, None)
    for a, n in zip(arrs, (ny, nc, nc)):
        assert bool((a[:64] == GUARD16).all()) and bool((a[64 + n * 64:] == GUARD16).all())
    mx, my = (w + mcu - 1) // mcu, (h + mcu - 1) // mcu
    row_bytes = mx * 6 * 256
    band = (256 << 20) // row_bytes
    assert row_bytes * my > 256 << 20 and band == 226 and h % mcu
    for m0 in sorted({band - 1, 2 * band - 1, 3 * band - 1, my - 2}):
        r0, r1 = m0 * mcu, min(h, (m0 + 2) * mcu)
        crop = buf[off + r0 * w * 3:off + r1 * w * 3].cpu().numpy()
        want = jt.jpeg_coefficients(crop, w, r1 - r0, ct, ss, q)
        got = [a[64 + m0 * mx * k * 64:][:len(wa) * 64].cpu().numpy().reshape(-1, 64)
               for a, k, wa in zip(arrs, (4, 1, 1), want)]
        same_coefficients(got, want, m0)
    del buf, arrs
    torch.cuda.empty_cache()


def test_trellis_quantize_dev_inside_a_larger_tensor(gpu_ctx):
    """Blocks at 16-byte (not 256-byte) aligned offsets of larger tensors, 1 to 20 001 blocks, with guards
    after d_out; natural and zig-zag order."""
    import torch
    from pixo_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(6)
    d = (rng.laplace(0, 40, (20001, 64)) * (rng.random((20001, 64)) < 0.6)).astype(np.float32)
    q = rng.integers(1, 100, 64).astype(np.float32)
    want = jt.trellis_quantize_blocks(d, q, 0.75)
    src = torch.from_numpy(np.concatenate([np.full(4, np.nan, np.float32), d.reshape(-1),
                                           np.full(64, np.nan, np.float32)])).cuda()
    for nb in (1, 63, 64, 65, 20001):
        for flags in (0, COEF_ZIGZAG):
            out = guarded(nb * 64, np.int16, GUARD16, base=8, tail=72)
            run(gpu_ctx, lib.pixo_b200_jpeg_trellis_quantize_dev, src.data_ptr() + 16, nb, q.ctypes.data_as(_lib.f32p),
                0.75, out.ptr(8), flags)
            got = out.get()
            assert_guard(got, [(8, nb * 64)], GUARD16, f"d_out {nb}")
            got = got[8:8 + nb * 64].reshape(nb, 64)
            assert np.array_equal(got, want[:nb][:, ZZ] if flags else want[:nb]), (nb, flags)


def test_trellis_quantize_dev_refuses_misaligned_blocks(gpu_ctx):
    import torch
    from pixo_b200 import _lib
    lib = _lib.load()
    d = torch.zeros(64 * 8 + 16, dtype=torch.float32, device="cuda")
    out = guarded(64 * 8, np.int16, GUARD16, base=8, tail=72)
    q = np.full(64, 3.0, np.float32)
    torch.cuda.synchronize()
    l0 = gpu_ctx.launch_count
    for src_off, dst_off in [(1, 0), (2, 0), (3, 0), (0, 1), (0, 3), (0, 4), (0, 7), (5, 2)]:
        rc = lib.pixo_b200_jpeg_trellis_quantize_dev(gpu_ctx.handle, d.data_ptr() + 4 * src_off, 8,
                                                     q.ctypes.data_as(_lib.f32p), 1.0, out.ptr(8 + dst_off), 0)
        assert rc == _lib.ERR_INVALID_ARGUMENT, (src_off, dst_off, rc)
    assert gpu_ctx.launch_count == l0
    gpu_ctx.sync()
    assert_guard(out.get(), [], GUARD16, "d_out of refused calls")
