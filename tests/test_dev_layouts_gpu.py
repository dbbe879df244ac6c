"""The device-pointer entry points at the layouts their callers pass: frames of a batch at padded and
odd strides, buffers at offsets that are not 16-byte aligned, batches across the 65 535-frames-per-launch
split.  The host entry points copy into the context's own aligned, tightly packed scratch, so only these
calls reach the kernels' per-image indexing, stride arithmetic, alignment-chosen fast paths and masked
end stores.

Every element around an input frame holds a poison that changes the result if a kernel reads it (random
bytes around PNG rows, 0/255 stripes around JPEG pixels, 0x7FFF around coefficient arrays), and every
element around an output region holds a guard that must survive the call.  Frames of one batch differ
(noise, smooth, flat, mixed), so a mix-up between images cannot pass.  Each frame is compared with the
oracle or zlib."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from pixo_b200 import ColorType, _lib, jpeg, parallel
from pixo_b200.jpeg import JpegOptions, Subsampling

pytestmark = pytest.mark.gpu

GUARD8, GUARD16, GUARD32, GUARD64 = 0xA5, 0x5A5A, 0x5A5A5A5A, 0x5A5A5A5A5A5A5A5A
POISON16 = 0x7FFF
OPTIMIZE_ALPHA, ZIGZAG = 0x100, 1
KINDS = ("noise", "smooth", "flat", "mixed")


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    """Every frame here must be finished by the GPU entropy stage."""
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was silently finished by the host entropy coder"


# ---- harness ------------------------------------------------------------------------------------------
class Buf:
    """One device allocation holding `host` (any numpy dtype); ptr(k) is the address of element k."""

    def __init__(self, host):
        self.t = torch.from_numpy(np.ascontiguousarray(host)).cuda()

    def ptr(self, k=0):
        return self.t.data_ptr() + k * self.t.element_size()

    def get(self):
        return self.t.cpu().numpy()


def noise_poison(seed):
    return lambda n: np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)


def stripes(n):
    return np.where((np.arange(n) // 3) % 2 == 0, 0, 255).astype(np.uint8)


def placed(frames, base, stride, fill):
    """frames (equal size, one dtype) at element base + i*stride; every other element from `fill`
    (a callable giving n elements, or a scalar)."""
    flen = frames[0].size
    size = base + (len(frames) - 1) * stride + flen + 64
    host = fill(size) if callable(fill) else np.full(size, fill, frames[0].dtype)
    for i, f in enumerate(frames):
        host[base + i * stride: base + i * stride + flen] = np.ascontiguousarray(f).reshape(-1)
    return Buf(host)


def guarded(n, dtype, guard, base=64, tail=64):
    """n output elements at element `base` of a buffer whose every element starts as `guard`."""
    return Buf(np.full(base + n + tail, guard, dtype))


def assert_guard(host, regions, guard, what):
    """Every element outside the (start, length) regions still holds `guard`."""
    mask = np.ones(host.size, bool)
    for s, n in regions:
        mask[s:s + n] = False
    bad = np.flatnonzero(mask & (host != guard))
    assert bad.size == 0, f"{what}: {bad.size} guard elements changed, first at {bad[:8].tolist()}"


def run(ctx, fn, *args):
    """The library works on its own stream: torch's uploads must have landed, and its results must have."""
    torch.cuda.synchronize()
    _lib.check(ctx.handle, fn(ctx.handle, *args))
    ctx.sync()


def content(kind, h, rb, bpp, seed):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, rb), dtype=np.uint8)
    if kind == "smooth":
        x = np.cumsum(rng.integers(-2, 3, (h, rb)), axis=1) + np.cumsum(rng.integers(-1, 2, (h, 1)), axis=0)
        return (x & 255).astype(np.uint8)
    if kind == "flat":
        return np.tile(rng.integers(0, 256, bpp, dtype=np.uint8), (h, rb // bpp + 1))[:, :rb].copy()
    pick = (np.arange(h) // 3) % 2 == 0
    return np.where(pick[:, None], content("noise", h, rb, bpp, seed), content("smooth", h, rb, bpp, seed + 1))


def png_frames(w, h, rb, bpp, n, seed):
    """n differing frames; with an alpha channel (bpp 2 / 4) about a third of the pixels are fully
    transparent with non-zero colour, so OPTIMIZE_ALPHA changes them."""
    out = []
    for i in range(n):
        f = content(KINDS[i % 4], h, rb, bpp, seed + 7 * i)
        if bpp in (2, 4) and rb == w * bpp:
            px = f.reshape(h, w, bpp)
            clear = np.random.default_rng(seed + i).random((h, w)) < 0.35
            px[..., :-1] = np.where(clear[..., None] & (px[..., :-1] == 0), 9, px[..., :-1])
            px[..., -1] = np.where(clear, 0, np.maximum(px[..., -1], 1))
        out.append(f.reshape(-1))
    return out


def png_ref(po, frame, w, h, rb, bpp, word):
    """pixo: maybe_optimize_alpha (GrayAlpha / Rgba only), then apply_filters_with_row_bytes"""
    if word & OPTIMIZE_ALPHA and bpp in (2, 4):
        frame = po.optimize_alpha(frame, 1 if bpp == 2 else 3)
    return po.apply_filters(frame, w, h, bpp, word & 0xFF, row_bytes=rb)


def scan_bytes(jpg: bytes) -> bytes:
    """entropy-coded segment of a baseline file: after the SOS header, before EOI"""
    i = 2
    while True:
        ln = int.from_bytes(jpg[i + 2:i + 4], "big")
        if jpg[i + 1] == 0xDA:
            return jpg[i + 2 + ln:-2]
        i += 2 + ln


# ---- Adler-32 -----------------------------------------------------------------------------------------
ADLER_LENGTHS = [0, 1, 15, 16, 17, 31, 5551, 5552, 5553, 65543, (1 << 20) + 3]


def test_adler32_dev_offsets_and_lengths(gpu_ctx):
    """Base offsets 0-15 reach k_adler32's head loop (bytes before the first 16-byte boundary) and its
    tail loop; the bytes around each range are random, so reading one of them changes the sum."""
    lib = _lib.load()
    data = noise_poison(3)((1 << 20) + 64)
    src = Buf(data)
    cases = [(off, n) for off in range(16) for n in ADLER_LENGTHS]
    out = guarded(len(cases), np.int32, GUARD32, base=4, tail=4)
    torch.cuda.synchronize()
    for k, (off, n) in enumerate(cases):
        _lib.check(gpu_ctx.handle, lib.pixo_b200_adler32_dev(gpu_ctx.handle, src.ptr(off + 16), n, out.ptr(4 + k)))
    gpu_ctx.sync()
    got = out.get()
    assert_guard(got, [(4, len(cases))], GUARD32, "d_out")
    for k, (off, n) in enumerate(cases):
        want = zlib.adler32(data[off + 16:off + 16 + n].tobytes())
        assert int(got[4 + k]) & 0xFFFFFFFF == want, (off, n)


def test_adler32_dev_beyond_4_gib(gpu_ctx):
    """One buffer longer than 2^32 bytes, at an odd address: byte weights and indices past 32 bits."""
    lib = _lib.load()
    n = (1 << 32) + 4099
    d = torch.randint(0, 256, (n + 8,), dtype=torch.uint8, device="cuda")
    out = guarded(1, np.int32, GUARD32, base=4, tail=4)
    run(gpu_ctx, lib.pixo_b200_adler32_dev, d.data_ptr() + 5, n, out.ptr(4))
    want, chunk = 1, 1 << 28
    for s in range(5, n + 5, chunk):
        want = zlib.adler32(d[s:min(s + chunk, n + 5)].cpu().numpy().tobytes(), want)
    got = out.get()
    assert_guard(got, [(4, 1)], GUARD32, "d_out")
    assert int(got[4]) & 0xFFFFFFFF == want
    del d
    torch.cuda.empty_cache()


# ---- PNG filter, batches ------------------------------------------------------------------------------
# (input offset, input stride padding, output offset, output stride padding)
PNG_LAYOUTS = [(0, 0, 0, 0), (1, 1, 5, 3), (7, 4099, 0, 3), (1, 4099, 5, 0)]


def png_filter_dev(ctx, frames, w, h, rb, bpp, word, layout, seed):
    """One pixo_b200_png_filter_dev call on `frames` laid out as `layout`; checks the guards and
    returns (filtered frames, their Adler-32s)."""
    in_off, in_pad, out_off, out_pad = layout
    n = len(frames)
    in_stride, out_len = rb * h + in_pad, h * (rb + 1)
    out_stride = out_len + out_pad
    src = placed(frames, in_off, in_stride, noise_poison(seed))
    dst = guarded((n - 1) * out_stride + out_len, np.uint8, GUARD8, base=64 + out_off)
    ad = guarded(n, np.int32, GUARD32, base=4, tail=4)
    run(ctx, _lib.load().pixo_b200_png_filter_dev, src.ptr(in_off), in_stride, n, w, h, rb, bpp, word,
        dst.ptr(64 + out_off), out_stride, ad.ptr(4))
    out, ads = dst.get(), ad.get()
    o0 = 64 + out_off
    assert_guard(out, [(o0 + i * out_stride, out_len) for i in range(n)], GUARD8, f"filtered output {layout}")
    assert_guard(ads, [(4, n)], GUARD32, "d_adler")
    return [out[o0 + i * out_stride:o0 + i * out_stride + out_len] for i in range(n)], ads[4:4 + n].view(np.uint32)


PNG_GEOMETRIES = ([(37, 5, b, None) for b in (1, 2, 3, 4)]            # area <= 4096: adaptive strategies are Sub
                  + [(1000, 70, b, None) for b in (1, 2, 3, 4)]       # several 16-row bands
                  + [(300, 20, 4, None), (1001, 50, 1, 126),           # sticky AdaptiveFast; row_bytes override
                     (30000, 3, 4, None), (30000, 40, 4, None)])       # rows longer than 32 KiB


@pytest.mark.parametrize("w,h,bpp,rb", PNG_GEOMETRIES)
def test_png_filter_dev_batches(po, gpu_ctx, w, h, bpp, rb):
    """All nine strategies on three differing frames per layout; OPTIMIZE_ALPHA on half the calls at
    bpp 2 and 4.  Every frame and every per-image Adler-32 against the oracle and zlib."""
    rb = rb or w * bpp
    frames = png_frames(w, h, rb, bpp, 3, w + h + bpp)
    refs = {}
    for li, layout in enumerate(PNG_LAYOUTS):
        for s in range(9):
            word = s | (OPTIMIZE_ALPHA if bpp in (2, 4) and rb == w * bpp and (s + li) % 2 else 0)
            if word not in refs:
                refs[word] = [png_ref(po, f, w, h, rb, bpp, word) for f in frames]
            got, ads = png_filter_dev(gpu_ctx, frames, w, h, rb, bpp, word, layout, li)
            for i, (g, r) in enumerate(zip(got, refs[word])):
                assert np.array_equal(g, r), (layout, hex(word), i, np.flatnonzero(g != r)[:5])
                assert int(ads[i]) == zlib.adler32(r.tobytes()), (layout, hex(word), i)


def test_png_filter_dev_sticky_adaptive_fast_batch(po, gpu_ctx):
    """Height <= 32: AdaptiveFast keeps row 0's winner for the whole image, and each image of a batch
    has its own winner (k_png_filter's per-image `decided` byte)."""
    w, h, bpp = 300, 20, 4
    rb = w * bpp
    frames = [f.reshape(h, rb) for f in png_frames(w, h, rb, bpp, 4, 11)]
    frames[0][0] = 200                       # a flat first row: Sub
    frames[1][0] = np.random.default_rng(1).choice(np.array([0, 1, 255], np.uint8), rb)  # raw bytes near 0: Up
    frames[3][0] = np.arange(rb) * 37 % 256  # a steep ramp: Up
    frames = [f.reshape(-1) for f in frames]
    for word in (7, 7 | OPTIMIZE_ALPHA):
        refs = [png_ref(po, f, w, h, rb, bpp, word) for f in frames]
        winners = [int(r[0]) for r in refs]
        assert len(set(winners)) >= 2, winners
        for r in refs:
            assert len(set(r.reshape(h, rb + 1)[:, 0].tolist())) == 1
        for layout in PNG_LAYOUTS:
            got, ads = png_filter_dev(gpu_ctx, frames, w, h, rb, bpp, word, layout, 5)
            for i, (g, r) in enumerate(zip(got, refs)):
                assert np.array_equal(g, r), (layout, hex(word), i, winners, int(g[0]))
                assert int(ads[i]) == zlib.adler32(r.tobytes())


def test_png_filter_dev_across_the_launch_split(po, gpu_ctx):
    """65 537 tiny images: the kernels run 65 535 images per launch, so the last two sit in a second
    launch with its own image base, output base and Adler-32 slots."""
    n, w, h, bpp = 65537, 8, 1, 4
    rb = w * bpp
    frames = np.random.default_rng(5).integers(0, 256, (n, rb), dtype=np.uint8)
    src = placed([frames.reshape(-1)], 3, 0, noise_poison(6))
    dst = guarded(n * (rb + 1), np.uint8, GUARD8)
    ad = guarded(n, np.int32, GUARD32, base=4, tail=4)
    run(gpu_ctx, _lib.load().pixo_b200_png_filter_dev, src.ptr(3), rb, n, w, h, rb, bpp, 4, dst.ptr(64), rb + 1,
        ad.ptr(4))
    out, ads = dst.get(), ad.get()
    assert_guard(out, [(64, n * (rb + 1))], GUARD8, "filtered output")
    assert_guard(ads, [(4, n)], GUARD32, "d_adler")
    got = out[64:64 + n * (rb + 1)].reshape(n, rb + 1)
    # one row with zeros above: the Paeth predictor is the left pixel
    want = np.empty_like(got)
    want[:, 0] = 4
    want[:, 1:] = frames - np.pad(frames, ((0, 0), (bpp, 0)))[:, :rb]
    for i in (0, 65534, 65535, 65536):
        assert np.array_equal(want[i], po.apply_filters(frames[i], w, h, bpp, 4)), i
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, f"{bad.size} images differ, first {bad[:8].tolist()}"
    want_ad = np.array([zlib.adler32(r.tobytes()) for r in want], np.uint32)
    bad = np.flatnonzero(ads[4:4 + n].view(np.uint32) != want_ad)
    assert bad.size == 0, f"{bad.size} Adler-32s differ, first {bad[:8].tolist()}"


def test_png_filter_dev_rejects_overlapping_frames(po, gpu_ctx):
    """With more than one image, strides below one frame would let images' CTAs read and write each
    other's bytes; they are refused before any launch.  A single image ignores its strides."""
    lib = _lib.load()
    w, h, bpp = 40, 6, 4
    rb = w * bpp
    frames = png_frames(w, h, rb, bpp, 2, 1)
    src = placed(frames, 0, rb * h, noise_poison(2))
    dst = guarded(2 * h * (rb + 1), np.uint8, GUARD8)
    torch.cuda.synchronize()
    l0 = gpu_ctx.launch_count
    for in_stride, out_stride, code in ((rb * h - 1, h * (rb + 1), _lib.ERR_INVALID_DATA_LENGTH),
                                        (0, h * (rb + 1), _lib.ERR_INVALID_DATA_LENGTH),
                                        (rb * h, h * (rb + 1) - 1, _lib.ERR_OUTPUT_TOO_SMALL),
                                        (rb * h, 0, _lib.ERR_OUTPUT_TOO_SMALL)):
        rc = lib.pixo_b200_png_filter_dev(gpu_ctx.handle, src.ptr(), in_stride, 2, w, h, rb, bpp, 6, dst.ptr(64),
                                          out_stride, None)
        assert rc == code, (in_stride, out_stride, rc)
    assert gpu_ctx.launch_count == l0
    gpu_ctx.sync()
    assert_guard(dst.get(), [], GUARD8, "output of a refused call")
    run(gpu_ctx, lib.pixo_b200_png_filter_dev, src.ptr(), 0, 1, w, h, rb, bpp, 6, dst.ptr(64), 0, None)
    assert np.array_equal(dst.get()[64:64 + h * (rb + 1)], png_ref(po, frames[0], w, h, rb, bpp, 6))


# ---- PNG filter, row bands ----------------------------------------------------------------------------
F_MINSUM, F_ADAPTIVE, F_ADAPTIVE_FAST, F_BIGRAMS = 5, 6, 7, 8


@pytest.mark.parametrize("w,h,bpp,word,cuts", [
    (1000, 70, 1, F_ADAPTIVE, [0, 1, 17, 50, 70]),
    (999, 70, 2, F_MINSUM, [0, 33, 34, 70]),
    (1001, 70, 3, F_ADAPTIVE_FAST, [0, 16, 48, 70]),
    (500, 70, 4, F_ADAPTIVE | OPTIMIZE_ALPHA, [0, 16, 33, 70]),
    (700, 50, 2, F_BIGRAMS | OPTIMIZE_ALPHA, [0, 7, 50]),
    (1000, 70, 4, F_BIGRAMS, [0, 16, 35, 70]),
    (30000, 40, 4, F_ADAPTIVE, [0, 13, 40]),
    (30000, 40, 4, F_BIGRAMS, [0, 21, 40]),
    (100, 40, 3, F_ADAPTIVE, [0, 10, 25, 40]),         # whole image area 4000: Sub
    (100, 50, 3, F_ADAPTIVE, [0, 10, 25, 50]),         # whole image area 5000: Adaptive, bands of 1000 px
    (100, 20, 4, F_ADAPTIVE_FAST, [0, 5, 20]),         # area 2000: Sub, so 20 rows do not make it sticky
])
def test_png_filter_rows_dev_bands(po, gpu_ctx, w, h, bpp, word, cuts):
    """One image in row bands with d_rows, d_row_above and d_out at odd offsets in poisoned or guarded
    buffers.  The bands' bytes equal the oracle's whole-image stream, and their Adler-32s combine to its."""
    rb = w * bpp
    img = png_frames(w, h, rb, bpp, 2, w + bpp)[1 if bpp == 4 else 0].reshape(h, rb)
    ref = png_ref(po, img.reshape(-1), w, h, rb, bpp, word)
    if word & OPTIMIZE_ALPHA:   # the row above a cut holds transparent pixels with non-zero colour
        for r0 in cuts[1:-1]:
            px = img[r0 - 1].reshape(w, bpp)
            assert ((px[:, -1] == 0) & (px[:, :-1] != 0).any(axis=1)).any()
    parts = []
    for k, (r0, r1) in enumerate(zip(cuts, cuts[1:])):
        rows = placed([img[r0:r1].reshape(-1)], 1 + 2 * k, 0, noise_poison(k))
        above = placed([img[r0 - 1]], 5, 0, noise_poison(k + 50)) if r0 else None
        n_out = (r1 - r0) * (rb + 1)
        dst = guarded(n_out, np.uint8, GUARD8, base=67)
        ad = guarded(1, np.int32, GUARD32, base=4, tail=4)
        run(gpu_ctx, _lib.load().pixo_b200_png_filter_rows_dev, rows.ptr(1 + 2 * k), above.ptr(5) if above else None,
            w, h, r1 - r0, rb, bpp, word, dst.ptr(67), ad.ptr(4))
        out, a = dst.get(), ad.get()
        assert_guard(out, [(67, n_out)], GUARD8, f"band {r0}:{r1}")
        assert_guard(a, [(4, 1)], GUARD32, "d_adler")
        got, want = out[67:67 + n_out], ref[r0 * (rb + 1):r1 * (rb + 1)]
        assert np.array_equal(got, want), (r0, r1, np.flatnonzero(got != want)[:5])
        adler = int(a[4]) & 0xFFFFFFFF
        assert adler == zlib.adler32(want.tobytes()), (r0, r1)
        parts.append((adler, n_out))
    assert parallel.adler32_combine(parts) == po.adler32(ref)


def test_png_filter_rows_dev_refuses_bands_of_a_sticky_image(po, gpu_ctx):
    """AdaptiveFast on an image of <= 32 rows (area > 4096) keeps row 0's filter for every row: a band
    without row 0 cannot know it, so such a band is refused; the whole image as one band is not."""
    lib = _lib.load()
    w, h, bpp = 300, 20, 4
    rb = w * bpp
    img = png_frames(w, h, rb, bpp, 1, 4)[0]
    rows = Buf(img)
    dst = guarded(h * (rb + 1), np.uint8, GUARD8)
    torch.cuda.synchronize()
    l0 = gpu_ctx.launch_count
    for r0, r1 in ((0, 10), (10, 20)):
        rc = lib.pixo_b200_png_filter_rows_dev(gpu_ctx.handle, rows.ptr(r0 * rb), rows.ptr((r0 - 1) * rb) if r0 else None,
                                               w, h, r1 - r0, rb, bpp, F_ADAPTIVE_FAST, dst.ptr(64), None)
        assert rc == _lib.ERR_UNSUPPORTED, (r0, r1, rc)
    assert gpu_ctx.launch_count == l0
    run(gpu_ctx, lib.pixo_b200_png_filter_rows_dev, rows.ptr(), None, w, h, h, rb, bpp, F_ADAPTIVE_FAST, dst.ptr(64), None)
    assert np.array_equal(dst.get()[64:64 + h * (rb + 1)], png_ref(po, img, w, h, rb, bpp, F_ADAPTIVE_FAST))


# ---- JPEG transform -----------------------------------------------------------------------------------
JPEG_MODES = [(2, 1), (2, 0), (0, 0), (0, 1)]   # (colour type, subsampling); Gray ignores subsampling


def jpeg_frames(po, w, h, ct, n, seed):
    ch = 3 if ct == 2 else 1
    grad = po.gen_gradient_rgb(w, h)
    out = []
    for i in range(n):
        kind = KINDS[i % 4]
        if kind == "smooth":
            f = grad if ch == 3 else grad[i % 3::3].copy()
        elif kind == "noise":
            f = po.gen_noise(w, h, ch, seed + i)
        else:
            f = content(kind, h, w * ch, ch, seed + i).reshape(-1)
        out.append(f)
    return out


def jpeg_ref(po, frame, w, h, ct, ss, q=80):
    """pixo's coefficients; pixo ignores the subsampling of Gray (src/jpeg/mod.rs:528-551)"""
    return po.jpeg_coefficients(frame, w, h, ct, ss if ct == 2 else 0, q)


# (pixel offset, pixel stride padding, coefficient stride padding in elements, flags)
COEF_LAYOUTS = [(0, 0, 0, 0), (3, 0, 8, ZIGZAG), (0, 5, 72, 0), (0, 4096, 72, ZIGZAG), (0, 0, 8, 0)]


@pytest.mark.parametrize("ct,ss", JPEG_MODES)
@pytest.mark.parametrize("w,h", [(530, 41), (513, 16), (1000, 7), (256, 256)])
def test_jpeg_coefficients_dev_padded_strides_and_histograms(po, gpu_ctx, w, h, ct, ss):
    """Three differing frames per call at padded pixel and coefficient strides, natural and zig-zag
    order, with every frame's histogram.  At 256x256 (RGB pitch a multiple of 16) the first, fourth and
    fifth layouts load by TMA and the others through the clamped loader: all must agree."""
    lib = _lib.load()
    ch = 3 if ct == 2 else 1
    n, flen = 3, w * h * ch
    _, _, lq, cq = jpeg.quant_tables(80)
    frames = jpeg_frames(po, w, h, ct, n, w + h)
    refs = [jpeg_ref(po, f, w, h, ct, ss) for f in frames]
    hists = [po.jpeg_histograms(*r, w, h, ct, ss if ct == 2 else 0) for r in refs]
    ny, nc = len(refs[0][0]), len(refs[0][1])
    zz = np.array([int(v) for v in po.zigzag_reorder(np.arange(64, dtype=np.int16))])
    seen = []
    for layout in COEF_LAYOUTS:
        px_off, px_pad, c_pad, flags = layout
        pixel_stride = flen + px_pad
        src = placed(frames, px_off, pixel_stride, stripes)
        y_stride, c_stride = ny * 64 + c_pad, max(nc, 1) * 64 + c_pad
        dy = guarded((n - 1) * y_stride + ny * 64, np.int16, GUARD16)
        dcb = guarded((n - 1) * c_stride + nc * 64, np.int16, GUARD16)
        dcr = guarded((n - 1) * c_stride + nc * 64, np.int16, GUARD16)
        dh = guarded(n * 536, np.int64, GUARD64, base=4, tail=4)
        run(gpu_ctx, lib.pixo_b200_jpeg_coefficients_dev, src.ptr(px_off), pixel_stride, n, w, h, ct, ss,
            lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p), dy.ptr(64), y_stride, dcb.ptr(64),
            dcr.ptr(64), c_stride, flags, dh.ptr(4))
        y, cb, cr, hist = dy.get(), dcb.get(), dcr.get(), dh.get()
        assert_guard(y, [(64 + i * y_stride, ny * 64) for i in range(n)], GUARD16, f"Y {layout}")
        for a, name in ((cb, "Cb"), (cr, "Cr")):
            assert_guard(a, [(64 + i * c_stride, nc * 64) for i in range(n)], GUARD16, f"{name} {layout}")
        assert_guard(hist, [(4, n * 536)], GUARD64, f"d_hist {layout}")
        got = []
        for i in range(n):
            arrs = [y[64 + i * y_stride:][:ny * 64], cb[64 + i * c_stride:][:nc * 64], cr[64 + i * c_stride:][:nc * 64]]
            arrs = [a.reshape(-1, 64) for a in arrs]
            if flags & ZIGZAG:
                arrs = [a[:, np.argsort(zz)] for a in arrs]
            for a, r, name in zip(arrs, refs[i], ("Y", "Cb", "Cr")):
                assert np.array_equal(a, r), (layout, i, name, int((a != r).sum()))
            assert np.array_equal(hist[4 + i * 536:4 + (i + 1) * 536].view(np.uint64), hists[i]), (layout, i)
            got.append(arrs)
        seen.append(got)
    for other in seen[1:]:   # TMA and clamped loads (at 256x256) give identical arrays
        assert all(np.array_equal(a, b) for fa, fb in zip(seen[0], other) for a, b in zip(fa, fb))


def test_jpeg_coefficients_dev_across_the_launch_split(po, gpu_ctx):
    """65 537 gray 8x8 frames with histograms: the transform and K3 run 65 535 frames per launch."""
    lib = _lib.load()
    n = 65537
    rng = np.random.default_rng(9)
    px = rng.integers(0, 256, (n, 64), dtype=np.uint8)
    px[::3] = (px[::3] // 32) * 32           # some frames with fewer distinct values, shorter blocks
    px[1::7] = px[1::7, :1]                   # and some flat ones
    _, _, lq, cq = jpeg.quant_tables(80)
    src = placed([px.reshape(-1)], 0, 0, stripes)
    dy = guarded(n * 64, np.int16, GUARD16)
    dh = guarded(n * 536, np.int64, GUARD64, base=4, tail=4)
    run(gpu_ctx, lib.pixo_b200_jpeg_coefficients_dev, src.ptr(), 64, n, 8, 8, 0, 1, lq.ctypes.data_as(_lib.f32p),
        cq.ctypes.data_as(_lib.f32p), dy.ptr(64), 64, None, None, 0, 0, dh.ptr(4))
    y, hist = dy.get(), dh.get()
    assert_guard(y, [(64, n * 64)], GUARD16, "Y")
    assert_guard(hist, [(4, n * 536)], GUARD64, "d_hist")
    y = y[64:64 + n * 64].reshape(n, 64)
    hist = hist[4:4 + n * 536].view(np.uint64).reshape(n, 536)
    # the frames stacked vertically are one 8 x (8n) gray image whose block i is frame i
    ry, _, _ = po.jpeg_coefficients(px.reshape(-1), 8, 8 * n, 0, 0, 80)
    bad = np.flatnonzero((y != ry).any(axis=1))
    assert bad.size == 0, f"{bad.size} frames differ, first {bad[:8].tolist()}"
    # one block per frame: one DC symbol, of the category of the frame's DC, and no chroma symbols
    cat = np.array([int(v).bit_length() for v in np.abs(ry[:, 0].astype(np.int64))])
    assert (hist[:, :12].sum(axis=1) == 1).all() and (hist[np.arange(n), cat] == 1).all()
    assert not hist[:, 12:24].any() and not hist[:, 280:].any()
    empty = np.zeros((0, 64), np.int16)
    for i in (0, 1, 65533, 65534, 65535, 65536):
        assert np.array_equal(hist[i], po.jpeg_histograms(ry[i:i + 1], empty, empty, 8, 8, 0, 0)), i


# ---- JPEG device encode -------------------------------------------------------------------------------
def encode_dev(ctx, frames, w, h, ct, ss, q, px_off, px_pad, cap):
    """pixo_b200_jpeg_encode_dev on `frames` at the given pixel layout into slots of `cap` bytes;
    checks the guards before the first slot, after the last and around the length / flag words."""
    n, flen = len(frames), frames[0].size
    src = placed(frames, px_off, flen + px_pad, stripes)
    scan = guarded(n * cap, np.uint8, GUARD8)
    lens = guarded(n, np.int64, GUARD64, base=2, tail=2)
    ovf = guarded(n, np.int32, GUARD32, base=2, tail=2)
    run(ctx, _lib.load().pixo_b200_jpeg_encode_dev, src.ptr(px_off), flen + px_pad, n, w, h, ct, q, ss, scan.ptr(64),
        cap, lens.ptr(2), ovf.ptr(2))
    s, ln, ov = scan.get(), lens.get(), ovf.get()
    assert_guard(s, [(64, n * cap)], GUARD8, "scan slots")
    assert_guard(ln, [(2, n)], GUARD64, "d_scan_len")
    assert_guard(ov, [(2, n)], GUARD32, "d_overflow")
    return [s[64 + i * cap:64 + (i + 1) * cap] for i in range(n)], ln[2:2 + n], ov[2:2 + n]


@pytest.mark.parametrize("ct,ss", JPEG_MODES)
def test_jpeg_encode_dev_batches(po, gpu_ctx, ct, ss):
    """Three differing frames at odd pixel offsets and strides, in slots whose size is 4 (mod 16), so
    the slots sit at different 16-byte phases."""
    for w, h in ((530, 41), (256, 256)):
        frames = jpeg_frames(po, w, h, ct, 3, 3 * w)
        refs = [scan_bytes(po.jpeg_encode(f, w, h, ct, 80, ss)) for f in frames]
        if ct == 0:
            assert refs == [scan_bytes(po.jpeg_encode(f, w, h, 0, 80, 0)) for f in frames]
        cap = (max(len(r) for r in refs) + 64 + 15) // 16 * 16 + 4
        for px_off, px_pad in ((0, 0), (3, 0), (0, 5), (5, 4099)):
            slots, lens, ovf = encode_dev(gpu_ctx, frames, w, h, ct, ss, 80, px_off, px_pad, cap)
            for i, r in enumerate(refs):
                assert ovf[i] == 0 and lens[i] == len(r), (w, h, px_off, px_pad, i)
                assert slots[i][:len(r)].tobytes() == r, (w, h, px_off, px_pad, i)


def test_jpeg_encode_dev_frame_too_large_for_its_slot(po, gpu_ctx):
    """A frame that does not fit its slot between two that do: only its overflow bit 0 is set, its
    length is the size it needs, and its neighbours' slots and the guard after the last are intact."""
    w, h = 256, 256
    frames = [po.gen_gradient_rgb(w, h), po.gen_noise(w, h, 3, 4),
              np.roll(po.gen_gradient_rgb(w, h).reshape(h, -1), 9, axis=0).reshape(-1)]
    refs = [scan_bytes(po.jpeg_encode(f, w, h, 2, 80, 1)) for f in frames]
    cap = (max(len(refs[0]), len(refs[2])) + 15) // 16 * 16 + 4
    assert len(refs[1]) > cap
    slots, lens, ovf = encode_dev(gpu_ctx, frames, w, h, 2, 1, 80, 1, 3, cap)
    assert ovf[0] == 0 and ovf[2] == 0 and ovf[1] & 1, ovf
    assert lens.tolist() == [len(r) for r in refs]
    for i in (0, 2):
        assert slots[i][:len(refs[i])].tobytes() == refs[i], i


# ---- caller coefficient arrays ------------------------------------------------------------------------
def embedded(a, off):
    """`a` (blocks x 64 int16) at element `off` of a device tensor holding 0x7FFF everywhere else (a
    value outside the baseline range: reading it fails the range check or changes the scan)."""
    host = np.full(off + a.size + 40, POISON16, np.int16)
    host[off:off + a.size] = a.reshape(-1)
    t = torch.from_numpy(host).cuda()
    return t[off:off + a.size].view(-1, 64)


@pytest.mark.parametrize("w,h,ct,ss", [(333, 222, 2, 1), (200, 75, 2, 0), (257, 129, 0, 0)])
def test_caller_coefficients_inside_a_larger_tensor(po, gpu_ctx, w, h, ct, ss):
    """Arrays at a 16-byte (not 256-byte) aligned offset of larger tensors: entropy_encode_dev with
    standard and optimised tables and a restart interval; band_histogram_dev; band_entropy_dev and
    its stream-ordered twin, spliced; all byte-identical to the oracle."""
    lib = _lib.load()
    frame = po.gen_noise(w, h, 3 if ct == 2 else 1, 21)
    ry, rcb, rcr = po.jpeg_coefficients(frame, w, h, ct, ss, 80)
    d = [embedded(ry, 24), embedded(rcb, 8) if ct else None, embedded(rcr, 40) if ct else None]
    torch.cuda.synchronize()
    for ri in (0, 7):
        for opt in (False, True):
            o = JpegOptions(w, h, ColorType(ct), 80, Subsampling(ss), ri or None, opt)
            want = po.jpeg_encode_from_coefficients(ry, rcb, rcr, w, h, ct, 80, ss, ri, opt)
            assert jpeg.entropy_encode_dev(*d, o, ctx=gpu_ctx) == want, (ri, opt)
    p = lambda t: None if t is None else t.data_ptr()
    zero = (C.c_int32 * 3)(0, 0, 0)
    dh = guarded(536, np.int64, GUARD64, base=4, tail=4)
    run(gpu_ctx, lib.pixo_b200_jpeg_band_histogram_dev, p(d[0]), p(d[1]), p(d[2]), w, h, ct, ss, zero, dh.ptr(4))
    hist = dh.get()
    assert_guard(hist, [(4, 536)], GUARD64, "d_hist")
    assert np.array_equal(hist[4:540].view(np.uint64), po.jpeg_histograms(ry, rcb, rcr, w, h, ct, ss))
    coder = parallel.DeviceBandCoder(gpu_ctx, d[0], d[1], d[2], w, h, ct, ss, len(ry), len(rcb))
    for opt in (False, True):
        want = po.jpeg_encode_from_coefficients(ry, rcb, rcr, w, h, ct, 80, ss, 0, opt)
        assert parallel.encode_tiled_local([coder], w, h, ct, 80, ss, opt) == want, opt
    # stream-ordered: coding and splice with the seed, offsets and flags in device memory
    raw = torch.empty((w * h * 3 + (2 << 20)) // 16 * 16, dtype=torch.uint8, device="cuda")
    out = torch.full((raw.numel() * 2,), GUARD8, dtype=torch.uint8, device="cuda")
    seed = torch.zeros(3, dtype=torch.int32, device="cuda")
    bits_tail = torch.zeros(2, dtype=torch.int64, device="cuda")
    offset = torch.tensor([0, 0, 1], dtype=torch.int64, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    out_len = torch.zeros(1, dtype=torch.int64, device="cuda")
    run(gpu_ctx, lib.pixo_b200_jpeg_band_entropy_dev_async, p(d[0]), p(d[1]), p(d[2]), w, h, ct, ss, seed.data_ptr(),
        None, raw.data_ptr(), raw.numel(), bits_tail.data_ptr(), flags.data_ptr())
    run(gpu_ctx, lib.pixo_b200_jpeg_band_splice_dev_async, raw.data_ptr(), offset.data_ptr(), out.data_ptr(),
        out.numel(), out_len.data_ptr(), flags.data_ptr())
    assert int(flags.item()) == 0
    want = scan_bytes(po.jpeg_encode_from_coefficients(ry, rcb, rcr, w, h, ct, 80, ss))
    assert int(out_len.item()) == len(want)
    got = out.cpu().numpy()
    assert got[:len(want)].tobytes() == want


def test_misaligned_caller_coefficients_are_refused(po, gpu_ctx):
    """Coefficient arrays that are not 16-byte aligned (a slice like t[3:]) are refused on the host
    with ERR_INVALID_ARGUMENT before any kernel sees them, by every entry point that takes them; the
    context then codes aligned arrays correctly."""
    lib = _lib.load()
    w, h, ct, ss = 64, 48, 2, 1
    ry, rcb, rcr = po.jpeg_coefficients(po.gen_noise(w, h, 3, 2), w, h, ct, ss, 80)
    aligned = [embedded(a, 8) for a in (ry, rcb, rcr)]
    buf = np.zeros(1 << 16, np.uint8)
    n = C.c_size_t()
    zero = (C.c_int32 * 3)(0, 0, 0)
    dh = guarded(536, np.int64, GUARD64, base=4, tail=4)
    raw = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    seed = torch.zeros(3, dtype=torch.int32, device="cuda")
    bits_tail = torch.zeros(2, dtype=torch.int64, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    nbits, tail = C.c_uint64(), C.c_uint32()
    torch.cuda.synchronize()
    for off in range(1, 8):
        for k in range(3):
            shifted = embedded((ry, rcb, rcr)[k], 8 + off)
            ptrs = [t.data_ptr() for t in aligned]
            ptrs[k] = shifted.data_ptr()
            torch.cuda.synchronize()
            l0 = gpu_ctx.launch_count
            calls = {
                "entropy_encode_dev": lambda: lib.pixo_b200_jpeg_entropy_encode_dev(
                    gpu_ctx.handle, *ptrs, w, h, ct, 80, ss, 0, 1, buf.ctypes.data, buf.size, C.byref(n)),
                "band_histogram_dev": lambda: lib.pixo_b200_jpeg_band_histogram_dev(
                    gpu_ctx.handle, *ptrs, w, h, ct, ss, zero, dh.ptr(4)),
                "band_entropy_dev": lambda: lib.pixo_b200_jpeg_band_entropy_dev(
                    gpu_ctx.handle, *ptrs, w, h, ct, ss, zero, None, raw.data_ptr(), raw.numel(), C.byref(nbits),
                    C.byref(tail)),
                "band_entropy_dev_async": lambda: lib.pixo_b200_jpeg_band_entropy_dev_async(
                    gpu_ctx.handle, *ptrs, w, h, ct, ss, seed.data_ptr(), None, raw.data_ptr(), raw.numel(),
                    bits_tail.data_ptr(), flags.data_ptr()),
            }
            for name, call in calls.items():
                assert call() == _lib.ERR_INVALID_ARGUMENT, (name, off, k)
                assert b"16-byte aligned" in lib.pixo_b200_last_error(gpu_ctx.handle), name
            assert gpu_ctx.launch_count == l0, (off, k)
    gpu_ctx.sync()
    assert_guard(dh.get(), [], GUARD64, "d_hist of refused calls")
    o = JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420, None, True)
    assert jpeg.entropy_encode_dev(*aligned, o, ctx=gpu_ctx) == \
        po.jpeg_encode_from_coefficients(ry, rcb, rcr, w, h, ct, 80, ss, 0, True)


# ---- Gray ignores subsampling -------------------------------------------------------------------------
def test_gray_with_s420_encodes_like_s444(po, gpu_ctx):
    """pixo ignores the subsampling of a Gray image (src/jpeg/mod.rs:528-551): S420 gives the S444 file,
    through encode and encode_batch."""
    w, h = 333, 222
    frames = np.stack(jpeg_frames(po, w, h, 0, 3, 8))
    for ri, opt in ((None, False), (5, True)):
        o420 = JpegOptions(w, h, ColorType.Gray, 80, Subsampling.S420, ri, opt)
        o444 = JpegOptions(w, h, ColorType.Gray, 80, Subsampling.S444, ri, opt)
        batch = jpeg.encode_batch(frames, o420, ctx=gpu_ctx)
        for k, f in enumerate(frames):
            want = po.jpeg_encode(f, w, h, 0, 80, 1, ri or 0, opt)
            assert want == po.jpeg_encode(f, w, h, 0, 80, 0, ri or 0, opt)
            assert jpeg.encode(f, o420, ctx=gpu_ctx) == want, (ri, opt, k)
            assert jpeg.encode(f, o444, ctx=gpu_ctx) == want, (ri, opt, k)
            assert batch[k] == want, (ri, opt, k)
