"""The CUDA palette quantisation (pixo_b200_png_quantize_filter[_dev]) against real pixo output
(tests/golden/quantize/) with no oracle in between, and against oracle/png_quantize.py / .c for modes,
palette sizes, filters and geometries pixo's wasm API cannot select, full-size batches and errors."""
import ctypes as C

import numpy as np
import pytest

from oracle import png_quantize as pq
from oracle import png_reduce as pr
from quantize_inputs import load_manifest, make_quantize_input
from test_png_quantize import fixture_palette, fixture_parts, quantize_case_input

pytestmark = pytest.mark.gpu

MANIFEST = load_manifest()
MODES = {"off": 0, "auto": 1, "force": 2}


@pytest.fixture(autouse=True)
def no_host_fallback(gpu_ctx):
    """No frame of this file is finished by host code."""
    from pixo_b200 import _lib
    yield
    assert _lib.load().pixo_b200_ctx_host_fallbacks(gpu_ctx.handle) == 0


def _opts(w, h, ct, mode="auto", max_colors=256, dither=True, strategy=6, oa=False, rct=False, rpal=False):
    from pixo_b200 import ColorType
    from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode
    return PngOptions(w, h, ColorType(ct), FilterStrategy(strategy), oa, rct, rpal,
                      QuantizationMode(MODES[mode]), max_colors, dither)


def _oracle(po, img, w, h, ct, mode, max_colors, dither, strategy, oa=False, rct=False, rpal=False, palette=None):
    """(kind, palette-or-Reduced, filtered, adler) as encode_into hands them to DEFLATE."""
    if not pq.should_quantize(img, ct, mode, min(max_colors, 256)):
        red = pr.reduce(img, w, h, ct, rct, rpal)
        f = po.apply_filters(pr.filter_input(red, oa), w, h, red.bytes_per_pixel, strategy, row_bytes=red.row_bytes)
        return "lossless", red, f, po.adler32(f)
    pal, idx = pq.quantize(img, w, h, ct, max_colors, dither, palette)
    f = po.apply_filters(idx, w, h, 1, pq.indexed_strategy(strategy))
    return "indexed", pal, f, po.adler32(f)


def _same(got, want):
    red, f, ad = got
    kind, wp, wf, wad = want
    if kind == "indexed":
        assert (red.color_type_byte, red.bit_depth, red.bytes_per_pixel) == (3, 8, 1)
        assert int(red.effective_color_type) == 2
        assert np.array_equal(red.palette, wp)
        assert red.trns == pq.trimmed_trns(wp)
    else:
        assert (red.color_type_byte, red.bit_depth, red.bytes_per_pixel, red.row_bytes) == \
            (wp.color_type_byte, wp.bit_depth, wp.bytes_per_pixel, wp.row_bytes)
        if wp.palette is None:
            assert red.palette is None
        else:
            assert np.array_equal(red.palette, wp.palette)
    assert np.array_equal(np.asarray(f), wf) and ad == wad


# ---- real pixo output ---------------------------------------------------------------------------------
@pytest.mark.parametrize("c", MANIFEST["png"], ids=lambda c: c["file"])
def test_gpu_reproduces_pixo_lossy(gpu_ctx, c):
    from pixo_b200 import ColorType, PixoError, _lib, png
    img = quantize_case_input(c)
    parts = fixture_parts(c)
    o = png.PngOptions.from_preset_with_lossless(c["w"], c["h"], c["preset"], False)
    o.color_type = ColorType(c["ct"])
    given = None
    if c["kind"] == "trunc":
        with pytest.raises(PixoError) as e:
            png.quantize_and_filter(img, o, ctx=gpu_ctx)
        assert e.value.code == _lib.ERR_UNSUPPORTED and "8192" in str(e.value)
        given = fixture_palette(parts)
    red, f, ad = png.quantize_and_filter(img, o, palette=given, ctx=gpu_ctx)
    assert parts["ihdr"][:4] == (c["w"], c["h"], red.bit_depth, red.color_type_byte)
    assert parts["PLTE"] == (None if red.palette is None else red.palette[:, :3].tobytes())
    assert parts["tRNS"] == red.trns
    assert bytes(f) == parts["raw"]
    assert ad == parts["adler"]


# ---- against the oracle --------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["force", "auto"])
@pytest.mark.parametrize("dither", [True, False])
@pytest.mark.parametrize("max_colors", [0, 1, 2, 16, 255, 256, 300])
def test_modes_and_palette_sizes(po, gpu_ctx, mode, dither, max_colors):
    from pixo_b200 import png
    w, h = 71, 45
    for ct, kind, n in ((2, "grad", 0), (3, "pal", 700), (3, "palo", 40)):
        img = make_quantize_input(kind, w, h, ct + 1, 11, n)
        got = png.quantize_and_filter(img, _opts(w, h, ct, mode, max_colors, dither), ctx=gpu_ctx)
        _same(got, _oracle(po, img, w, h, ct, mode, max_colors, dither, 6))


def test_early_out_with_sampler_misses(po, gpu_ctx):
    """<= max_colors histogram colours: key-ordered palette, exact lookup, nearest entry for colours the
    stride-2 sampler missed (opaque and translucent), no dithering even when asked."""
    from pixo_b200 import png
    w, h = 400, 260
    for ct in (2, 3):
        img = make_quantize_input("missed", w, h, ct + 1, 5, 400).reshape(-1, ct + 1).copy()
        if ct == 3:
            img[1::7, 3] = 90                       # translucent colours on unsampled pixels
        img = img.reshape(-1)
        for dither in (True, False):
            got = png.quantize_and_filter(img, _opts(w, h, ct, "force", 256, dither), ctx=gpu_ctx)
            want = _oracle(po, img, w, h, ct, "force", 256, dither, 6)
            assert len(want[1]) <= 256
            _same(got, want)


@pytest.mark.parametrize("dither", [True, False])
def test_translucent_pixels(po, gpu_ctx, dither):
    from pixo_b200 import png
    w, h = 90, 70
    img = make_quantize_input("grad", w, h, 4, 3)
    got = png.quantize_and_filter(img, _opts(w, h, 3, "force", 64, dither), ctx=gpu_ctx)
    want = _oracle(po, img, w, h, 3, "force", 64, dither, 6)
    assert (want[1][:, 3] < 255).any()
    _same(got, want)


@pytest.mark.parametrize("strategy", range(9))
def test_filter_strategies_on_index_rows(po, gpu_ctx, strategy):
    from pixo_b200 import png
    w, h = 90, 70
    img = make_quantize_input("grad", w, h, 3, 7)
    for dither in (True, False):
        got = png.quantize_and_filter(img, _opts(w, h, 2, "force", 32, dither, strategy), ctx=gpu_ctx)
        _same(got, _oracle(po, img, w, h, 2, "force", 32, dither, strategy))


@pytest.mark.parametrize("h", [1, 2, 31, 32, 33, 64, 65, 97])
def test_warp_and_row_group_boundaries(po, gpu_ctx, h):
    from pixo_b200 import png
    for w in (1, 2, 3, 7, 33, 63, 64, 65, 200):
        ct = 3 if (w + h) % 2 else 2
        # a gradient while it has at most 8192 histogram colours, then colours in blocks
        img = make_quantize_input("grad", w, h, ct + 1, w * 100 + h) if w * h <= 6000 else \
            make_quantize_input("palblk", w, h, ct + 1, w * 100 + h, 2000)
        got = png.quantize_and_filter(img, _opts(w, h, ct, "force", 24, True), ctx=gpu_ctx)
        _same(got, _oracle(po, img, w, h, ct, "force", 24, True, 6))


def test_caller_palette(po, gpu_ctx):
    from pixo_b200 import png
    w, h = 150, 90
    img = make_quantize_input("grad", w, h, 4, 9)
    pal = make_quantize_input("pal", 37, 1, 4, 4, 37).reshape(-1, 4)
    for dither in (True, False):
        got = png.quantize_and_filter(img, _opts(w, h, 3, "force", 256, dither), palette=pal, ctx=gpu_ctx)
        _same(got, _oracle(po, img, w, h, 3, "force", 256, dither, 6, palette=pal))


# ---- full size, batched, through the device entry point ----------------------------------------------
def _run_dev(ctx, frames, w, h, ct, opts, in_stride=None, out_stride=None, palettes=None, reduce=False):
    import torch
    from pixo_b200 import png
    dev = torch.device("cuda", ctx.device)
    n, bpp = len(frames), ct + 1
    in_stride = in_stride or w * h * bpp
    out_stride = out_stride or h * (w * bpp + 1)
    d_in = torch.empty((n - 1) * in_stride + w * h * bpp, dtype=torch.uint8, device=dev)
    for i, fr in enumerate(frames):
        d_in[i * in_stride:i * in_stride + fr.size] = torch.from_numpy(fr).to(dev)
    d_out = torch.empty((n - 1) * out_stride + h * (w * bpp + 1), dtype=torch.uint8, device=dev)
    d_ad = torch.zeros(n, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    if reduce:
        infos = png.reduce_and_filter_dev(d_in, in_stride, n, opts, d_out, out_stride, d_ad, ctx=ctx)
    else:
        infos = png.quantize_and_filter_dev(d_in, in_stride, n, opts, d_out, out_stride, d_ad, palettes=palettes,
                                            ctx=ctx)
    ctx.sync()
    outs = [d_out[i * out_stride:i * out_stride + h * (infos[i].row_bytes + 1)].cpu().numpy() for i in range(n)]
    ads = [int(a) & 0xFFFFFFFF for a in d_ad.cpu().numpy()]
    del d_in, d_out
    return infos, outs, ads


def test_4k_mixed_batch(po, gpu_ctx):
    """16 dithered 4K RGBA frames, Auto: frames that quantise match the oracle, frames that do not match
    reduce_and_filter_dev's output for the same flags."""
    from pixo_b200.png import PngOptions
    w, h = 3840, 2160
    makers = [("palblk", 1000), ("pal", 4000), ("noise", 0), ("pal", 200)]
    frames = [make_quantize_input(makers[i % 4][0], w, h, 4, 40 + i, makers[i % 4][1]) for i in range(16)]
    opts = PngOptions.from_preset_with_lossless(w, h, 1, False)
    infos, outs, ads = _run_dev(gpu_ctx, frames, w, h, 3, opts)
    lossless = PngOptions.from_preset(w, h, 1)
    rinfos, routs, rads = _run_dev(gpu_ctx, frames, w, h, 3, lossless, reduce=True)
    kinds = []
    for i, fr in enumerate(frames):
        if pq.should_quantize(fr, 3, "auto", 256):
            _same((infos[i], outs[i], ads[i]), _oracle(po, fr, w, h, 3, "auto", 256, True, 6))
            kinds.append("q")
        else:
            a, b = infos[i], rinfos[i]
            assert (a.color_type_byte, a.bit_depth, a.row_bytes, a.trns) == (b.color_type_byte, b.bit_depth, b.row_bytes, b.trns)
            assert (a.palette is None and b.palette is None) or np.array_equal(a.palette, b.palette)
            assert np.array_equal(outs[i], routs[i]) and ads[i] == rads[i]
            kinds.append("l")
    assert kinds == ["q", "q", "l", "l"] * 4


def test_offsets_beyond_4_gib(po, gpu_ctx):
    w, h = 256, 128
    frames = [make_quantize_input("grad", w, h, 4, 7), make_quantize_input("pal", w, h, 4, 8, 20),
              make_quantize_input("pal", w, h, 4, 9, 900)]
    stride = (1 << 31) + 4096
    opts = _opts(w, h, 3, "auto", 256, True, 4, True, True, True)
    infos, outs, ads = _run_dev(gpu_ctx, frames, w, h, 3, opts, in_stride=stride, out_stride=stride)
    for fr, red, f, ad in zip(frames, infos, outs, ads):
        _same((red, f, ad), _oracle(po, fr, w, h, 3, "auto", 256, True, 4, True, True, True))


def test_dev_caller_palettes(po, gpu_ctx):
    w, h = 96, 80
    frames = [make_quantize_input("grad", w, h, 4, s) for s in (1, 2, 3)]
    pal = make_quantize_input("pal", 20, 1, 4, 4, 20).reshape(-1, 4)
    opts = _opts(w, h, 3, "force", 256, True)
    infos, outs, ads = _run_dev(gpu_ctx, frames, w, h, 3, opts, palettes=[None, pal, None])
    for k, (fr, red, f, ad) in enumerate(zip(frames, infos, outs, ads)):
        _same((red, f, ad), _oracle(po, fr, w, h, 3, "force", 256, True, 6, palette=pal if k == 1 else None))


# ---- errors and exports --------------------------------------------------------------------------------
def test_errors(gpu_ctx):
    from pixo_b200 import PixoError, _lib, png
    img = make_quantize_input("pal", 4, 4, 4, 1, 16)
    lib = _lib.load()
    info = png._Reduced()
    out = np.empty(4096, np.uint8)
    n = C.c_size_t()
    pal = np.zeros((300, 4), np.uint8)

    def call(data=img, w=4, h=4, ct=3, word=6 | 0x1000, mc=256, p=None, plen=0, cap=out.size):
        return lib.pixo_b200_png_quantize_filter(gpu_ctx.handle, data.ctypes.data, data.size, w, h, ct, word, mc,
                                                 None if p is None else p.ctypes.data, plen, C.byref(info),
                                                 out.ctypes.data, cap, C.byref(n), None)
    assert call() == 0 and info.color_type_byte == 3
    assert call(word=6 | 0x800 | 0x1000) == _lib.ERR_INVALID_ARGUMENT      # Auto and Force together
    assert call(word=6 | 0x4000) == _lib.ERR_INVALID_ARGUMENT               # unknown flag
    assert call(word=9 | 0x1000) == _lib.ERR_INVALID_ARGUMENT               # unknown strategy
    assert call(mc=70000) == _lib.ERR_INVALID_ARGUMENT                      # max_colors is a u16
    assert call(p=pal, plen=257) == _lib.ERR_INVALID_ARGUMENT
    assert call(p=pal, plen=0) == _lib.ERR_INVALID_ARGUMENT
    assert call(plen=3) == _lib.ERR_INVALID_ARGUMENT
    assert call(w=5) == _lib.ERR_INVALID_DATA_LENGTH
    assert call(w=0) == _lib.ERR_INVALID_DIMENSIONS
    assert call(w=(1 << 24) + 1, h=1) == _lib.ERR_IMAGE_TOO_LARGE
    assert call(ct=4) == _lib.ERR_UNSUPPORTED_COLOR
    assert call(cap=3) == _lib.ERR_OUTPUT_TOO_SMALL and n.value == 4 * (4 + 1)
    # the existing entry points keep rejecting the new flags
    for flag in (0x800, 0x1000, 0x2000):
        assert lib.pixo_b200_png_filter(gpu_ctx.handle, img.ctypes.data, 4, 4, 16, 4, 6 | flag, out.ctypes.data,
                                        None) == _lib.ERR_INVALID_ARGUMENT
        assert lib.pixo_b200_png_reduce_filter(gpu_ctx.handle, img.ctypes.data, img.size, 4, 4, 3, 6 | flag,
                                               C.byref(info), out.ctypes.data, out.size, C.byref(n),
                                               None) == _lib.ERR_INVALID_ARGUMENT
    # a _dev palette length above 256
    lens = np.array([257], np.uint32)
    pals = np.zeros((1, 256, 4), np.uint8)
    with pytest.raises(PixoError):
        _lib.check(gpu_ctx.handle, lib.pixo_b200_png_quantize_filter_dev(
            gpu_ctx.handle, 16, 64, 1, 4, 4, 3, 6 | 0x1000, 256, pals.ctypes.data, lens.ctypes.data, C.byref(info),
            16, 80, None))


def test_exports(lib):
    for name in ("pixo_b200_png_quantize_filter", "pixo_b200_png_quantize_filter_dev"):
        assert hasattr(lib, name)
