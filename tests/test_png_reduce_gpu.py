"""The CUDA colour-type / palette reduction (pixo_b200_png_reduce_filter[_dev]) against real pixo output
(tests/golden/reduce/ and the tiny reduced fixtures of tests/golden/) with no oracle in between, and
against oracle/png_reduce.py for flag combinations pixo's wasm API cannot produce, full-size frames and
batches."""
import os

import numpy as np
import pytest

from oracle import png_reduce as pr
from reduce_inputs import GOLD, load_manifest, make_reduce_input, png_parts, skipped_golden_cases
from test_png_reduce import expect_matches, golden_case_input, reduce_case_input

pytestmark = pytest.mark.gpu

MANIFEST = load_manifest()
SKIPPED = skipped_golden_cases()


def _product(ctx, img, w, h, ct, preset=None, strategy=6, rct=False, rpal=False, oa=False):
    from pixo_b200 import ColorType, png
    from pixo_b200.png import FilterStrategy, PngOptions
    if preset is not None:
        o = png.PngOptions.from_preset(w, h, preset)
        o.color_type = ColorType(ct)
    else:
        o = PngOptions(w, h, ColorType(ct), FilterStrategy(strategy), oa, rct, rpal)
    return png.reduce_and_filter(img, o, ctx=ctx)


def _oracle(po, img, w, h, ct, strategy, rct, rpal, oa):
    red = pr.reduce(img, w, h, ct, rct, rpal)
    f = po.apply_filters(pr.filter_input(red, oa), w, h, red.bytes_per_pixel, strategy, row_bytes=red.row_bytes)
    return red, f, po.adler32(f)


def _same(red, want, f, wf, ad, wad):
    assert (red.color_type_byte, red.bit_depth, red.bytes_per_pixel, red.row_bytes) == \
        (want.color_type_byte, want.bit_depth, want.bytes_per_pixel, want.row_bytes)
    assert int(red.effective_color_type) == want.effective_color_type
    if want.palette is None:
        assert red.palette is None
    else:
        assert np.array_equal(red.palette, want.palette) and red.trns == want.trns
    assert np.array_equal(np.asarray(f), wf) and ad == wad


# ---- real pixo output ---------------------------------------------------------------------------------
@pytest.mark.parametrize("c", MANIFEST["png"], ids=lambda c: c["file"])
def test_gpu_reproduces_pixo_reduction(gpu_ctx, c):
    img = reduce_case_input(c)
    parts = png_parts(open(os.path.join(GOLD, "reduce", c["file"]), "rb").read())
    red, f, ad = _product(gpu_ctx, img, c["w"], c["h"], c["ct"], preset=c["preset"])
    assert red.trns == parts["tRNS"]
    expect_matches(parts, red, f, ad, c)


@pytest.mark.parametrize("c", SKIPPED, ids=lambda c: c["file"])
def test_gpu_reproduces_reduced_golden_fixtures(gpu_ctx, c):
    img = golden_case_input(c)
    parts = png_parts(open(os.path.join(GOLD, c["file"]), "rb").read())
    red, f, ad = _product(gpu_ctx, img, c["w"], c["h"], c["ct"], preset=c["preset"])
    expect_matches(parts, red, f, ad, c)


# ---- flag combinations, against the oracle -------------------------------------------------------------
FLAG_CASES = []
for ct in (0, 1, 2, 3):
    for kind, n in (("graypal", 2), ("graypal", 4), ("graypal", 16), ("graypal", 200), ("pal", 5), ("pal", 40),
                    ("noise", 0), ("opaque", 0), ("grayalpha", 0)):
        if ct < 2 and kind != "noise":
            continue
        if kind in ("opaque", "grayalpha") and ct != 3:
            continue
        FLAG_CASES.append((ct, kind, n))


@pytest.mark.parametrize("rct,rpal", [(False, True), (True, False), (True, True), (False, False)],
                         ids=["palette", "colortype", "both", "neither"])
@pytest.mark.parametrize("ct,kind,n", FLAG_CASES)
def test_flag_combinations_match_oracle(po, gpu_ctx, ct, kind, n, rct, rpal):
    w, h = 37, 23
    img = make_reduce_input(kind, w, h, ct + 1, 5, n)
    for st, oa in ((6, True), (4, False)):
        red, f, ad = _product(gpu_ctx, img, w, h, ct, strategy=st, rct=rct, rpal=rpal, oa=oa)
        want, wf, wad = _oracle(po, img, w, h, ct, st, rct, rpal, oa)
        _same(red, want, f, wf, ad, wad)


def test_gray_bit_depths(po, gpu_ctx):
    """RGB gray -> Gray at 1, 2, 4 and 8 bits, and opaque gray RGBA -> Gray (colour type only)."""
    depths = set()
    for ct in (2, 3):
        for n in (2, 4, 16, 17, 256):
            w, h = 45, 19
            img = make_reduce_input("graypal", w, h, ct + 1, n, n)
            red, f, ad = _product(gpu_ctx, img, w, h, ct, rct=True)
            want, wf, wad = _oracle(po, img, w, h, ct, 6, True, False, False)
            _same(red, want, f, wf, ad, wad)
            assert red.color_type_byte == 0
            depths.add(red.bit_depth)
    assert depths == {1, 2, 4, 8}


# ---- the hash sets ------------------------------------------------------------------------------------
def _keys_image(keys, w, h, seed=0):
    """RGBA image of the given 32-bit keys (r<<24|g<<16|b<<8|a), each present, scattered."""
    keys = np.asarray(keys, np.uint32)
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, keys.size, w * h)
    idx[rng.permutation(w * h)[:keys.size]] = np.arange(keys.size)
    k = keys[idx]
    return np.stack([(k >> s) & 255 for s in (24, 16, 8, 0)], 1).astype(np.uint8).reshape(-1)


@pytest.mark.parametrize("name", ["alpha_only", "red_only", "transparent_black", "alpha_257"])
def test_hash_set_stress(po, gpu_ctx, name):
    w, h = 300, 200
    if name == "alpha_only":
        keys = (0x12345600 | np.arange(256)).astype(np.uint32)
    elif name == "red_only":
        keys = ((np.arange(256) << 24) | 0x00808080 | 255).astype(np.uint32)
    elif name == "transparent_black":
        keys = np.array([0, 0x000000FF, 0xFFFFFFFF, 0xFFFFFF00, 0x01020304], np.uint32)
    else:
        keys = np.concatenate([(0xABCDEF00 | np.arange(256)), [0x00000001]]).astype(np.uint32)
    img = _keys_image(keys, w, h)
    red, f, ad = _product(gpu_ctx, img, w, h, 3, rct=True, rpal=True, oa=True)
    want, wf, wad = _oracle(po, img, w, h, 3, 6, True, True, True)
    _same(red, want, f, wf, ad, wad)
    assert (red.palette is None) == (keys.size > 256)


def test_257th_colour_in_the_last_pixel_of_a_4k_frame(po, gpu_ctx):
    w, h = 3840, 2160
    img = _keys_image((np.arange(256) * 0x01010101).astype(np.uint32) | 255, w, h, 3).reshape(-1, 4)
    img[-1] = (1, 2, 3, 4)
    red, f, ad = _product(gpu_ctx, img.reshape(-1), w, h, 3, rct=True, rpal=True, oa=True)
    assert red.palette is None and red.color_type_byte == 6
    img[-1] = img[0]
    red, f, ad = _product(gpu_ctx, img.reshape(-1), w, h, 3, rct=True, rpal=True, oa=True)
    want, wf, wad = _oracle(po, img.reshape(-1), w, h, 3, 6, True, True, True)
    _same(red, want, f, wf, ad, wad)
    assert len(red.palette) == 256


def test_colour_seen_by_one_cta_only(po, gpu_ctx):
    """Colours that only the CTA of one stretch of the frame sees still reach the image's set."""
    w, h = 1024, 512
    img = np.zeros((h * w, 3), np.uint8)
    img[:] = (10, 20, 30)
    img[300_000:300_010] = (200, 100, 50)      # inside one analysis CTA's run
    img[-5:] = (1, 1, 1)
    red, f, ad = _product(gpu_ctx, img.reshape(-1), w, h, 2, rct=True, rpal=True)
    want, wf, wad = _oracle(po, img.reshape(-1), w, h, 2, 6, True, True, False)
    _same(red, want, f, wf, ad, wad)
    assert len(red.palette) == 3


# ---- full size, batched, through the device entry point ----------------------------------------------
def _run_dev(ctx, frames, w, h, ct, opts, in_stride=None, out_stride=None):
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
    infos = png.reduce_and_filter_dev(d_in, in_stride, n, opts, d_out, out_stride, d_ad, ctx=ctx)
    ctx.sync()
    outs = [d_out[i * out_stride:i * out_stride + h * (infos[i].row_bytes + 1)].cpu().numpy() for i in range(n)]
    return infos, outs, [int(a) & 0xFFFFFFFF for a in d_ad.cpu().numpy()]


def test_4k_batch_matches_oracle(po, gpu_ctx):
    from pixo_b200 import ColorType
    from pixo_b200.png import PngOptions
    w, h = 3840, 2160
    frames = [make_reduce_input("palblk", w, h, 4, 1, 200), make_reduce_input("pal", w, h, 4, 2, 256),
              make_reduce_input("pal", w, h, 4, 3, 257), make_reduce_input("opaque", w, h, 4, 4),
              make_reduce_input("grayalpha", w, h, 4, 5), make_reduce_input("noise", w, h, 4, 6)]
    opts = PngOptions.from_preset(w, h, 1)
    opts.color_type = ColorType.Rgba
    infos, outs, ads = _run_dev(gpu_ctx, frames, w, h, 3, opts)
    kinds = []
    for fr, red, f, ad in zip(frames, infos, outs, ads):
        want, wf, wad = _oracle(po, fr, w, h, 3, 6, True, True, True)
        _same(red, want, f, wf, ad, wad)
        kinds.append(red.color_type_byte)
    assert kinds == [3, 3, 6, 2, 4, 6]


def test_offsets_beyond_4_gib(po, gpu_ctx):
    """Input and output strides that put the last frames past 2^32 bytes."""
    from pixo_b200 import ColorType
    from pixo_b200.png import FilterStrategy, PngOptions
    w, h = 256, 128
    frames = [make_reduce_input("pal", w, h, 4, 7, 17), make_reduce_input("grayalpha", w, h, 4, 8),
              make_reduce_input("pal", w, h, 4, 9, 3)]
    stride = (1 << 31) + 4096
    opts = PngOptions(w, h, ColorType.Rgba, FilterStrategy.Paeth, True, True, True)
    infos, outs, ads = _run_dev(gpu_ctx, frames, w, h, 3, opts, in_stride=stride, out_stride=stride)
    for fr, red, f, ad in zip(frames, infos, outs, ads):
        want, wf, wad = _oracle(po, fr, w, h, 3, 4, True, True, True)
        _same(red, want, f, wf, ad, wad)


# ---- errors --------------------------------------------------------------------------------------------
def test_errors(gpu_ctx):
    import ctypes as C
    from pixo_b200 import PixoError, _lib, png
    from pixo_b200.png import PngOptions
    img = np.zeros(4 * 4 * 4, np.uint8)
    for w, h, code in ((0, 4, _lib.ERR_INVALID_DIMENSIONS), (4, 0, _lib.ERR_INVALID_DIMENSIONS),
                       ((1 << 24) + 1, 1, _lib.ERR_IMAGE_TOO_LARGE), (5, 4, _lib.ERR_INVALID_DATA_LENGTH)):
        with pytest.raises(PixoError) as e:
            png.reduce_and_filter(img, PngOptions(w, h, 3, 6, True, True, True), ctx=gpu_ctx)
        assert e.value.code == code
    lib = _lib.load()
    info = png._Reduced()
    out = np.empty(4096, np.uint8)
    n = C.c_size_t()
    for ct, word, code in ((4, 6, _lib.ERR_UNSUPPORTED_COLOR), (3, 9, _lib.ERR_INVALID_ARGUMENT),
                           (3, 6 | 0x800, _lib.ERR_INVALID_ARGUMENT), (3, 6 | 0x80000000, _lib.ERR_INVALID_ARGUMENT)):
        rc = lib.pixo_b200_png_reduce_filter(gpu_ctx.handle, img.ctypes.data, img.size, 4, 4, ct, word, C.byref(info),
                                             out.ctypes.data, out.size, C.byref(n), None)
        assert rc == code
    # too small an output reports the size it needs
    rc = lib.pixo_b200_png_reduce_filter(gpu_ctx.handle, img.ctypes.data, img.size, 4, 4, 3, 0x600 | 6, C.byref(info),
                                         out.ctypes.data, 3, C.byref(n), None)
    assert rc == _lib.ERR_OUTPUT_TOO_SMALL and n.value == 4 * (1 + 1)
    # the filter entry points keep rejecting the reduce flags
    for flag in (0x200, 0x400):
        rc = lib.pixo_b200_png_filter(gpu_ctx.handle, img.ctypes.data, 4, 4, 16, 4, 6 | flag, out.ctypes.data, None)
        assert rc == _lib.ERR_INVALID_ARGUMENT
