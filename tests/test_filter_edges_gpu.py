"""The PNG filter kernels on rows built at their decision edges (tests/filter_inputs.py): best scores equal to the
early-exit threshold or one above it, Paeth and Up ties, and rows whose winner is decided by the bytes at one
position of k_png_band's or k_png_filter's scoring (lane-0 and warp vector starts, the 4 096-byte iteration, the
trailing whole words, the ragged last word, the 32 KiB segment seams, transparent pixels under optimize_alpha).
Every image is compared with the oracle byte for byte, filter-type bytes included, and its Adler-32 with zlib,
through png_filter, png_filter_dev (batches, aligned and odd layouts) and png_filter_rows_dev (band cuts that are
not multiples of 16)."""
import zlib

import numpy as np
import pytest

import filter_inputs as I
from pixo_b200 import ColorType, _lib, png
from pixo_b200.png import FilterStrategy, PngOptions
from test_dev_layouts_gpu import GUARD8, GUARD32, OPTIMIZE_ALPHA, assert_guard, guarded, noise_poison, placed, run

pytestmark = pytest.mark.gpu

LAYOUTS = [(0, 0, 0, 0), (1, 1, 5, 3)]   # (input offset, input stride padding, output offset, output padding)


@pytest.fixture(scope="module")
def images():
    return {"band": I.band_images(), "row": I.row_images() + [I.longest_band_image()], "alpha": I.alpha_images(),
            "sticky": I.sticky_images(), "bigrams": I.bigram_images()}


def _ref(po, data, im, st, height=None):
    d = po.optimize_alpha(data, 1 if im.oa == 2 else 3) if im.oa else data
    return po.apply_filters(d, im.width, height or im.height, im.bpp, st, row_bytes=im.rb)


def _word(im, st):
    return st | (OPTIMIZE_ALPHA if im.oa else 0)


def _host(ctx, im, st):
    ct = {2: ColorType.GrayAlpha, 4: ColorType.Rgba}.get(im.oa, ColorType.Rgba)
    opts = PngOptions(im.width, im.height, ct, FilterStrategy(st), bool(im.oa))
    return png.apply_filters_with_row_bytes(im.data, im.width, im.height, im.rb, im.bpp, opts, with_adler=True,
                                            ctx=ctx)


def _dev(ctx, frames, im, word, layout):
    in_off, in_pad, out_off, out_pad = layout
    n, h, rb = len(frames), im.height, im.rb
    in_stride, out_len = rb * h + in_pad, h * (rb + 1)
    out_stride = out_len + out_pad
    src = placed(frames, in_off, in_stride, noise_poison(n + in_off))
    dst = guarded((n - 1) * out_stride + out_len, np.uint8, GUARD8, base=64 + out_off)
    ad = guarded(n, np.int32, GUARD32, base=4, tail=4)
    run(ctx, _lib.load().pixo_b200_png_filter_dev, src.ptr(in_off), in_stride, n, im.width, h, rb, im.bpp, word,
        dst.ptr(64 + out_off), out_stride, ad.ptr(4))
    out, ads = dst.get(), ad.get()
    o0 = 64 + out_off
    assert_guard(out, [(o0 + i * out_stride, out_len) for i in range(n)], GUARD8, f"filtered output {layout}")
    assert_guard(ads, [(4, n)], GUARD32, "d_adler")
    return [out[o0 + i * out_stride:o0 + i * out_stride + out_len] for i in range(n)], ads[4:4 + n].view(np.uint32)


def _check(got, ref, ad, what):
    assert np.array_equal(got, ref), (what, np.flatnonzero(got != ref)[:5])
    assert int(ad) == zlib.adler32(ref.tobytes()), what


@pytest.mark.parametrize("group", ["band", "row", "alpha", "sticky", "bigrams"])
def test_host_entry_point(po, gpu_ctx, images, group):
    """png_filter: every image, all nine strategies"""
    for im in images[group]:
        for st in range(9):
            got, ad = _host(gpu_ctx, im, st)
            _check(got, _ref(po, im.data, im, st), ad, (im.name, st))


@pytest.mark.parametrize("group", ["band", "row", "alpha", "sticky", "bigrams"])
def test_device_batches(po, gpu_ctx, images, group):
    """png_filter_dev: each image batched with its rows in reverse order (the same geometry, other routes), at an
    aligned layout (cp.async rows) and an odd one (staged rows), guards around every slot"""
    for im in images[group]:
        rev = im.data.reshape(im.height, im.rb)[::-1].reshape(-1).copy()
        for st in im.strategies:
            refs = [_ref(po, im.data, im, st), _ref(po, rev, im, st)]
            for layout in LAYOUTS:
                got, ads = _dev(gpu_ctx, [im.data, rev], im, _word(im, st), layout)
                for g, r, a in zip(got, refs, ads):
                    _check(g, r, a, (im.name, st, layout))


def test_row_bands(po, gpu_ctx, images):
    """png_filter_rows_dev on cuts that are not multiples of 16: band starts fall on constructed rows"""
    for im in images["band"][::3] + images["alpha"]:
        img = im.data.reshape(im.height, im.rb)
        cuts = [0, 7, 14, 23, im.height]
        for st in im.strategies:
            ref = _ref(po, im.data, im, st)
            for k, (r0, r1) in enumerate(zip(cuts, cuts[1:])):
                rows = placed([img[r0:r1].reshape(-1)], 1 + 2 * k, 0, noise_poison(k))
                above = placed([img[r0 - 1]], 5, 0, noise_poison(k + 50)) if r0 else None
                n_out = (r1 - r0) * (im.rb + 1)
                dst = guarded(n_out, np.uint8, GUARD8, base=67)
                ad = guarded(1, np.int32, GUARD32, base=4, tail=4)
                run(gpu_ctx, _lib.load().pixo_b200_png_filter_rows_dev, rows.ptr(1 + 2 * k),
                    above.ptr(5) if above else None, im.width, im.height, r1 - r0, im.rb, im.bpp, _word(im, st),
                    dst.ptr(67), ad.ptr(4))
                out, a = dst.get(), ad.get()
                assert_guard(out, [(67, n_out)], GUARD8, f"band {r0}:{r1}")
                _check(out[67:67 + n_out], ref[r0 * (im.rb + 1):r1 * (im.rb + 1)], int(a[4]) & 0xFFFFFFFF,
                       (im.name, st, r0, r1))
