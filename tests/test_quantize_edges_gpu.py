"""The PNG quantiser (png_quantize.cu, png_host.cpp) on inputs built at its decision edges (tests/quantize_edge_inputs.py):
tied and near-missed palette distances at every lane split and palette size, on the table, the translucent search,
the early out's misses and the dither; every table cell and every opaque colour; k-means and median cut ties; the Auto
and early-out thresholds at each sampler stride; 8 192 against 8 193 histogram colours; batches across the 64-image
sort chunk; dither errors at full scale.  Each case runs through quantize_and_filter, quantize_and_filter_dev (at a
16-byte-aligned base and at an offset of 1) and, one per family, png.encode.  Palettes, tRNS, index rows, Adler-32,
decisions and refusals are compared with tests/quantize_ref.py, which test_quantize_edges.py holds equal to the
oracle on every case; the whole-table and every-colour images are compared with the C oracle."""
import zlib

import numpy as np
import pytest

import png_encode_ref as E
import quantize_edge_inputs as I
import quantize_ref as R
from oracle import png_quantize as pq
from test_dev_layouts_lossy_gpu import DITHER, QAUTO, QFORCE, png_dev

pytestmark = pytest.mark.gpu

FAMILIES = ["tie", "sweep", "early", "kmeans", "cut", "decision", "dither"]
LAYOUTS = [(0, 0, 0, 0), (1, 0, 1, 0)]        # frame at a 16-byte-aligned base, then at an offset of 1


@pytest.fixture(autouse=True)
def no_host_fallback(gpu_ctx):
    """No frame of this file is finished by host code."""
    from pixo_b200 import _lib
    yield
    assert _lib.load().pixo_b200_ctx_host_fallbacks(gpu_ctx.handle) == 0


@pytest.fixture(scope="module")
def cases():
    fams = {"tie": I.tie_cases, "sweep": I.sweep_cases, "early": I.early_cases, "kmeans": I.kmeans_cases,
            "cut": I.cut_cases, "decision": I.decision_cases, "dither": I.dither_cases}
    out = {}
    for fam, make in fams.items():
        out[fam] = []
        for c in make():
            try:
                out[fam].append((c, c.run()))
            except R.Refused:
                out[fam].append((c, "refused"))
    return out


def _opts(c, strategy=0):
    from pixo_b200 import ColorType
    from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode
    mode = QuantizationMode.Force if c.mode == "force" else QuantizationMode.Auto
    return PngOptions(c.w, c.h, ColorType(c.ct), FilterStrategy(strategy), quantization_mode=mode, max_colors=c.m,
                      dithering=c.dither, compression_level=6)


def _word(c):
    return (QFORCE if c.mode == "force" else QAUTO) | (DITHER if c.dither else 0)


def _same(c, want, red, f, ad):
    if want == "refused":
        raise AssertionError(f"{c.name}: not refused")
    f = np.asarray(f)
    if want.kind == "lossless":
        assert red.color_type_byte != 3 and red.palette is None, c.name
        assert len(f) == c.h * (c.w * (c.ct + 1) + 1), c.name
    else:
        assert (red.color_type_byte, red.bit_depth, red.bytes_per_pixel) == (3, 8, 1), c.name
        assert np.array_equal(red.palette, want.palette), c.name
        assert red.trns == R.trimmed_trns(want.palette), c.name
        rows = f.reshape(c.h, c.w + 1)
        assert (rows[:, 0] == 0).all(), c.name
        got = rows[:, 1:].reshape(-1)
        assert np.array_equal(got, want.indices), (c.name, np.flatnonzero(got != want.indices)[:5])
    assert int(ad) & 0xFFFFFFFF == zlib.adler32(f.tobytes()), c.name


@pytest.mark.parametrize("family", FAMILIES)
def test_host_entry_point(gpu_ctx, cases, family):
    """png.quantize_and_filter: every case"""
    from pixo_b200 import PixoError, _lib, png
    for c, want in cases[family]:
        if want == "refused":
            with pytest.raises(PixoError) as e:
                png.quantize_and_filter(c.data, _opts(c), palette=c.palette, ctx=gpu_ctx)
            assert e.value.code == _lib.ERR_UNSUPPORTED and "8192" in str(e.value), c.name
            continue
        red, f, ad = png.quantize_and_filter(c.data, _opts(c), palette=c.palette, ctx=gpu_ctx)
        _same(c, want, red, f, ad)


@pytest.mark.parametrize("family", FAMILIES)
def test_device_entry_point(gpu_ctx, cases, family):
    """png.quantize_and_filter_dev through the C ABI, one frame per call at each layout, guards around the output"""
    from pixo_b200 import PixoError, _lib
    fn = _lib.load().pixo_b200_png_quantize_filter_dev
    for c, want in cases[family]:
        pals = np.zeros((1, 256, 4), np.uint8)
        lens = np.zeros(1, np.uint32)
        if c.palette is not None:
            pals[0, :len(c.palette)], lens[0] = c.palette, len(c.palette)
        extra = (c.m, pals.ctypes.data if c.palette is not None else None,
                 lens.ctypes.data if c.palette is not None else None)
        for layout in LAYOUTS:
            if want == "refused":
                with pytest.raises(PixoError) as e:
                    png_dev(gpu_ctx, fn, [c.data], c.w, c.h, c.ct, _word(c), layout, *extra)
                assert e.value.code == _lib.ERR_UNSUPPORTED, c.name
                continue
            reds, outs, ads = png_dev(gpu_ctx, fn, [c.data], c.w, c.h, c.ct, _word(c), layout, *extra)
            _same(c, want, reds[0], outs[0], ads[0])


def test_encode_one_case_per_family(gpu_ctx, cases):
    """png.encode: whole files, byte for byte, for the first case of each family that quantises"""
    from pixo_b200 import png
    for fam in FAMILIES:
        c, want = next((c, w) for c, w in cases[fam] if w != "refused" and w.kind != "lossless")
        o = _opts(c, strategy=4)
        assert png.encode(c.data, o, palette=c.palette, ctx=gpu_ctx) == \
            E.encode(c.data, o, palette=c.palette, parallel_feature=True), c.name


@pytest.mark.parametrize("n", [63, 64, 65, 128, 129])
def test_batches_across_the_sort_chunk(gpu_ctx, n):
    """n frames in one Auto call that share colours, holding 4 and 5 of them in turn: frame i quantises exactly when
    it is odd, whichever 64-image sort chunk and key bits it falls in"""
    from pixo_b200 import _lib
    frames = I.batch_frames(n)
    w, h = 16, 8
    c = I.Case("batch", w, h, 2, frames[0], mode="auto", m=4, dither=True)
    fn = _lib.load().pixo_b200_png_quantize_filter_dev
    reds, outs, ads = png_dev(gpu_ctx, fn, frames, w, h, 2, _word(c), LAYOUTS[0], 4, None, None)
    for i, f in enumerate(frames):
        c.data = f
        want = c.run()
        assert (want.kind != "lossless") == (i % 2 == 1)
        _same(c, want, reds[i], outs[i], ads[i])


def _oracle_rows(img, w, h, pal, dither):
    return pq.map_indices(img, w, h, 2, pal, dither, False)


@pytest.mark.parametrize("name", ["sweep", "random256", "bw"])
def test_every_table_cell(gpu_ctx, name):
    """512 x 512 RGB holding each 6-6-6 cell's colour once: the index rows are the whole table"""
    from pixo_b200 import png
    pal = I.table_palettes()[name]
    img = I.all_cells()
    c = I.Case("cells", 512, 512, 2, img, palette=pal)
    red, f, ad = png.quantize_and_filter(img, _opts(c), palette=pal, ctx=gpu_ctx)
    want = R.Result("given", palette=pal, indices=_oracle_rows(img, 512, 512, pal, False))
    _same(c, want, red, f, ad)


@pytest.mark.parametrize("name,dither", [("sweep", False), ("random256", False), ("bw", False), ("random256", True),
                                         ("bw", True)])
def test_every_opaque_colour(gpu_ctx, name, dither):
    """4096 x 4096 RGB holding every opaque colour once, mapped and dithered"""
    from pixo_b200 import png
    pal = I.table_palettes()[name]
    img = I.all_colours()
    c = I.Case("colours", 4096, 4096, 2, img, dither=dither, palette=pal)
    red, f, ad = png.quantize_and_filter(img, _opts(c), palette=pal, ctx=gpu_ctx)
    want = R.Result("given", palette=pal, indices=_oracle_rows(img, 4096, 4096, pal, dither))
    _same(c, want, red, f, ad)
