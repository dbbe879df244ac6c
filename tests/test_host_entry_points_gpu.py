"""Each host-buffer entry point against its device twin on the same frame: the host call stages the
frame into the context's scratch, runs the `_dev` entry point and copies the results back to the
caller's ordinary (pageable) numpy memory.  The frames are large enough that both copies take the
pinned paths (input of 4 MiB or more through the staging ring, results of 1 MiB or more through the
pinned buffer and the host pool), so a piece copied out of place or left out cannot pass."""
import zlib

import numpy as np
import pytest
import torch

from pixo_b200 import ColorType, _lib, jpeg, png
from pixo_b200 import resize as rs
from pixo_b200.jpeg import Subsampling
from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode

pytestmark = pytest.mark.gpu

MIB = 1 << 20


def frame(w, h, bpp, seed):
    """Noise on a gradient: too many colours for a palette, coefficients of every size."""
    rng = np.random.default_rng(seed)
    x = np.arange(w)[None, :, None] * 3 + np.arange(h)[:, None, None] + np.arange(bpp)[None, None, :] * 50
    return ((x + rng.integers(0, 40, (h, w, bpp))) & 255).astype(np.uint8).reshape(-1)


def few_colours(w, h, n, seed):
    """RGBA pixels of n colours: quantisation designs its palette from at most 8192 of them."""
    rng = np.random.default_rng(seed)
    colours = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    return colours[rng.integers(0, n, w * h)].reshape(-1)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_dev(ctx, fn, *args):
    """The library works on its own stream: torch's uploads must have landed, and its results must have."""
    torch.cuda.synchronize()
    _lib.check(ctx.handle, fn(ctx.handle, *args))
    ctx.sync()


def assert_same_info(a, b):
    assert (a.color_type_byte, a.bit_depth, a.effective_color_type, a.bytes_per_pixel, a.row_bytes, a.trns) == \
        (b.color_type_byte, b.bit_depth, b.effective_color_type, b.bytes_per_pixel, b.row_bytes, b.trns)
    assert (a.palette is None) == (b.palette is None)
    if a.palette is not None:
        assert np.array_equal(a.palette, b.palette)


@pytest.mark.parametrize("ct,ss,trellis,hist", [
    (ColorType.Rgb, Subsampling.S444, False, True),
    (ColorType.Rgb, Subsampling.S420, True, False),
    (ColorType.Gray, Subsampling.S420, False, True),
])
def test_jpeg_coefficients(gpu_ctx, ct, ss, trellis, hist):
    w, h = (1536, 1024) if ct == ColorType.Rgb else (2048, 2048)
    bpp = 3 if ct == ColorType.Rgb else 1
    px = frame(w, h, bpp, 1)
    assert px.size >= 4 * MIB
    got = jpeg.compute_all_coefficients(px, w, h, ct, ss, 85, histograms=hist, use_trellis=trellis, ctx=gpu_ctx)
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    assert ny * 128 >= MIB
    _, _, lum, chr_ = jpeg.quant_tables(85)
    lum, chr_ = np.ascontiguousarray(lum, np.float32), np.ascontiguousarray(chr_, np.float32)
    d_px, d_y = dev(px), torch.zeros((ny, 64), dtype=torch.int16, device="cuda")
    d_cb, d_cr = (torch.zeros((max(nc, 1), 64), dtype=torch.int16, device="cuda") for _ in range(2))
    d_hist = torch.zeros(536, dtype=torch.int64, device="cuda") if hist else None
    run_dev(gpu_ctx, _lib.load().pixo_b200_jpeg_coefficients_dev, d_px.data_ptr(), px.size, 1, w, h, int(ct), int(ss),
            lum.ctypes.data_as(_lib.f32p), chr_.ctypes.data_as(_lib.f32p), d_y.data_ptr(), ny * 64,
            d_cb.data_ptr() if nc else None, d_cr.data_ptr() if nc else None, nc * 64,
            jpeg.COEF_TRELLIS if trellis else 0, d_hist.data_ptr() if hist else None)
    assert np.array_equal(got[0], d_y.cpu().numpy())
    assert np.array_equal(got[1], d_cb.cpu().numpy()[:nc])
    assert np.array_equal(got[2], d_cr.cpu().numpy()[:nc])
    if hist:
        assert got[3].sum() > 0
        assert np.array_equal(got[3], d_hist.cpu().numpy().view(np.uint64))


@pytest.mark.parametrize("strategy", [FilterStrategy.Adaptive, FilterStrategy.Bigrams])
def test_png_filter(gpu_ctx, strategy):
    w, h, bpp = 1024, 1024, 4
    px = frame(w, h, bpp, 2)
    out, adler = png.apply_filters(px, w, h, bpp, PngOptions(w, h, ColorType.Rgba, strategy), with_adler=True,
                                   ctx=gpu_ctx)
    n = h * (w * bpp + 1)
    d_out, d_adler = torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    d_px = dev(px)
    run_dev(gpu_ctx, _lib.load().pixo_b200_png_filter_dev, d_px.data_ptr(), px.size, 1, w, h, w * bpp, bpp,
            int(strategy), d_out.data_ptr(), n, d_adler.data_ptr())
    assert np.array_equal(out, d_out.cpu().numpy())
    assert adler == int(d_adler.cpu().numpy().view(np.uint32)[0]) == zlib.adler32(out.tobytes())


def test_png_reduce_filter(gpu_ctx):
    w, h = 1024, 1024
    px = frame(w, h, 4, 3)
    o = PngOptions.from_preset(w, h, 1)
    info, out, adler = png.reduce_and_filter(px, o, ctx=gpu_ctx)
    assert out.size >= MIB
    n = h * (w * 4 + 1)
    d_out, d_adler = torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    d_px = dev(px)
    torch.cuda.synchronize()
    (dinfo,) = png.reduce_and_filter_dev(d_px, px.size, 1, o, d_out, n, d_adler, ctx=gpu_ctx)
    gpu_ctx.sync()
    assert_same_info(info, dinfo)
    assert np.array_equal(out, d_out.cpu().numpy()[:h * (dinfo.row_bytes + 1)])
    assert adler == int(d_adler.cpu().numpy().view(np.uint32)[0]) == zlib.adler32(out.tobytes())


@pytest.mark.parametrize("palette", [False, True])
def test_png_quantize_filter(gpu_ctx, palette):
    w, h = 1024, 1024
    px = few_colours(w, h, 3000, 4)
    o = PngOptions(w, h, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, QuantizationMode.Force, 256, True)
    pal = np.random.default_rng(5).integers(0, 256, (200, 4), dtype=np.uint8) if palette else None
    info, out, adler = png.quantize_and_filter(px, o, palette=pal, ctx=gpu_ctx)
    assert info.bit_depth == 8 and out.size >= MIB
    n = h * (w * 4 + 1)
    d_out, d_adler = torch.zeros(n, dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    d_px = dev(px)
    torch.cuda.synchronize()
    (dinfo,) = png.quantize_and_filter_dev(d_px, px.size, 1, o, d_out, n, d_adler,
                                           palettes=[pal] if palette else None, ctx=gpu_ctx)
    gpu_ctx.sync()
    assert_same_info(info, dinfo)
    assert np.array_equal(out, d_out.cpu().numpy()[:h * (dinfo.row_bytes + 1)])
    assert adler == int(d_adler.cpu().numpy().view(np.uint32)[0]) == zlib.adler32(out.tobytes())


def test_adler32(gpu_ctx):
    data = frame(1500, 1000, 3, 6)
    assert data.size >= 4 * MIB
    d_data, d_sum = dev(data), torch.zeros(1, dtype=torch.int32, device="cuda")
    run_dev(gpu_ctx, _lib.load().pixo_b200_adler32_dev, d_data.data_ptr(), data.size, d_sum.data_ptr())
    want = zlib.adler32(data.tobytes())
    assert png.adler32(data, ctx=gpu_ctx) == int(d_sum.cpu().numpy().view(np.uint32)[0]) == want


@pytest.mark.parametrize("alg", [rs.ResizeAlgorithm.Bilinear, rs.ResizeAlgorithm.Lanczos3])
def test_resize(gpu_ctx, alg):
    sw, sh, dw, dh = 1024, 1024, 900, 700
    px = frame(sw, sh, 4, 7)
    o = rs.ResizeOptions.builder(sw, sh).dst(dw, dh).color_type(ColorType.Rgba).algorithm(alg).build()
    out = rs.resize(px, o, ctx=gpu_ctx)
    assert out.size >= MIB
    d_out = torch.zeros(out.size, dtype=torch.uint8, device="cuda")
    d_px = dev(px)
    torch.cuda.synchronize()
    rs.resize_dev(d_px, px.size, 1, o, d_out, out.size, ctx=gpu_ctx)
    gpu_ctx.sync()
    assert np.array_equal(out, d_out.cpu().numpy())
