"""The exact number of kernel launches (pixo_b200_ctx_launch_count) each public entry point makes on one
small fixed input, for each of its branches.  The count is public: a change in how launches are made
or counted must not change it."""
import os

import numpy as np
import pytest

import pixo_b200
from pixo_b200 import ColorType, jpeg, parallel, png, synthetic
from pixo_b200 import resize as rs
from pixo_b200.jpeg import JpegOptions, Subsampling
from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode

pytestmark = pytest.mark.gpu

W, H = 96, 64


def rgb():
    img = synthetic.gradient_rgb(W, H).reshape(H, W, 3).astype(np.int32)
    img += np.random.default_rng(1).integers(-12, 13, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8).reshape(-1)


def gray():
    return rgb().reshape(-1, 3)[:, 1].copy()


def rgba(w=W, h=H):
    img = synthetic.gradient_rgb(w, h).reshape(h, w, 3)
    alpha = np.full((h, w, 1), 255, np.uint8)
    alpha[: h // 4] = 128
    return np.concatenate([img, alpha], -1).reshape(-1)


def palette_image():
    pal = np.array([[200, 10, 10, 255], [10, 200, 10, 255], [10, 10, 200, 128], [0, 0, 0, 0], [9, 9, 9, 255]], np.uint8)
    idx = (np.arange(H)[:, None] // 5 + np.arange(W)[None, :] // 7) % 5
    return pal[idx].reshape(-1)


class segments:
    """PIXO_B200_SEGMENTS for the calls inside the block."""

    def __init__(self, n):
        self.n = n

    def __enter__(self):
        self.old = os.environ.get("PIXO_B200_SEGMENTS")
        os.environ["PIXO_B200_SEGMENTS"] = str(self.n)

    def __exit__(self, *a):
        if self.old is None:
            del os.environ["PIXO_B200_SEGMENTS"]
        else:
            os.environ["PIXO_B200_SEGMENTS"] = self.old


def coefficients(ctx, ct=ColorType.Rgb, ss=Subsampling.S420):
    import torch
    y, cb, cr = jpeg.compute_all_coefficients(gray() if ct == ColorType.Gray else rgb(), W, H, ct, ss, 80, ctx=ctx)
    d = [torch.from_numpy(np.ascontiguousarray(a if len(a) else np.zeros((1, 64), np.int16))).cuda() for a in (y, cb, cr)]
    torch.cuda.synchronize()
    return d, len(y), len(cb)


def entropy_dev(ctx, ct, ss, opt, nseg=None):
    d, _, _ = coefficients(ctx, ct, ss)
    o = JpegOptions(W, H, ct, 80, ss, None, opt)
    chroma = ct != ColorType.Gray
    if nseg is None:
        return lambda: jpeg.entropy_encode_dev(d[0], d[1] if chroma else None, d[2] if chroma else None, o, ctx=ctx)

    def call():
        with segments(nseg):
            jpeg.entropy_encode_dev(d[0], d[1], d[2], o, ctx=ctx)
    return call


def band(ctx, stage, nseg=None):
    d, ny, nc = coefficients(ctx)
    coder = parallel.DeviceBandCoder(ctx, d[0], d[1], d[2], W, H, ColorType.Rgb, Subsampling.S420, ny, nc)
    seed = np.zeros(3, np.int32)

    def entropy():
        if nseg is None:
            return coder.entropy(seed, None)
        with segments(nseg):
            return coder.entropy(seed, None)
    if stage == "histogram":
        return lambda: coder.histogram(seed)
    if stage == "entropy":
        return entropy
    nbits, tail = entropy()
    return lambda: coder.splice(nbits, 0, 0, True)


def trellis_dev(ctx):
    import torch
    dct = torch.from_numpy(np.random.default_rng(2).normal(0, 60, (300, 64)).astype(np.float32)).cuda()
    q = jpeg.quant_tables(80)[2]
    return lambda: jpeg.trellis_quantize_dev(dct, q, 1.0, ctx=ctx)


def progressive_dev(ctx):
    d, _, _ = coefficients(ctx)
    return lambda: jpeg.progressive_scans_dev(*d, W, H, ctx=ctx)


def filt(strategy, w=W, h=H, oa=False):
    img = rgba(w, h)
    o = PngOptions(w, h, ColorType.Rgba, strategy, oa)
    return lambda ctx: (lambda: png.apply_filters(img, w, h, 4, o, with_adler=True, ctx=ctx))


def reduce(img, preset=1):
    return lambda ctx: (lambda: png.reduce_and_filter(img, PngOptions.from_preset(W, H, preset), ctx=ctx))


def quantize(dither, mode=QuantizationMode.Force, colors=16):
    img = rgba()
    o = PngOptions(W, H, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, mode, colors, dither)
    return lambda ctx: (lambda: png.quantize_and_filter(img, o, ctx=ctx))


def resize(alg, ct=ColorType.Rgba, dst=(57, 41)):
    img = rgba() if ct == ColorType.Rgba else gray()
    o = rs.ResizeOptions.builder(W, H).dst(*dst).color_type(ct).algorithm(alg).build()
    return lambda ctx: (lambda: rs.resize(img, o, ctx=ctx))


def jpeg_encode(ct, ss, opt=False, ri=None, trellis=False):
    data = gray() if ct == ColorType.Gray else rgb()
    o = JpegOptions(W, H, ct, 80, ss, ri, opt, False, trellis)
    return lambda ctx: (lambda: jpeg.encode(data, o, ctx=ctx))


def coef(ct, ss, **kw):
    data = gray() if ct == ColorType.Gray else rgb()
    return lambda ctx: (lambda: jpeg.compute_all_coefficients(data, W, H, ct, ss, 80, ctx=ctx, **kw))


def progressive(opt, trellis=True):
    o = JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420, None, opt, True, trellis)
    return lambda ctx: (lambda: jpeg.encode_progressive(rgb(), o, ctx=ctx))


# name -> ctx -> the call whose launches are counted (set-up runs outside the count)
CASES = {
    "coefficients_gray": coef(ColorType.Gray, Subsampling.S420),
    "coefficients_420": coef(ColorType.Rgb, Subsampling.S420),
    "coefficients_444": coef(ColorType.Rgb, Subsampling.S444),
    "coefficients_420_zigzag_histograms": coef(ColorType.Rgb, Subsampling.S420, zigzag=True, histograms=True),
    "coefficients_420_trellis": coef(ColorType.Rgb, Subsampling.S420, use_trellis=True),
    "coefficients_gray_trellis": coef(ColorType.Gray, Subsampling.S420, use_trellis=True),
    "encode_gray": jpeg_encode(ColorType.Gray, Subsampling.S420),
    "encode_420": jpeg_encode(ColorType.Rgb, Subsampling.S420),
    "encode_444_optimized_restart": jpeg_encode(ColorType.Rgb, Subsampling.S444, True, 2),
    "encode_420_trellis": jpeg_encode(ColorType.Rgb, Subsampling.S420, True, trellis=True),
    "encode_batch_420": lambda ctx: (lambda: jpeg.encode_batch(np.stack([rgb()] * 3),
                                                               JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420),
                                                               ctx=ctx)),
    "encode_batch_420_optimized": lambda ctx: (lambda: jpeg.encode_batch(
        np.stack([rgb()] * 8), JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420, None, True), ctx=ctx)),
    "progressive": progressive(False, False),
    "progressive_optimized_trellis": progressive(True),
    "progressive_batch": lambda ctx: (lambda: jpeg.encode_progressive_batch(
        np.stack([rgb()] * 2), JpegOptions.max(W, H, 80), ctx=ctx)),
    "progressive_scans_dev": progressive_dev,
    "trellis_dev": trellis_dev,
    "entropy_dev_420": lambda ctx: entropy_dev(ctx, ColorType.Rgb, Subsampling.S420, False),
    "entropy_dev_gray_optimized": lambda ctx: entropy_dev(ctx, ColorType.Gray, Subsampling.S420, True),
    "entropy_dev_420_segments": lambda ctx: entropy_dev(ctx, ColorType.Rgb, Subsampling.S420, False, 3),
    "band_histogram": lambda ctx: band(ctx, "histogram"),
    "band_entropy": lambda ctx: band(ctx, "entropy"),
    "band_entropy_segments": lambda ctx: band(ctx, "entropy", 2),
    "band_splice": lambda ctx: band(ctx, "splice"),
    "band_splice_segments": lambda ctx: band(ctx, "splice", 2),
    "png_adaptive": filt(FilterStrategy.Adaptive),
    "png_adaptive_optimize_alpha": filt(FilterStrategy.Adaptive, oa=True),
    "png_adaptive_fast_sticky": filt(FilterStrategy.AdaptiveFast, w=160, h=32),   # over 4096 px, 32 rows
    "png_adaptive_fast": filt(FilterStrategy.AdaptiveFast),
    "png_bigrams": filt(FilterStrategy.Bigrams),
    "png_small_sub": filt(FilterStrategy.Adaptive, h=16),   # 4096 px or fewer: Sub
    "adler32": lambda ctx: (lambda: png.adler32(rgba(), ctx=ctx)),
    "reduce_palette": reduce(palette_image()),
    "reduce_gray": reduce(np.stack([gray()] * 3 + [np.full(W * H, 255, np.uint8)], -1).reshape(-1)),
    "reduce_unchanged": reduce(rgba()),
    "quantize": quantize(False),
    "quantize_dither": quantize(True),
    "quantize_auto": quantize(True, QuantizationMode.Auto, 256),
    "resize_nearest": resize(rs.ResizeAlgorithm.Nearest),
    "resize_bilinear": resize(rs.ResizeAlgorithm.Bilinear),
    "resize_lanczos3": resize(rs.ResizeAlgorithm.Lanczos3),
    "resize_lanczos3_gray": resize(rs.ResizeAlgorithm.Lanczos3, ColorType.Gray, (131, 29)),
}

# taken from the parent of the commit that moved every launch into pixo::launch
EXPECTED = {
    "adler32": 1,
    "band_entropy": 2,
    "band_entropy_segments": 2,
    "band_histogram": 1,
    "band_splice": 4,
    "band_splice_segments": 4,
    "coefficients_420": 1,
    "coefficients_420_trellis": 4,
    "coefficients_420_zigzag_histograms": 2,
    "coefficients_444": 1,
    "coefficients_gray": 1,
    "coefficients_gray_trellis": 2,
    "encode_420": 2,
    # optimised tables: K1, K3, k_huff_tables, then one k_huff per group (each frame was a k_huff of its own)
    "encode_420_trellis": 4,
    "encode_444_optimized_restart": 4,
    "encode_batch_420": 4,
    "encode_batch_420_optimized": 8,   # two groups of 4: 12 when each frame had a k_huff of its own
    "encode_gray": 2,
    "entropy_dev_420": 1,
    "entropy_dev_420_segments": 5,
    "entropy_dev_gray_optimized": 3,   # K3, k_huff_tables, k_huff
    "png_adaptive": 1,
    "png_adaptive_fast": 1,
    "png_adaptive_fast_sticky": 2,
    "png_adaptive_optimize_alpha": 1,
    "png_bigrams": 1,
    "png_small_sub": 1,
    # progressive scans: k_prog_place and k_seg_fit in, k_prog_pack out (one splice per frame string, written
    # straight into the slot): 10, 32, 16 and 10 with a string per scan and a copy out of a stage buffer
    "progressive": 12,
    "progressive_batch": 36,               # k_huff_tables once per group (two groups of one)
    "progressive_optimized_trellis": 18,   # k_huff_tables after K3
    "progressive_scans_dev": 11,
    "quantize": 8,
    "quantize_auto": 8,
    "quantize_dither": 8,
    "reduce_gray": 4,
    "reduce_palette": 4,
    "reduce_unchanged": 2,
    "resize_bilinear": 1,
    "resize_lanczos3": 2,
    "resize_lanczos3_gray": 2,
    "resize_nearest": 1,
    "trellis_dev": 1,
}


def count(ctx, name):
    call = CASES[name](ctx)
    ctx.sync()
    l0 = ctx.launch_count
    call()
    ctx.sync()
    return ctx.launch_count - l0


@pytest.mark.parametrize("name", sorted(CASES))
def test_launch_count(gpu_ctx, name):
    assert count(gpu_ctx, name) == EXPECTED[name]


def test_launch_count_on_a_fresh_context():
    """A context's first calls set kernel attributes; they launch no more than later calls do."""
    with pixo_b200.Context(0) as ctx:
        for name in ("coefficients_444", "encode_420_trellis", "png_bigrams", "png_adaptive", "reduce_palette",
                     "quantize_dither"):
            assert count(ctx, name) == EXPECTED[name], name
