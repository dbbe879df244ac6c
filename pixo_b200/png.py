"""Mirror of pixo::png's filter stage and pixo::compress::adler32 for the accelerated path.

  apply_filters / apply_filters_with_row_bytes   src/png/filter.rs:52-206
  FilterStrategy                                 src/png/mod.rs:345-364
  adler32                                        src/compress/adler32.rs:11
  reduce_and_filter[_dev]                        maybe_reduce_color_type -> maybe_optimize_alpha ->
                                                 apply_filters_with_row_bytes, src/png/mod.rs:521-568,683-1147
  quantize_and_filter[_dev]                      encode_into's quantisation branch (quantize_image ->
                                                 encode_indexed_into) or the above, src/png/mod.rs:469-511
  encode / encode_into / encode_on_device        png::encode / encode_into, whole files at the fast and balanced
                                                 presets, src/png/mod.rs:437-630
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum

import numpy as np

from . import _lib
from .color import ColorType
from .context import Context, default_context


class FilterStrategy(enum.IntEnum):
    NoFilter = 0  # FilterStrategy::None
    Sub = 1
    Up = 2
    Average = 3
    Paeth = 4
    MinSum = 5
    Adaptive = 6
    AdaptiveFast = 7
    Bigrams = 8


OPTIMIZE_ALPHA = 0x100  # PIXO_B200_PNG_OPTIMIZE_ALPHA
REDUCE_COLOR_TYPE = 0x200  # PIXO_B200_PNG_REDUCE_COLOR_TYPE
REDUCE_PALETTE = 0x400  # PIXO_B200_PNG_REDUCE_PALETTE
QUANTIZE_AUTO = 0x800  # PIXO_B200_PNG_QUANTIZE_AUTO
QUANTIZE_FORCE = 0x1000  # PIXO_B200_PNG_QUANTIZE_FORCE
DITHER = 0x2000  # PIXO_B200_PNG_DITHER
OPTIMAL_COMPRESSION = 0x4000  # PIXO_B200_PNG_OPTIMAL_COMPRESSION (the encode calls refuse it)
IDAT_CHUNK = 256 * 1024  # write_idat_chunks' chunk size, src/png/mod.rs:606-616


class QuantizationMode(enum.IntEnum):
    """pixo::png::QuantizationMode (src/png/mod.rs:70-79)."""
    Off = 0
    Auto = 1
    Force = 2


@dataclasses.dataclass
class PngOptions:
    """The fields of pixo::png::PngOptions (src/png/mod.rs:41-118) the library reads."""
    width: int = 0
    height: int = 0
    color_type: ColorType = ColorType.Rgba
    filter_strategy: FilterStrategy = FilterStrategy.Adaptive
    optimize_alpha: bool = False   # applied on the fly (Rgba / GrayAlpha), src/png/mod.rs:633-671
    reduce_color_type: bool = False  # reduce_and_filter* only, src/png/mod.rs:683-836
    reduce_palette: bool = False     # reduce_and_filter* only, src/png/mod.rs:838-900
    # QuantizationOptions (src/png/mod.rs:81-100), quantize_and_filter* only
    quantization_mode: QuantizationMode = QuantizationMode.Off
    max_colors: int = 256
    dithering: bool = False
    compression_level: int = 2          # the DEFLATE level, 1-9 (encode* only)
    optimal_compression: bool = False   # pixo's max preset; the encode calls refuse it

    @classmethod
    def from_preset(cls, width: int, height: int, preset: int) -> "PngOptions":
        """PngOptions::from_preset (src/png/mod.rs:129-197): 0 fast, 2 max, anything else balanced."""
        if preset == 0:
            return cls(width, height, ColorType.Rgba, FilterStrategy.AdaptiveFast, False, False, False,
                       compression_level=2)
        if preset == 2:
            return cls(width, height, ColorType.Rgba, FilterStrategy.Bigrams, True, True, True,
                       compression_level=9, optimal_compression=True)
        return cls(width, height, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, compression_level=6)

    @classmethod
    def from_preset_with_lossless(cls, width: int, height: int, preset: int, lossless: bool) -> "PngOptions":
        """PngOptions::from_preset_with_lossless (src/png/mod.rs:203-213): lossy selects Auto quantisation with
        dithering and 256 colours, as PngOptionsBuilder::lossy does."""
        o = cls.from_preset(width, height, preset)
        if not lossless:
            o.quantization_mode, o.max_colors, o.dithering = QuantizationMode.Auto, 256, True
        return o

    def strategy_word(self) -> int:
        """The strategy word of pixo_b200_png_reduce_filter* / quantize_filter*: strategy | flags (the
        quantisation flags only when quantisation is selected)."""
        w = (int(self.filter_strategy) | (OPTIMIZE_ALPHA if self.optimize_alpha else 0)
             | (REDUCE_COLOR_TYPE if self.reduce_color_type else 0) | (REDUCE_PALETTE if self.reduce_palette else 0))
        if self.quantization_mode == QuantizationMode.Auto:
            w |= QUANTIZE_AUTO
        elif self.quantization_mode == QuantizationMode.Force:
            w |= QUANTIZE_FORCE
        return w | (DITHER if self.dithering and self.quantization_mode != QuantizationMode.Off else 0)


class _Reduced(C.Structure):
    """pixo_b200_png_reduced (include/pixo_b200.h)."""
    _fields_ = [("color_type_byte", C.c_uint8), ("bit_depth", C.c_uint8), ("effective_color_type", C.c_uint8),
                ("bytes_per_pixel", C.c_uint8), ("palette_len", C.c_uint32), ("trns_len", C.c_uint32),
                ("reserved", C.c_uint32), ("row_bytes", C.c_uint64), ("palette", (C.c_uint8 * 4) * 256)]


@dataclasses.dataclass
class ReducedImage:
    """pixo::png's ReducedImage (src/png/mod.rs:673-680) without the rows: what IHDR, PLTE and tRNS need."""
    color_type_byte: int
    bit_depth: int
    effective_color_type: ColorType
    bytes_per_pixel: int
    row_bytes: int
    palette: np.ndarray | None   # (n, 4) uint8 RGBA in PLTE order
    trns: bytes | None           # tRNS payload (a quantised image's is trimmed after its last alpha below 255)

    @classmethod
    def _from_c(cls, r: _Reduced) -> "ReducedImage":
        n = int(r.palette_len)
        pal = np.ctypeslib.as_array(r.palette).reshape(256, 4)[:n].copy() if n else None
        trns = pal[:int(r.trns_len), 3].tobytes() if (n and r.trns_len) else None
        return cls(int(r.color_type_byte), int(r.bit_depth), ColorType(int(r.effective_color_type)),
                   int(r.bytes_per_pixel), int(r.row_bytes), pal, trns)


def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
    return np.frombuffer(data, dtype=np.uint8)


def apply_filters_with_row_bytes(data, width, height, row_bytes, bytes_per_pixel, options: PngOptions,
                                 with_adler=False, ctx: Context | None = None):
    """filter::apply_filters_with_row_bytes (src/png/filter.rs:64): filtered rows, each
    prefixed by its filter-type byte; optionally also the Adler-32 of that stream."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    if d.size != int(row_bytes) * int(height):
        raise _lib.PixoError(_lib.ERR_INVALID_DATA_LENGTH,
                             f"Invalid data length: expected {int(row_bytes) * int(height)} bytes, got {d.size}")
    out = np.empty(int(height) * (int(row_bytes) + 1), np.uint8)
    ad = C.c_uint32()
    rc = _lib.load().pixo_b200_png_filter(ctx.handle, d.ctypes.data, int(width), int(height),
                                          int(row_bytes), int(bytes_per_pixel),
                                          int(options.filter_strategy) | (OPTIMIZE_ALPHA if options.optimize_alpha else 0),
                                          out.ctypes.data,
                                          C.byref(ad) if with_adler else None)
    _lib.check(ctx.handle, rc)
    return (out, ad.value) if with_adler else out


def apply_filters(data, width, height, bytes_per_pixel, options: PngOptions, **kw):
    """filter::apply_filters (src/png/filter.rs:52)."""
    return apply_filters_with_row_bytes(data, width, height, int(width) * int(bytes_per_pixel),
                                        bytes_per_pixel, options, **kw)


def adler32(data, ctx: Context | None = None) -> int:
    """compress::adler32::adler32 (src/compress/adler32.rs:11)."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    out = C.c_uint32()
    _lib.check(ctx.handle, _lib.load().pixo_b200_adler32(ctx.handle, d.ctypes.data if d.size else None,
                                                         d.size, C.byref(out)))
    return out.value


def apply_filters_rows_dev(d_rows, d_row_above, width, image_height, band_rows, row_bytes, bytes_per_pixel,
                           strategy: FilterStrategy, d_out, d_adler=None, optimize_alpha=False,
                           ctx: Context | None = None):
    """A band of rows of one image on the device (anything with .data_ptr()): see
    pixo_b200_png_filter_rows_dev.  Asynchronous on the context's stream."""
    ctx = ctx or default_context()
    p = lambda t: None if t is None else int(t.data_ptr())
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_filter_rows_dev(
        ctx.handle, p(d_rows), p(d_row_above), int(width), int(image_height), int(band_rows), int(row_bytes),
        int(bytes_per_pixel), int(strategy) | (OPTIMIZE_ALPHA if optimize_alpha else 0), p(d_out), p(d_adler)))


def reduce_and_filter(data, options: PngOptions, ctx: Context | None = None):
    """maybe_reduce_color_type -> maybe_optimize_alpha -> apply_filters_with_row_bytes as encode_into runs
    them (src/png/mod.rs:521-568): (ReducedImage, filtered stream, its Adler-32).  See
    pixo_b200_png_reduce_filter."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    w, h = int(options.width), int(options.height)
    out = np.empty(max(h * (w * ColorType(options.color_type).bytes_per_pixel() + 1), 1), np.uint8)
    info, n, ad = _Reduced(), C.c_size_t(), C.c_uint32()
    rc = _lib.load().pixo_b200_png_reduce_filter(ctx.handle, d.ctypes.data if d.size else None, d.size, w, h,
                                                 int(options.color_type), options.strategy_word(), C.byref(info),
                                                 out.ctypes.data, out.size, C.byref(n), C.byref(ad))
    _lib.check(ctx.handle, rc)
    return ReducedImage._from_c(info), out[:n.value], ad.value


def reduce_and_filter_dev(d_data, in_stride, n_images, options: PngOptions, d_out, out_stride, d_adler=None,
                          ctx: Context | None = None):
    """Device-resident batch (anything with .data_ptr()): see pixo_b200_png_reduce_filter_dev.  Returns the
    n_images ReducedImage descriptions; the filtered streams and checksums are still being written
    asynchronously on the context's stream."""
    ctx = ctx or default_context()
    infos = (_Reduced * max(int(n_images), 1))()
    p = lambda t: None if t is None else int(t.data_ptr())
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_reduce_filter_dev(
        ctx.handle, p(d_data), int(in_stride), int(n_images), int(options.width), int(options.height),
        int(options.color_type), options.strategy_word(), infos, p(d_out), int(out_stride), p(d_adler)))
    return [ReducedImage._from_c(infos[i]) for i in range(int(n_images))]


def quantize_and_filter(data, options: PngOptions, palette=None, ctx: Context | None = None):
    """What encode_into hands DEFLATE with options.quantization_mode / max_colors / dithering: a quantised
    image (colour type 3, 8-bit indices) or, when pixo would not quantise, reduce_and_filter's result.
    palette: optional (n, 4) RGBA median-cut palette to map with (pixo's truncation case).  Returns
    (ReducedImage, filtered stream, its Adler-32).  See pixo_b200_png_quantize_filter."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    w, h = int(options.width), int(options.height)
    out = np.empty(max(h * (w * ColorType(options.color_type).bytes_per_pixel() + 1), 1), np.uint8)
    info, n, ad = _Reduced(), C.c_size_t(), C.c_uint32()
    pal = None if palette is None else np.ascontiguousarray(palette, np.uint8).reshape(-1, 4)
    rc = _lib.load().pixo_b200_png_quantize_filter(
        ctx.handle, d.ctypes.data if d.size else None, d.size, w, h, int(options.color_type), options.strategy_word(),
        int(options.max_colors), None if pal is None else pal.ctypes.data, 0 if pal is None else len(pal),
        C.byref(info), out.ctypes.data, out.size, C.byref(n), C.byref(ad))
    _lib.check(ctx.handle, rc)
    return ReducedImage._from_c(info), out[:n.value], ad.value


def quantize_and_filter_dev(d_data, in_stride, n_images, options: PngOptions, d_out, out_stride, d_adler=None,
                            palettes=None, ctx: Context | None = None):
    """Device-resident batch (anything with .data_ptr()): see pixo_b200_png_quantize_filter_dev.  palettes:
    optional list of n_images entries, each None (design it) or an (n, 4) RGBA palette.  Returns the
    n_images ReducedImage descriptions; the filtered streams and checksums are still being written
    asynchronously on the context's stream."""
    ctx = ctx or default_context()
    n_images = int(n_images)
    infos = (_Reduced * max(n_images, 1))()
    p = lambda t: None if t is None else int(t.data_ptr())
    pals, lens = _palette_table(palettes, n_images)
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_quantize_filter_dev(
        ctx.handle, p(d_data), int(in_stride), n_images, int(options.width), int(options.height),
        int(options.color_type), options.strategy_word(), int(options.max_colors),
        None if pals is None else pals.ctypes.data, None if lens is None else lens.ctypes.data, infos, p(d_out),
        int(out_stride), p(d_adler)))
    return [ReducedImage._from_c(infos[i]) for i in range(n_images)]


def adler32_combine(adler_a: int, adler_b: int, len_b: int) -> int:
    """Adler-32 of A ++ B from the two checksums and len(B)."""
    return int(_lib.load().pixo_b200_adler32_combine(int(adler_a), int(adler_b), int(len_b)))


def _palette_table(palettes, n_images):
    """n_images x 256 x 4 palettes and their lengths for the batch calls (None: every frame designs its own)."""
    if palettes is None:
        return None, None
    pals = np.zeros((max(n_images, 1), 256, 4), np.uint8)
    lens = np.zeros(max(n_images, 1), np.uint32)
    for i, q in enumerate(palettes):
        if q is not None:
            q = np.asarray(q, np.uint8).reshape(-1, 4)
            pals[i, :len(q)] = q
            lens[i] = len(q)
    return pals, lens


def _encode_word(options: PngOptions) -> int:
    return options.strategy_word() | (OPTIMAL_COMPRESSION if options.optimal_compression else 0)


def encode_capacity(width: int, height: int, color_type) -> int:
    """The largest file pixo_b200_png_encode* can write for a frame of this geometry: a stored-block zlib stream (the
    most pixo writes for n bytes) in IDAT chunks of 256 KiB with the signature, IHDR and IEND, either of the unreduced
    filtered rows or, for RGB and RGBA, of 8-bit palette indices with the largest PLTE and tRNS."""
    def file(n, small):
        zb = 2 + n + (n // 65535 + 1) * 5 + 4
        return 8 + 25 + small + zb + 12 * -(-zb // IDAT_CHUNK) + 12
    ct, w, h = ColorType(color_type), int(width), int(height)
    plain = file(h * (w * ct.bytes_per_pixel() + 1), 0)
    return plain if ct not in (ColorType.Rgb, ColorType.Rgba) else max(plain, file(h * (w + 1), 780 + 268))


def encode(data, options: PngOptions, palette=None, ctx: Context | None = None) -> bytes:
    """png::encode (src/png/mod.rs:424-435): the whole PNG file pixo writes for `data` with `options` at the fast
    and balanced presets, byte for byte.  palette: optional (n, 4) RGBA median-cut palette for a frame that
    quantises (pixo's truncation case).  See pixo_b200_png_encode."""
    out = bytearray()
    encode_into(out, data, options, palette, ctx)
    return bytes(out)


def encode_into(output: bytearray, data, options: PngOptions, palette=None, ctx: Context | None = None) -> None:
    """png::encode_into (src/png/mod.rs:437-630): output is cleared, then holds the file."""
    ctx = ctx or default_context()
    output.clear()
    d = _as_u8(data)
    w, h = int(options.width), int(options.height)
    cap = encode_capacity(w, h, options.color_type) if w and h else 0
    out = np.empty(max(cap, 1), np.uint8)
    n = C.c_size_t()
    pal = None if palette is None else np.ascontiguousarray(palette, np.uint8).reshape(-1, 4)
    rc = _lib.load().pixo_b200_png_encode(
        ctx.handle, d.ctypes.data if d.size else None, d.size, w, h, int(options.color_type), _encode_word(options),
        int(options.compression_level), int(options.max_colors), None if pal is None else pal.ctypes.data,
        0 if pal is None else len(pal), out.ctypes.data, cap, C.byref(n))
    _lib.check(ctx.handle, rc)
    output += out[:n.value].tobytes()


def encode_on_device(d_data, in_stride, n_images, options: PngOptions, d_out, out_cap_each, palettes=None,
                     ctx: Context | None = None):
    """n device frames (anything with .data_ptr()) of options' geometry -> n whole PNG files, file i in the device
    slot at d_out + i * out_cap_each.  palettes: optional list of n_images entries, each None or an (n, 4) RGBA
    palette.  Returns (lengths, status, infos): numpy arrays of each file's length and its status (0,
    ERR_OUTPUT_TOO_SMALL with the length it needs, or ERR_UNSUPPORTED for a filtered stream of 2^31 bytes or more;
    the slot is then untouched), and the ReducedImage of each frame.  Waits for the device: see
    pixo_b200_png_encode_on_device."""
    ctx = ctx or default_context()
    n_images = int(n_images)
    infos = (_Reduced * max(n_images, 1))()
    out_lens = np.zeros(max(n_images, 1), np.uint64)
    status = np.zeros(max(n_images, 1), np.int32)
    pals, lens = _palette_table(palettes, n_images)
    p = lambda t: None if t is None else int(t.data_ptr())
    szp = C.POINTER(C.c_size_t)
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_encode_on_device(
        ctx.handle, p(d_data), int(in_stride), n_images, int(options.width), int(options.height),
        int(options.color_type), _encode_word(options), int(options.compression_level), int(options.max_colors),
        None if pals is None else pals.ctypes.data, None if lens is None else lens.ctypes.data, p(d_out),
        int(out_cap_each), out_lens.ctypes.data_as(szp), status.ctypes.data_as(C.POINTER(C.c_int32)), infos))
    return out_lens[:n_images], status[:n_images], [ReducedImage._from_c(infos[i]) for i in range(n_images)]
