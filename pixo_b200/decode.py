"""Mirror of pixo::decode (src/decode/jpeg.rs for baseline JPEGs, src/decode/png.rs), decoded on the GPU.

  JpegImage                 pixo::decode::JpegImage (width, height, pixels, color_type)
  decode_jpeg               pixo::decode::decode_jpeg: pixel-identical, pixo's errors and messages
  jpeg_info                 the geometry and colour type decode_jpeg would return, host only
  decode_jpeg_batch_dev     many files -> frames in one device tensor, queued on the context's stream
  PngImage                  pixo::decode::PngImage (width, height, pixels, color_type)
  decode_png                pixo::decode::decode_png: pixel-identical, pixo's errors and messages
  png_info                  the geometry and colour type decode_png would return, host only (IDAT CRCs excepted)
  decode_png_batch_dev      many files -> frames in one device tensor; returns with every file's status known
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from . import _lib
from .color import ColorType
from .context import Context, default_context


@dataclasses.dataclass
class JpegImage:
    width: int
    height: int
    pixels: np.ndarray
    color_type: ColorType


def _bytes(data) -> bytes:
    return data.tobytes() if isinstance(data, np.ndarray) else bytes(data)


def jpeg_info(data) -> tuple[int, int, ColorType]:
    """(width, height, color_type) of the image decode_jpeg would return; raises PixoError with pixo's error."""
    b = _bytes(data)
    w, h, ct = C.c_uint32(), C.c_uint32(), C.c_uint32()
    _lib.check(None, _lib.load().pixo_b200_jpeg_decode_info(b, len(b), C.byref(w), C.byref(h), C.byref(ct)))
    return w.value, h.value, ColorType(ct.value)


def decode_jpeg(data, ctx: Context | None = None) -> JpegImage:
    """pixo::decode::decode_jpeg on the GPU: packed Gray or RGB pixels."""
    ctx = ctx or default_context()
    b = _bytes(data)
    w, h, ct = jpeg_info(b)
    out = np.empty(max(w * h * ColorType(ct).bytes_per_pixel(), 1), np.uint8)
    rw, rh, rct = C.c_uint32(), C.c_uint32(), C.c_uint32()
    _lib.check(ctx.handle, _lib.load().pixo_b200_jpeg_decode(ctx.handle, b, len(b), out.ctypes.data, out.size,
                                                             C.byref(rw), C.byref(rh), C.byref(rct)))
    return JpegImage(w, h, out[:w * h * ColorType(ct).bytes_per_pixel()], ct)


@dataclasses.dataclass
class DecodedBatch:
    """Frames of a batch decode: frame i is frames[offsets[i] : offsets[i] + nbytes(i)], packed, with geometry
    geometries[i] = (width, height, color_type); a file pixo rejects has geometry None and its PixoError in errors."""
    frames: object                     # torch.uint8 tensor on the context's device
    offsets: list
    geometries: list
    errors: list


def _batch_dev(blobs, info, entry_point, ctx, align, failed_text) -> DecodedBatch:
    """Decodes the blobs into one device tensor through entry_point (pixo_b200_*_decode_to_device).  info(b) gives
    (width, height, color_type, producible); only a producible file gets a slot.  A file the call fails has geometry
    None, and PixoError(status, failed_text) where info raised no error."""
    import torch
    ctx = ctx or default_context()
    geoms, errors, offsets, total = [], [], [], 0
    for b in blobs:
        try:
            w, h, ct, producible = info(b)
            geoms.append((w, h, ct))
            errors.append(None)
        except _lib.PixoError as e:
            geoms.append(None)
            errors.append(e)
            producible = False
        offsets.append(total)
        if producible:
            total += -(-w * h * ColorType(ct).bytes_per_pixel() // align) * align
    # allocated on the stream that writes it: torch's caching allocator then neither hands the memory out while the
    # decode is still writing it nor lets the decode write memory that earlier work on another stream still reads
    dev = torch.device("cuda", ctx.device)
    sp = _lib.load().pixo_b200_ctx_stream(ctx.handle)
    stream = torch.cuda.ExternalStream(sp, device=dev) if sp else torch.cuda.default_stream(dev)
    with torch.cuda.stream(stream):
        frames = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    n = len(blobs)
    ptrs = (C.c_char_p * max(n, 1))(*blobs)
    lens = (C.c_size_t * max(n, 1))(*[len(b) for b in blobs])
    offs = (C.c_size_t * max(n, 1))(*offsets)
    status = (C.c_int32 * max(n, 1))()
    _lib.check(ctx.handle, entry_point(ctx.handle, C.cast(ptrs, C.c_void_p), lens, n, frames.data_ptr(), offs, status))
    for i in range(n):
        if status[i]:
            geoms[i] = None
            if errors[i] is None:
                errors[i] = _lib.PixoError(status[i], failed_text)
    return DecodedBatch(frames, offsets, geoms, errors)


def decode_jpeg_batch_dev(files, ctx: Context | None = None, align: int = 256) -> DecodedBatch:
    """Decodes the files into one device tensor (pixo_b200_jpeg_decode_to_device); the decode is queued on the
    context's stream when this returns, and the tensor belongs to that stream (work on another stream must wait for
    it, e.g. through ctx.sync()).  Each frame starts on an `align`-byte boundary."""
    return _batch_dev([_bytes(f) for f in files], lambda b: (*jpeg_info(b), True),
                      _lib.load().pixo_b200_jpeg_decode_to_device, ctx, align, "invalid argument")


@dataclasses.dataclass
class PngImage:
    width: int
    height: int
    pixels: np.ndarray
    color_type: ColorType


def _png_info(b: bytes):
    """(width, height, color_type, producible): producible is False when the IDAT data cannot produce the frame's
    rows, so that decode_png is certain to fail on the device."""
    w, h, ct, ok = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_int32()
    _lib.check(None, _lib.load().pixo_b200_png_decode_info(b, len(b), C.byref(w), C.byref(h), C.byref(ct),
                                                           C.byref(ok)))
    return w.value, h.value, ColorType(ct.value), bool(ok.value)


def png_info(data) -> tuple[int, int, ColorType]:
    """(width, height, color_type) of the image decode_png would return; raises PixoError with pixo's error for
    every failure decided before inflating, except an IDAT chunk's CRC in a file that has no other such failure."""
    return _png_info(_bytes(data))[:3]


def decode_png(data, ctx: Context | None = None) -> PngImage:
    """pixo::decode::decode_png on the GPU: packed Gray, GrayAlpha, RGB or RGBA pixels."""
    ctx = ctx or default_context()
    b = _bytes(data)
    w, h, ct, producible = _png_info(b)
    # a file whose stream cannot produce its rows only has its error to report: no frame is allocated for it
    out = np.empty(w * h * ColorType(ct).bytes_per_pixel() if producible else 0, np.uint8)
    rw, rh, rct = C.c_uint32(), C.c_uint32(), C.c_uint32()
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_decode(ctx.handle, b, len(b), out.ctypes.data if out.size else None,
                                                            out.size, C.byref(rw), C.byref(rh), C.byref(rct)))
    return PngImage(w, h, out, ct)


def decode_png_batch_dev(files, ctx: Context | None = None, align: int = 256) -> DecodedBatch:
    """Decodes the files into one device tensor (pixo_b200_png_decode_to_device).  The call waits for the device
    once per pass, so every file's status is known when it returns; the frames are written in the context's stream
    order, and the tensor belongs to that stream.  Each frame starts on an `align`-byte boundary.  A file whose rows
    (height * (1 + scanline bytes)) are more than its IDAT data can produce is certain to fail and gets no slot."""
    return _batch_dev([_bytes(f) for f in files], _png_info, _lib.load().pixo_b200_png_decode_to_device, ctx, align,
                      "png decode failed")
