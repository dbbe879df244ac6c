"""Mirror of pixo::resize (src/resize.rs) for the accelerated path.

  ResizeAlgorithm            src/resize.rs:33-45 (default Bilinear), numbered as src/wasm.rs:156-166
  ResizeOptions.builder      src/resize.rs:81-146 (destination = source, colour type RGBA by default)
  resize / resize_into       src/resize.rs:162-191
  resize_dev                 a batch of device-resident frames (pixo_b200_resize_dev)
  weights                    Lanczos3's contribution table of one axis (pixo_b200_resize_weights)
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum

import numpy as np

from . import _lib
from .color import ColorType
from .context import Context, default_context


class ResizeAlgorithm(enum.IntEnum):
    Nearest = 0
    Bilinear = 1
    Lanczos3 = 2


@dataclasses.dataclass
class ResizeOptions:
    """pixo::resize::ResizeOptions."""
    src_width: int
    src_height: int
    dst_width: int
    dst_height: int
    color_type: ColorType = ColorType.Rgba
    algorithm: ResizeAlgorithm = ResizeAlgorithm.Bilinear

    @classmethod
    def builder(cls, src_width: int, src_height: int) -> "ResizeOptionsBuilder":
        return ResizeOptionsBuilder(src_width, src_height)

    def bytes_per_pixel(self) -> int:
        return ColorType(self.color_type).bytes_per_pixel()


class ResizeOptionsBuilder:
    """pixo::resize::ResizeOptionsBuilder: dst / color_type / algorithm, then build()."""

    def __init__(self, src_width: int, src_height: int):
        self._o = ResizeOptions(int(src_width), int(src_height), int(src_width), int(src_height))

    def dst(self, width: int, height: int) -> "ResizeOptionsBuilder":
        self._o.dst_width, self._o.dst_height = int(width), int(height)
        return self

    def color_type(self, color_type: ColorType) -> "ResizeOptionsBuilder":
        self._o.color_type = color_type
        return self

    def algorithm(self, algorithm: ResizeAlgorithm) -> "ResizeOptionsBuilder":
        self._o.algorithm = algorithm
        return self

    def build(self) -> ResizeOptions:
        return dataclasses.replace(self._o)


def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
    return np.frombuffer(data, dtype=np.uint8)


def resize_into(output: np.ndarray, data, options: ResizeOptions, ctx: Context | None = None) -> int:
    """resize_into: writes the resized pixels to the start of `output` (a uint8 array) and returns their
    count.  Raises PixoError with pixo's errors, or ERR_OUTPUT_TOO_SMALL when `output` is too short."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    if output.dtype != np.uint8 or not output.flags.c_contiguous:
        raise ValueError("output must be a contiguous uint8 array")
    n = C.c_size_t()
    rc = _lib.load().pixo_b200_resize(ctx.handle, d.ctypes.data if d.size else None, d.size, int(options.src_width),
                                      int(options.src_height), int(options.dst_width), int(options.dst_height),
                                      int(options.color_type), int(options.algorithm),
                                      output.ctypes.data if output.size else None, output.size, C.byref(n))
    _lib.check(ctx.handle, rc)
    return n.value


def resize(data, options: ResizeOptions, ctx: Context | None = None) -> np.ndarray:
    """resize: the resized pixels, same colour type."""
    w, h = int(options.dst_width), int(options.dst_height)
    size = w * h * ColorType(options.color_type).bytes_per_pixel() if 0 <= int(options.color_type) <= 3 else 0
    out = np.empty(max(size, 1) if 0 < w <= 1 << 24 and 0 < h <= 1 << 24 else 1, np.uint8)
    n = resize_into(out, data, options, ctx)
    return out[:n]


def resize_dev(d_src, src_stride: int, n_images: int, options: ResizeOptions, d_dst, dst_stride: int,
               ctx: Context | None = None):
    """Device-resident batch (anything with .data_ptr()): see pixo_b200_resize_dev.  Asynchronous on the
    context's stream."""
    ctx = ctx or default_context()
    p = lambda t: None if t is None else int(t.data_ptr())
    _lib.check(ctx.handle, _lib.load().pixo_b200_resize_dev(
        ctx.handle, p(d_src), int(src_stride), int(n_images), int(options.src_width), int(options.src_height),
        int(options.dst_width), int(options.dst_height), int(options.color_type), int(options.algorithm), p(d_dst),
        int(dst_stride)))


def weights(src_size: int, dst_size: int):
    """Lanczos3's contribution table of one axis: (start, count, offset, weights), see
    pixo_b200_resize_weights.  Host only."""
    L = _lib.load()
    n = C.c_size_t()
    dst = int(dst_size)
    start, count = np.empty(max(dst, 1), np.uint32), np.empty(max(dst, 1), np.uint32)
    offset = np.empty(max(dst, 1), np.uint64)
    _lib.check(None, L.pixo_b200_resize_weights(int(src_size), dst, start.ctypes.data, count.ctypes.data,
                                                offset.ctypes.data, None, 0, C.byref(n)))
    w = np.empty(max(n.value, 1), np.float32)
    _lib.check(None, L.pixo_b200_resize_weights(int(src_size), dst, None, None, None, w.ctypes.data, w.size,
                                                C.byref(n)))
    return start[:dst], count[:dst], offset[:dst], w[:n.value]
