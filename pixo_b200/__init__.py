"""pixo_b200 — H100 (sm_90a) drop-in for the data-parallel stages of pixo's JPEG/PNG encoders.

Python mirror of the reference's public API for this path:
  pixo_b200.jpeg  <->  pixo::jpeg   (encode, encode_into, JpegOptions, Subsampling)
  pixo_b200.png   <->  pixo::png    (encode, encode_into, filter::apply_filters*, FilterStrategy, PngOptions) and
                       pixo::compress::adler32
  pixo_b200.resize <-> pixo::resize (resize, resize_into, ResizeOptions, ResizeAlgorithm)
  pixo_b200.decode <-> pixo::decode (decode_jpeg, JpegImage, decode_png, PngImage)
All arithmetic happens in libpixo_b200.so (hand-written CUDA behind a C ABI, include/pixo_b200.h).
"""
from ._lib import PixoError, SO_PATH, load  # noqa: F401
from .color import ColorType  # noqa: F401
from .context import Context, default_context  # noqa: F401
from . import decode, jpeg, png, resize  # noqa: F401

__all__ = ["PixoError", "ColorType", "Context", "default_context", "decode", "jpeg", "png", "resize", "load", "SO_PATH"]
