"""ctypes binding of libpixo_b200.so — the only thing this package computes with.

There is no CPU fallback: if the shared library is missing the import fails loudly, and if no
CUDA device is present every compute call raises PixoError (status PIXO_B200_ERR_CUDA).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("PIXO_B200_SO") or os.path.join(_HERE, "libpixo_b200.so")

u8p = C.POINTER(C.c_uint8)
i16p = C.POINTER(C.c_int16)
f32p = C.POINTER(C.c_float)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
szp = C.POINTER(C.c_size_t)
vp = C.c_void_p

# status codes (include/pixo_b200.h)
OK = 0
ERR_INVALID_QUALITY, ERR_INVALID_DIMENSIONS, ERR_IMAGE_TOO_LARGE, ERR_UNSUPPORTED_COLOR = 1, 2, 3, 4
ERR_INVALID_DATA_LENGTH, ERR_INVALID_RESTART, ERR_INVALID_ARGUMENT, ERR_OUTPUT_TOO_SMALL = 5, 6, 7, 8
ERR_UNSUPPORTED, ERR_CUDA, ERR_OOM = 9, 10, 11
ERR_INVALID_DECODE, ERR_UNSUPPORTED_DECODE = 12, 13
ERR_INVALID_COMPRESSION_LEVEL = 14

# every symbol include/pixo_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "pixo_b200_version": (C.c_int, []),
    "pixo_b200_device_count": (C.c_int, []),
    "pixo_b200_ctx_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
    "pixo_b200_ctx_destroy": (None, [vp]),
    "pixo_b200_last_error": (C.c_char_p, [vp]),
    "pixo_b200_ctx_set_stream": (C.c_int, [vp, vp]),
    "pixo_b200_ctx_stream": (vp, [vp]),
    "pixo_b200_ctx_sync": (C.c_int, [vp]),
    "pixo_b200_ctx_launch_count": (C.c_uint64, [vp]),
    "pixo_b200_ctx_set_host_threads": (C.c_int, [vp, C.c_int]),
    "pixo_b200_ctx_host_fallbacks": (C.c_uint64, [vp]),
    "pixo_b200_ctx_set_scan_capacity": (C.c_int, [vp, C.c_size_t, C.c_int]),
    "pixo_b200_dev_alloc": (C.c_int, [vp, C.c_size_t, C.POINTER(vp)]),
    "pixo_b200_dev_free": (C.c_int, [vp, vp]),
    "pixo_b200_host_alloc_pinned": (C.c_int, [vp, C.c_size_t, C.POINTER(vp)]),
    "pixo_b200_host_free_pinned": (C.c_int, [vp, vp]),
    "pixo_b200_upload": (C.c_int, [vp, vp, vp, C.c_size_t]),
    "pixo_b200_download": (C.c_int, [vp, vp, vp, C.c_size_t]),
    "pixo_b200_quant_tables": (None, [C.c_int, u8p, u8p, f32p, f32p]),
    "pixo_b200_jpeg_block_counts": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, szp, szp]),
    "pixo_b200_jpeg_coefficients": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                              f32p, f32p, vp, vp, vp, C.c_uint32, vp]),
    "pixo_b200_jpeg_coefficients_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                                  C.c_uint32, C.c_uint32, f32p, f32p, vp, C.c_size_t,
                                                  vp, vp, C.c_size_t, C.c_uint32, vp]),
    "pixo_b200_jpeg_trellis_quantize_dev": (C.c_int, [vp, vp, C.c_size_t, f32p, C.c_float, vp, C.c_uint32]),
    "pixo_b200_jpeg_encode": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                        C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                        C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_encode_batch": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                              C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                              C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_encode_progressive": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                                    C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                    vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_encode_progressive_batch": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                                          C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                          C.c_uint32, C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_progressive_scans_dev": (C.c_int, [vp, vp, C.c_size_t, vp, vp, C.c_size_t, C.c_uint32,
                                                       C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp,
                                                       C.c_size_t, vp, vp]),
    "pixo_b200_jpeg_encode_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                            C.c_uint32, C.c_uint32, vp, C.c_size_t, vp, vp]),
    "pixo_b200_jpeg_encode_dev_opts": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp, C.c_size_t, vp,
                                                 vp, vp]),
    "pixo_b200_jpeg_encode_dev_progressive": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                                        C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                        C.c_uint32, vp, C.c_size_t, vp, vp, vp]),
    "pixo_b200_jpeg_entropy_encode": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                                C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp,
                                                C.c_size_t, szp]),
    "pixo_b200_jpeg_entropy_encode_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32,
                                                    C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp,
                                                    C.c_size_t, szp]),
    "pixo_b200_jpeg_band_last_dc": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, C.POINTER(C.c_int32)]),
    "pixo_b200_jpeg_band_histogram_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                    C.POINTER(C.c_int32), vp]),
    "pixo_b200_jpeg_band_entropy_dev": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                  C.POINTER(C.c_int32), u64p, vp, C.c_size_t, u64p, u32p]),
    "pixo_b200_jpeg_band_splice_dev": (C.c_int, [vp, vp, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, vp,
                                                 C.c_size_t, u64p]),
    "pixo_b200_jpeg_band_entropy_dev_async": (C.c_int, [vp, vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                        vp, u64p, vp, C.c_size_t, vp, vp]),
    "pixo_b200_jpeg_band_splice_dev_async": (C.c_int, [vp, vp, vp, vp, C.c_size_t, vp, vp]),
    "pixo_b200_jpeg_band_dev_progressive_summary": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, C.c_uint64,
                                                              C.c_uint64, C.POINTER(C.c_int32), u32p]),
    "pixo_b200_jpeg_band_dev_progressive": (C.c_int, [vp, vp, vp, vp, C.c_size_t, C.c_size_t, C.c_uint64, C.c_uint64,
                                                      C.c_uint64, C.c_uint64, C.POINTER(C.c_int32), u32p, vp, vp, vp,
                                                      C.c_size_t, szp, u64p, u32p]),
    "pixo_b200_jpeg_band_dev_progressive_splice": (C.c_int, [vp, vp, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32,
                                                             C.c_uint32, vp, C.c_size_t, u64p]),
    "pixo_b200_jpeg_band_entropy": (C.c_int, [vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                              C.POINTER(C.c_int32), u64p, vp, C.c_size_t, u64p, u32p]),
    "pixo_b200_jpeg_band_histogram": (C.c_int, [vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                C.POINTER(C.c_int32), u64p]),
    "pixo_b200_jpeg_band_splice": (C.c_int, [vp, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_write_headers": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                               u64p, vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_write_headers_dht": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                   C.c_uint32, vp, vp, C.c_size_t, szp]),
    "pixo_b200_jpeg_progressive_file": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                  C.c_uint32, vp, vp, u64p, vp, C.c_size_t, szp]),
    "pixo_b200_png_filter_rows_dev": (C.c_int, [vp, vp, vp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_size_t,
                                                C.c_uint32, C.c_uint32, vp, vp]),
    "pixo_b200_adler32_combine": (C.c_uint32, [C.c_uint32, C.c_uint32, C.c_uint64]),
    "pixo_b200_png_filter": (C.c_int, [vp, vp, C.c_uint32, C.c_uint32, C.c_size_t, C.c_uint32,
                                       C.c_uint32, vp, u32p]),
    "pixo_b200_png_filter_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                           C.c_size_t, C.c_uint32, C.c_uint32, vp, C.c_size_t, vp]),
    "pixo_b200_png_reduce_filter": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                              vp, vp, C.c_size_t, szp, u32p]),
    "pixo_b200_png_reduce_filter_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                                  C.c_uint32, C.c_uint32, vp, vp, C.c_size_t, vp]),
    "pixo_b200_png_quantize_filter": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                C.c_uint32, vp, C.c_uint32, vp, vp, C.c_size_t, szp, u32p]),
    "pixo_b200_png_quantize_filter_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                                    C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp, vp, C.c_size_t,
                                                    vp]),
    "pixo_b200_resize": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                   C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_resize_dev": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                       C.c_uint32, C.c_uint32, C.c_uint32, vp, C.c_size_t]),
    "pixo_b200_jpeg_decode_info": (C.c_int, [vp, C.c_size_t, u32p, u32p, u32p]),
    "pixo_b200_jpeg_decode": (C.c_int, [vp, vp, C.c_size_t, vp, C.c_size_t, u32p, u32p, u32p]),
    "pixo_b200_jpeg_decode_to_device": (C.c_int, [vp, vp, szp, C.c_uint32, vp, szp, C.POINTER(C.c_int32)]),
    "pixo_b200_png_decode_info": (C.c_int, [vp, C.c_size_t, u32p, u32p, u32p, C.POINTER(C.c_int32)]),
    "pixo_b200_png_decode": (C.c_int, [vp, vp, C.c_size_t, vp, C.c_size_t, u32p, u32p, u32p]),
    "pixo_b200_png_decode_to_device": (C.c_int, [vp, vp, szp, C.c_uint32, vp, szp, C.POINTER(C.c_int32)]),
    "pixo_b200_resize_weights": (C.c_int, [C.c_uint32, C.c_uint32, vp, vp, vp, vp, C.c_size_t, szp]),
    "pixo_b200_adler32": (C.c_int, [vp, vp, C.c_size_t, u32p]),
    "pixo_b200_adler32_dev": (C.c_int, [vp, vp, C.c_size_t, vp]),
    "pixo_b200_deflate_zlib": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_deflate_zlib_on_device": (C.c_int, [vp, vp, C.c_size_t, szp, C.c_uint32, C.c_uint32, vp, C.c_size_t, szp,
                                             C.POINTER(C.c_int32)]),
    "pixo_b200_png_encode": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                       C.c_uint32, vp, C.c_uint32, vp, C.c_size_t, szp]),
    "pixo_b200_png_encode_on_device": (C.c_int, [vp, vp, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                 C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_size_t, szp,
                                                 C.POINTER(C.c_int32), vp]),
}


class PixoError(RuntimeError):
    """Mirror of pixo::Error (src/error.rs:10-47); `.code` is the pixo_b200_status."""

    def __init__(self, code: int, message: str):
        super().__init__(message)
        self.code = code


_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ImportError(
                f"{SO_PATH} is missing: build it with `python -m pixo_b200.build` "
                "(nvcc, sm_90a). pixo_b200 has no CPU fallback.")
        lib = C.CDLL(SO_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the ABI drifted from the header
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(ctx, rc: int):
    if rc != 0:
        msg = load().pixo_b200_last_error(ctx)
        raise PixoError(rc, (msg or b"").decode("utf-8", "replace"))
