"""Mirror of pixo::compress::deflate::deflate_zlib_packed (src/compress/deflate.rs:1074) at levels 1-9, on the GPU.

  deflate_zlib_packed(data, level)     one host buffer -> its zlib stream (bytes)
  deflate_zlib_packed_dev(...)         n device streams -> their zlib streams in device slots
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .context import Context, default_context


def deflate_zlib_packed(data, level: int, ctx: Context | None = None) -> bytes:
    """The zlib stream pixo's deflate_zlib_packed writes for `data` at `level` (1-9), byte for byte."""
    ctx = ctx or default_context()
    d = np.frombuffer(bytes(data), np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) \
        else np.ascontiguousarray(data, np.uint8).reshape(-1)
    cap = 2 + d.size + (d.size // 65535 + 1) * 5 + 4
    out = np.empty(cap, np.uint8)
    n = C.c_size_t()
    rc = _lib.load().pixo_b200_deflate_zlib(ctx.handle, d.ctypes.data if d.size else None, d.size, int(level),
                                            out.ctypes.data, cap, C.byref(n))
    _lib.check(ctx.handle, rc)
    return out[:n.value].tobytes()


def deflate_zlib_packed_dev(d_streams, stride: int, lens, level: int, d_out, out_cap_each: int,
                            ctx: Context | None = None):
    """n device streams (anything with .data_ptr()), stream i at d_streams + i * stride with lens[i] bytes, each to
    its slot at d_out + i * out_cap_each: see pixo_b200_deflate_zlib_on_device.  Returns (lengths, status) as numpy
    arrays; status[i] is 0 or ERR_OUTPUT_TOO_SMALL (that slot is left untouched, lengths[i] is what it needs)."""
    ctx = ctx or default_context()
    ln = np.ascontiguousarray(lens, np.uint64)
    n = ln.size
    out_lens = np.zeros(n, np.uint64)
    status = np.zeros(n, np.int32)
    szp = C.POINTER(C.c_size_t)
    rc = _lib.load().pixo_b200_deflate_zlib_on_device(
        ctx.handle, int(d_streams.data_ptr()) if n else None, int(stride), ln.ctypes.data_as(szp), n, int(level),
        int(d_out.data_ptr()) if n else None, int(out_cap_each), out_lens.ctypes.data_as(szp),
        status.ctypes.data_as(C.POINTER(C.c_int32)))
    _lib.check(ctx.handle, rc)
    return out_lens, status
