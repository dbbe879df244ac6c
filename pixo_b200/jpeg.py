"""Mirror of pixo::jpeg for the accelerated path (src/jpeg/mod.rs:88-447).

`encode` / `encode_into` keep the reference's names, argument meaning and error behaviour;
the transform stages run on the GPU through libpixo_b200.so, the entropy stage on the host
inside the same library.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum

import numpy as np

from . import _lib
from .color import ColorType
from .context import Context, default_context


class Subsampling(enum.IntEnum):
    """pixo::jpeg::Subsampling (src/jpeg/mod.rs:96-102)."""
    S444 = 0
    S420 = 1


@dataclasses.dataclass
class JpegOptions:
    """pixo::jpeg::JpegOptions (src/jpeg/mod.rs:121-174): same fields, same defaults."""
    width: int = 0
    height: int = 0
    color_type: ColorType = ColorType.Rgb
    quality: int = 75
    subsampling: Subsampling = Subsampling.S444
    restart_interval: int | None = None
    optimize_huffman: bool = False
    progressive: bool = False
    trellis_quant: bool = False

    @classmethod
    def fast(cls, width, height, quality):
        return cls(width, height, ColorType.Rgb, quality, Subsampling.S444, None, False, False, False)

    @classmethod
    def balanced(cls, width, height, quality):
        return cls(width, height, ColorType.Rgb, quality, Subsampling.S444, None, True, False, False)

    @classmethod
    def max(cls, width, height, quality):
        return cls(width, height, ColorType.Rgb, quality, Subsampling.S420, None, True, True, True)

    @classmethod
    def from_preset(cls, width, height, quality, preset):
        return {0: cls.fast, 2: cls.max}.get(preset, cls.balanced)(width, height, quality)


def output_capacity(width: int, height: int) -> int:
    """Upper bound on a baseline JPEG's size: ~260 B per block worst case (63 sixteen-bit codes
    + ten-bit amplitudes), x2 for 0xFF stuffing, three full-resolution components, RSTn
    markers, headers."""
    nb = ((int(width) + 7) // 8) * ((int(height) + 7) // 8) * 3
    return nb * 600 + 4096


def _restart(options) -> int:
    """Some(0) is InvalidRestartInterval in the reference (src/jpeg/mod.rs:339-345); None -> 0."""
    if options.restart_interval is not None and int(options.restart_interval) == 0:
        raise _lib.PixoError(_lib.ERR_INVALID_RESTART, "Invalid restart interval 0")
    return int(options.restart_interval or 0)


def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
    return np.frombuffer(data, dtype=np.uint8)


def quant_tables(quality: int):
    """QuantizationTables::with_quality (src/jpeg/quantize.rs:42-89): (lum_zz, chr_zz, lum, chr)."""
    lz = np.zeros(64, np.uint8); cz = np.zeros(64, np.uint8)
    ln = np.zeros(64, np.float32); cn = np.zeros(64, np.float32)
    _lib.load().pixo_b200_quant_tables(int(quality), lz.ctypes.data_as(_lib.u8p), cz.ctypes.data_as(_lib.u8p),
                                       ln.ctypes.data_as(_lib.f32p), cn.ctypes.data_as(_lib.f32p))
    return lz, cz, ln, cn


def block_counts(width, height, color_type=ColorType.Rgb, subsampling=Subsampling.S420):
    ny = C.c_size_t(); nc = C.c_size_t()
    _lib.check(None, _lib.load().pixo_b200_jpeg_block_counts(width, height, int(color_type), int(subsampling),
                                                             C.byref(ny), C.byref(nc)))
    return ny.value, nc.value


COEF_ZIGZAG, COEF_TRELLIS = 1, 2   # flags of pixo_b200_jpeg_coefficients* (include/pixo_b200.h)


def compute_all_coefficients(data, width, height, color_type=ColorType.Rgb,
                             subsampling=Subsampling.S420, quality=None, lum_q=None, chr_q=None,
                             zigzag=False, histograms=False, ctx: Context | None = None, use_trellis=False):
    """compute_all_coefficients (src/jpeg/mod.rs:932-966) -> (y, cb, cr[, hist]) int16 [n,64].
    use_trellis: trellis-quantise every block, as pixo's max preset does (no histograms then: pixo's
    tables come from the plain-rounded coefficients)."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    bpp = 1 if int(color_type) == ColorType.Gray else 3
    if d.size != int(width) * int(height) * bpp and width and height and int(color_type) in (0, 2):
        raise _lib.PixoError(_lib.ERR_INVALID_DATA_LENGTH,
                             f"Invalid data length: expected {int(width) * int(height) * bpp} bytes, got {d.size}")
    if lum_q is None:
        _, _, lum_q, chr_q = quant_tables(75 if quality is None else quality)
    lum_q = np.ascontiguousarray(lum_q, np.float32); chr_q = np.ascontiguousarray(chr_q, np.float32)
    ny, nc = block_counts(width, height, color_type, subsampling)
    y = np.empty((ny, 64), np.int16)
    cb = np.empty((max(nc, 1), 64), np.int16)
    cr = np.empty((max(nc, 1), 64), np.int16)
    hist = np.zeros(536, np.uint64) if histograms else None
    rc = _lib.load().pixo_b200_jpeg_coefficients(
        ctx.handle, d.ctypes.data, width, height, int(color_type), int(subsampling),
        lum_q.ctypes.data_as(_lib.f32p), chr_q.ctypes.data_as(_lib.f32p), y.ctypes.data,
        cb.ctypes.data, cr.ctypes.data, (COEF_ZIGZAG if zigzag else 0) | (COEF_TRELLIS if use_trellis else 0),
        hist.ctypes.data if histograms else None)
    _lib.check(ctx.handle, rc)
    out = (y, cb[:nc], cr[:nc])
    return out + (hist,) if histograms else out


def trellis_lambda(quality: int) -> float:
    """trellis_quantize_adaptive's lambda (src/jpeg/trellis.rs:304-321), in binary32 as pixo computes it."""
    q = int(quality)
    f = np.float32
    if q >= 80:
        return float(f(f(0.5) + f(100 - q) * f(0.025)))
    if q >= 50:
        return float(f(f(1.0) + f(80 - q) * f(0.033)))
    return float(f(f(2.0) + f(50 - q) * f(0.04)))


def trellis_quantize_dev(d_dct, quant_table, lam=None, d_out=None, zigzag=False, ctx: Context | None = None):
    """trellis::trellis_quantize (src/jpeg/trellis.rs:67-208) for a batch of blocks on the device:
    d_dct float32 [n, 64] (natural order, anything with .data_ptr()), quant_table 64 natural-order
    entries, lam None for pixo's default 1.0.  Writes / returns d_out int16 [n, 64] (a new torch tensor
    on the same device when None)."""
    ctx = ctx or default_context()
    if d_out is None:
        import torch
        d_out = torch.empty(d_dct.shape, dtype=torch.int16, device=d_dct.device)
    q = np.ascontiguousarray(quant_table, np.float32).reshape(64)
    n = int(d_dct.numel()) // 64
    rc = _lib.load().pixo_b200_jpeg_trellis_quantize_dev(
        ctx.handle, int(d_dct.data_ptr()), n, q.ctypes.data_as(_lib.f32p), 1.0 if lam is None else float(lam),
        int(d_out.data_ptr()), COEF_ZIGZAG if zigzag else 0)
    _lib.check(ctx.handle, rc)
    return d_out


def trellis_quantize(dct, quant_table, lam=None, ctx: Context | None = None) -> np.ndarray:
    """trellis::trellis_quantize on host blocks: dct float32 [64] or [n, 64] -> int16 of the same shape."""
    import torch
    a = np.ascontiguousarray(dct, np.float32)
    dev = torch.device("cuda", (ctx or default_context()).device)
    out = trellis_quantize_dev(torch.from_numpy(a.reshape(-1, 64)).to(dev), quant_table, lam, ctx=ctx)
    return out.cpu().numpy().reshape(a.shape)


def trellis_quantize_adaptive(dct, quant_table, quality, ctx: Context | None = None) -> np.ndarray:
    """trellis::trellis_quantize_adaptive (src/jpeg/trellis.rs:304-321)."""
    return trellis_quantize(dct, quant_table, trellis_lambda(quality), ctx=ctx)


def encode_into(output: bytearray, data, options: JpegOptions, ctx: Context | None = None) -> None:
    """pixo::jpeg::encode_into (src/jpeg/mod.rs:328): clears and refills `output`."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    cap = output_capacity(options.width, options.height)
    buf = np.empty(cap, np.uint8)
    n = C.c_size_t()
    restart = _restart(options)
    rc = _lib.load().pixo_b200_jpeg_encode(
        ctx.handle, d.ctypes.data, d.size, int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling),
        restart, int(bool(options.optimize_huffman)),
        int(bool(options.progressive)), int(bool(options.trellis_quant)), buf.ctypes.data, cap,
        C.byref(n))
    _lib.check(ctx.handle, rc)
    del output[:]
    output.extend(buf[: n.value].tobytes())


def encode(data, options: JpegOptions, ctx: Context | None = None) -> bytes:
    """pixo::jpeg::encode (src/jpeg/mod.rs:88)."""
    out = bytearray()
    encode_into(out, data, options, ctx)
    return bytes(out)


def encode_batch(frames: np.ndarray, options: JpegOptions, ctx: Context | None = None,
                 capacity_each: int | None = None) -> list[bytes]:
    """n frames of identical geometry ([n, h*w*bpp] uint8) -> n JPEG byte strings.
    capacity_each defaults to min(worst case, 2x the raw frame size)."""
    restart = _restart(options)
    ctx = ctx or default_context()
    f = np.ascontiguousarray(frames, np.uint8)
    n = f.shape[0]
    each = f.size // max(n, 1)
    cap = capacity_each or min(output_capacity(options.width, options.height), 2 * each + 4096)
    out = np.empty((n, cap), np.uint8)
    lens = (C.c_size_t * n)()
    rc = _lib.load().pixo_b200_jpeg_encode_batch(
        ctx.handle, f.ctypes.data, each, n, int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling),
        restart, int(bool(options.optimize_huffman)), out.ctypes.data,
        cap, lens)
    _lib.check(ctx.handle, rc)
    return [out[i, : lens[i]].tobytes() for i in range(n)]


def progressive_capacity(width: int, height: int) -> int:
    """Upper bound on a progressive file's size: a coefficient costs at most 31 bits (16-bit code +
    15 amplitude bits) plus its share of ZRLs and EOB runs, x2 for 0xFF stuffing, three full-resolution
    components, headers."""
    nb = ((int(width) + 7) // 8) * ((int(height) + 7) // 8) * 3
    return nb * 64 * 9 + 4096


def encode_progressive_into(output: bytearray, data, options: JpegOptions, ctx: Context | None = None) -> None:
    """pixo::jpeg::encode_into with progressive scans (src/jpeg/mod.rs:395-410, 872-927) whatever
    options.progressive says: SOF2 and the 7 scans of pixo's simple_progressive_script, quirks included
    (include/pixo_b200.h, pixo_b200_jpeg_encode_progressive).  Clears and refills `output`."""
    ctx = ctx or default_context()
    d = _as_u8(data)
    cap = min(progressive_capacity(options.width, options.height), 2 * d.size + 65536)
    buf = np.empty(cap, np.uint8)
    n = C.c_size_t()
    restart = _restart(options)
    rc = _lib.load().pixo_b200_jpeg_encode_progressive(
        ctx.handle, d.ctypes.data, d.size, int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling), restart,
        int(bool(options.optimize_huffman)), int(bool(options.trellis_quant)), buf.ctypes.data, cap, C.byref(n))
    _lib.check(ctx.handle, rc)
    del output[:]
    output.extend(buf[: n.value].tobytes())


def encode_progressive(data, options: JpegOptions, ctx: Context | None = None) -> bytes:
    """The progressive file pixo writes for `options` with progressive = true (JpegOptions.max: its
    max preset)."""
    out = bytearray()
    encode_progressive_into(out, data, options, ctx)
    return bytes(out)


def encode_progressive_batch(frames: np.ndarray, options: JpegOptions, ctx: Context | None = None,
                             capacity_each: int | None = None) -> list[bytes]:
    """n frames of identical geometry ([n, h*w*bpp] uint8) -> n progressive files."""
    restart = _restart(options)
    ctx = ctx or default_context()
    f = np.ascontiguousarray(frames, np.uint8)
    n = f.shape[0]
    each = f.size // max(n, 1)
    cap = capacity_each or min(progressive_capacity(options.width, options.height), 2 * each + 8192)
    out = np.empty((n, cap), np.uint8)
    lens = (C.c_size_t * n)()
    rc = _lib.load().pixo_b200_jpeg_encode_progressive_batch(
        ctx.handle, f.ctypes.data, each, n, int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling), restart,
        int(bool(options.optimize_huffman)), int(bool(options.trellis_quant)), out.ctypes.data, cap, lens)
    _lib.check(ctx.handle, rc)
    return [out[i, : lens[i]].tobytes() for i in range(n)]


def dht_array(tables) -> np.ndarray:
    """{(class, id): (bits[16], values)} (a file's DHT, e.g. tests' jpeg_progressive_scans.dht) ->
    the 4 x (16 counts + 256 values) uint8 array progressive_scans_dev takes."""
    a = np.zeros((4, 272), np.uint8)
    for k, key in enumerate([(0, 0), (0, 1), (1, 0), (1, 1)]):
        if key in tables:
            bits, vals = tables[key]
            a[k, :16] = bits
            a[k, 16:16 + len(vals)] = vals
    return a


def progressive_scans_dev(d_y, d_cb, d_cr, width, height, color_type=ColorType.Rgb,
                          subsampling=Subsampling.S420, tables=None, n_frames=1, y_stride=None, c_stride=None,
                          d_out=None, out_cap_each=None, d_scan_len=None, d_overflow=None,
                          ctx: Context | None = None):
    """The progressive scan stage on device coefficient arrays (int16 torch tensors in
    compute_all_coefficients' layout, natural order, 16-byte aligned; frame i at i * stride elements).
    tables: None for the standard tables, a uint8 [4, 272] array (dht_array) or a DHT dict.
    Returns (d_out, d_scan_len [n, 7], d_overflow [n]) - new tensors when not given - once the context's stream
    has written them, so that they can be read on any stream."""
    import torch
    ctx = ctx or default_context()
    ny, nc = block_counts(width, height, color_type, subsampling)
    dev = d_y.device
    y_stride = ny * 64 if y_stride is None else int(y_stride)
    c_stride = nc * 64 if c_stride is None else int(c_stride)
    if out_cap_each is None:
        out_cap_each = (progressive_capacity(width, height) + 15) // 16 * 16
    if d_out is None:
        d_out = torch.empty(n_frames * out_cap_each, dtype=torch.uint8, device=dev)
    if d_scan_len is None:
        d_scan_len = torch.empty((n_frames, 7), dtype=torch.int64, device=dev)
    if d_overflow is None:
        d_overflow = torch.empty(n_frames, dtype=torch.int32, device=dev)
    dht = None
    if tables is not None:
        dht = np.ascontiguousarray(dht_array(tables) if isinstance(tables, dict) else tables, np.uint8)
    ptr = lambda t: None if t is None else int(t.data_ptr())
    rc = _lib.load().pixo_b200_jpeg_progressive_scans_dev(
        ctx.handle, ptr(d_y), y_stride, ptr(d_cb), ptr(d_cr), c_stride, int(n_frames), int(width), int(height),
        int(color_type), int(subsampling), None if dht is None else dht.ctypes.data, ptr(d_out), int(out_cap_each),
        ptr(d_scan_len), ptr(d_overflow))
    _lib.check(ctx.handle, rc)
    ctx.sync()   # the call itself waits only for the bit counts; its splice into d_out is queued
    return d_out, d_scan_len, d_overflow


DHT_BYTES = 4 * 272   # a frame's tables in pixo_b200_jpeg_encode_dev_opts' d_dht


def encode_dev(d_frames, pixel_stride, n_images, options: JpegOptions, d_scan, scan_cap_each, d_scan_len,
               d_overflow, d_dht=None, ctx: Context | None = None) -> None:
    """pixo_b200_jpeg_encode_dev_opts: n_images device frames (frame i at d_frames + i * pixel_stride bytes)
    -> frame i's scan bytes at d_scan + i * scan_cap_each, its length in d_scan_len[i], its flags in
    d_overflow[i] and, when d_dht is given, its tables in d_dht[i] (DHT_BYTES each).  The buffers are
    anything with .data_ptr() (torch tensors) or device addresses.  options supplies the geometry, quality,
    restart interval and optimize_huffman; progressive raises ERR_UNSUPPORTED and trellis_quant is ignored,
    as pixo's baseline encode_scan ignores it.  Queued on the context's stream; nothing is synchronised.
    jpeg_file(options, dht, scan) makes a frame's file."""
    if options.progressive:
        raise _lib.PixoError(_lib.ERR_UNSUPPORTED, "progressive is not a device scan option: use encode_progressive")
    restart = _restart(options)
    ctx = ctx or default_context()
    ptr = lambda t: None if t is None else (int(t) if isinstance(t, int) else int(t.data_ptr()))
    rc = _lib.load().pixo_b200_jpeg_encode_dev_opts(
        ctx.handle, ptr(d_frames), int(pixel_stride), int(n_images), int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling), restart,
        int(bool(options.optimize_huffman)), ptr(d_scan), int(scan_cap_each), ptr(d_scan_len), ptr(d_overflow),
        ptr(d_dht))
    _lib.check(ctx.handle, rc)


def write_headers_dht(options: JpegOptions, dht) -> bytes:
    """SOI .. SOS of a baseline file whose Huffman tables are `dht` (DHT_BYTES, the layout encode_dev
    writes per frame)."""
    d = np.ascontiguousarray(np.asarray(dht, np.uint8).reshape(-1))
    if d.size != DHT_BYTES:
        raise _lib.PixoError(_lib.ERR_INVALID_ARGUMENT, f"a DHT block is {DHT_BYTES} bytes, got {d.size}")
    buf = np.zeros(2048, np.uint8)
    n = C.c_size_t()
    _lib.check(None, _lib.load().pixo_b200_jpeg_write_headers_dht(
        int(options.width), int(options.height), int(options.color_type), int(options.quality),
        int(options.subsampling), _restart(options), d.ctypes.data, buf.ctypes.data, buf.size, C.byref(n)))
    return buf[: n.value].tobytes()


def jpeg_file(options: JpegOptions, dht, scan) -> bytes:
    """One frame of encode_dev as a file: headers for its tables, its scan bytes, EOI."""
    return write_headers_dht(options, dht) + bytes(scan) + b"\xff\xd9"


def encode_progressive_dev(d_frames, pixel_stride, n_images, options: JpegOptions, d_out, out_cap_each, d_scan_len,
                           d_overflow, d_dht=None, ctx: Context | None = None) -> None:
    """pixo_b200_jpeg_encode_dev_progressive: pixo's progressive scans (options.optimize_huffman and
    options.trellis_quant as given; options.progressive is not read) of n_images device frames (frame i at
    d_frames + i * pixel_stride bytes) -> frame i's 7 segments back to back at d_out + i * out_cap_each, their
    lengths in d_scan_len[i] (7 int64), its flags in d_overflow[i] (bit 0: did not fit, bit 4: input the stage
    cannot carry) and, when d_dht is given, its tables in d_dht[i] (DHT_BYTES).  The buffers are anything with
    .data_ptr() (torch tensors) or device addresses.  Queued on the context's stream; nothing is synchronised.
    progressive_file(options, dht, segments, lens) makes a frame's file."""
    restart = _restart(options)
    ctx = ctx or default_context()
    ptr = lambda t: None if t is None else (int(t) if isinstance(t, int) else int(t.data_ptr()))
    rc = _lib.load().pixo_b200_jpeg_encode_dev_progressive(
        ctx.handle, ptr(d_frames), int(pixel_stride), int(n_images), int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling), restart,
        int(bool(options.optimize_huffman)), int(bool(options.trellis_quant)), ptr(d_out), int(out_cap_each),
        ptr(d_scan_len), ptr(d_overflow), ptr(d_dht))
    _lib.check(ctx.handle, rc)


def progressive_file(options: JpegOptions, dht, segments, lens) -> bytes:
    """A whole progressive file from one frame's tables (DHT_BYTES, or None for the standard ones), its 7
    segments back to back (bytes or a uint8 array, at least sum(lens) long) and their 7 lengths."""
    ln = np.ascontiguousarray(np.asarray(lens, np.uint64).reshape(-1))
    if ln.size != 7:
        raise _lib.PixoError(_lib.ERR_INVALID_ARGUMENT, f"a progressive file has 7 scans, got {ln.size} lengths")
    seg = _as_u8(segments)
    if seg.size < int(ln.sum()):
        raise _lib.PixoError(_lib.ERR_INVALID_ARGUMENT, f"segments hold {seg.size} bytes, the lengths {int(ln.sum())}")
    d = None
    if dht is not None:
        d = np.ascontiguousarray(np.asarray(dht, np.uint8).reshape(-1))
        if d.size != DHT_BYTES:
            raise _lib.PixoError(_lib.ERR_INVALID_ARGUMENT, f"a DHT block is {DHT_BYTES} bytes, got {d.size}")
    buf = np.zeros(4096 + int(ln.sum()), np.uint8)
    n = C.c_size_t()
    _lib.check(None, _lib.load().pixo_b200_jpeg_progressive_file(
        int(options.width), int(options.height), int(options.color_type), int(options.quality),
        int(options.subsampling), _restart(options), None if d is None else d.ctypes.data,
        seg.ctypes.data if seg.size else None, ln.ctypes.data_as(_lib.u64p), buf.ctypes.data, buf.size, C.byref(n)))
    return buf[: n.value].tobytes()


def entropy_encode(y, cb, cr, options: JpegOptions, ctx: Context | None = None) -> bytes:
    """Host entropy stage on its own (no device needed)."""
    y = np.ascontiguousarray(y, np.int16)
    cb = np.ascontiguousarray(cb if len(cb) else np.zeros((1, 64)), np.int16)
    cr = np.ascontiguousarray(cr if len(cr) else np.zeros((1, 64)), np.int16)
    cap = output_capacity(options.width, options.height)
    buf = np.empty(cap, np.uint8)
    n = C.c_size_t()
    rc = _lib.load().pixo_b200_jpeg_entropy_encode(
        ctx.handle if ctx else None, y.ctypes.data, cb.ctypes.data, cr.ctypes.data,
        int(options.width), int(options.height), int(options.color_type), int(options.quality),
        int(options.subsampling), _restart(options),
        int(bool(options.optimize_huffman)), buf.ctypes.data, cap, C.byref(n))
    _lib.check(ctx.handle if ctx else None, rc)
    return buf[: n.value].tobytes()


def entropy_encode_dev(d_y, d_cb, d_cr, options: JpegOptions, ctx: Context | None = None) -> bytes:
    """Entropy-code coefficient arrays that live on the device (anything with .data_ptr(), e.g.
    int16 torch tensors in compute_all_coefficients' layout, 16-byte aligned) into a complete JPEG:
    Huffman statistics, bit packing, stuffing and restart markers run on the GPU."""
    ctx = ctx or default_context()
    cap = output_capacity(options.width, options.height)
    buf = np.empty(cap, np.uint8)
    n = C.c_size_t()
    ptr = lambda t: None if t is None else int(t.data_ptr())
    rc = _lib.load().pixo_b200_jpeg_entropy_encode_dev(
        ctx.handle, ptr(d_y), ptr(d_cb), ptr(d_cr), int(options.width), int(options.height),
        int(options.color_type), int(options.quality), int(options.subsampling),
        _restart(options), int(bool(options.optimize_huffman)), buf.ctypes.data, cap,
        C.byref(n))
    _lib.check(ctx.handle, rc)
    return buf[: n.value].tobytes()
