"""Multi-GPU host logic: one process per GPU (torch.distributed over NCCL/NVLink; gloo in the CPU
tests).  Nothing here moves pixels or coefficients between GPUs.

  * batches (BASELINE configs C2/C3/C5): frame i -> rank i % world (`shard_frames`).  Ranks never
    exchange data; only the timing reduction in bench.py is collective.
  * one gigapixel frame (config C4, `encode_tiled`): contiguous bands of MCU rows per rank.  Every
    MCU depends only on its own (clamped) pixels, so a band is transformed as an image of its own
    (bands start on MCU rows: no halo) - the analogue of the reference's
    compute_all_coefficients_parallel (src/jpeg/mod.rs:1137-1215).  The ENTROPY stage is distributed
    too: each rank Huffman-codes its own band into a raw bit string, two tiny all-gathers carry what
    crosses a band boundary (the DC predictors: 3 x i16; the band's bit count and last 7 bits), every
    rank then shifts its string to its bit offset in the frame's stream, completes the byte it
    shares with its predecessor, stuffs 0xFF and (last band) 1-pads, and only the finished scan
    bytes (~1/10 of the raw frame) are gathered to rank 0, which adds headers and EOI.  The file is
    byte-identical to a single-GPU (and to the reference's) encode.
  * PNG filter stream + Adler-32 of one image in row bands (`adler32_combine`): each band's
    checksum over its slice of the filtered stream, combined in band order.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from . import _lib


def shard_frames(n_frames: int, world: int, rank: int) -> list[int]:
    """Frame indices owned by `rank` (round robin keeps ragged batches balanced)."""
    return list(range(rank, n_frames, world))


@dataclasses.dataclass
class Band:
    rank: int
    mcu_row0: int
    mcu_row1: int      # exclusive
    px_row0: int
    px_row1: int       # exclusive, clipped to the image height
    y_blocks: int
    c_blocks: int


def plan_bands(width: int, height: int, world: int, gray: bool = False, s420: bool = True) -> list[Band]:
    """Contiguous MCU-row bands, as equal as possible; ranks beyond the number of MCU rows get
    empty bands."""
    mcu = 16 if (s420 and not gray) else 8
    mcus_x = (width + mcu - 1) // mcu
    mcus_y = (height + mcu - 1) // mcu
    ypm = 4 if (s420 and not gray) else 1
    bands = []
    for r in range(world):
        r0 = mcus_y * r // world
        r1 = mcus_y * (r + 1) // world
        n = (r1 - r0) * mcus_x
        bands.append(Band(r, r0, r1, r0 * mcu, min(r1 * mcu, height), n * ypm, 0 if gray else n))
    return bands


def band_pixels(frame: np.ndarray, width: int, height: int, bpp: int, band: Band) -> np.ndarray:
    """The rows of `frame` a band needs (a view): bands are MCU aligned, so no halo rows."""
    rows = np.asarray(frame, np.uint8).reshape(height, width * bpp)
    return rows[band.px_row0:band.px_row1]


# ---- what crosses a band boundary ----------------------------------------------------------------

def dc_seeds(last_dcs: np.ndarray, nonempty: list[bool], rank: int) -> np.ndarray:
    """DC predictors band `rank` starts from: the last DCs of the nearest non-empty band before it
    (0 for the first).  last_dcs: [world, 3]."""
    for r in range(rank - 1, -1, -1):
        if nonempty[r]:
            return np.asarray(last_dcs[r], np.int32).copy()
    return np.zeros(3, np.int32)


def bit_offsets(nbits: list[int], tails: list[int], rank: int) -> tuple[int, int, bool]:
    """(start_bit, tail_in, is_last) of band `rank` in the frame's stream.  start_bit = bits of all
    bands before it; tail_in = the last start_bit % 8 bits of the stream so far, taken from the
    nearest non-empty band (a non-empty band holds at least one MCU, i.e. more than 7 bits)."""
    start = int(sum(nbits[:rank]))
    s = start & 7
    tail_in = 0
    if s:
        for r in range(rank - 1, -1, -1):
            if nbits[r]:
                assert nbits[r] >= 7
                tail_in = int(tails[r]) & ((1 << s) - 1)
                break
    is_last = not any(nbits[r] for r in range(rank + 1, len(nbits)))
    return start, tail_in, is_last


class DeviceBandCoder:
    """The band stages on this rank's GPU (libpixo_b200: K3, k_huff<RAW>, k_seg_*)."""

    def __init__(self, ctx, d_y, d_cb, d_cr, width, band_height, color_type, subsampling, ny, nc):
        import torch
        self.ctx, self.lib, self.torch = ctx, _lib.load(), torch
        self.d_y, self.d_cb, self.d_cr = d_y, d_cb, d_cr
        self.geo = (int(width), int(band_height), int(color_type), int(subsampling))
        self.ny, self.nc = int(ny), int(nc)
        self.dev = d_y.device
        self.raw = None
        self.out = None

    def _p(self, t):
        return None if t is None else int(t.data_ptr())

    def last_dc(self) -> np.ndarray:
        out = (C.c_int32 * 3)()
        _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_last_dc(
            self.ctx.handle, self._p(self.d_y), self._p(self.d_cb), self._p(self.d_cr), self.ny, self.nc, out))
        return np.array(out[:], np.int32)

    def histogram(self, seed: np.ndarray):
        """536 counters of this band (torch int64 on the device, ready for all_reduce)."""
        # (the library clears the counters itself, on ITS stream: a torch-side fill could land after it)
        hist = self.torch.empty(536, dtype=self.torch.int64, device=self.dev)
        if not self.ny:
            hist.zero_()
        if self.ny:
            s = (C.c_int32 * 3)(*[int(v) for v in seed])
            _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_histogram_dev(
                self.ctx.handle, self._p(self.d_y), self._p(self.d_cb), self._p(self.d_cr), *self.geo, s,
                int(hist.data_ptr())))
            self.ctx.sync()
        return hist

    def entropy(self, seed: np.ndarray, hist: np.ndarray | None) -> tuple[int, int]:
        if not self.ny:
            return 0, 0
        w, bh = self.geo[0], self.geo[1]
        # as many bytes as the band's pixels + 1 MiB: lets a long band be coded in segments (short
        # look-back chains), whose raw strings need more room than the finished JPEG; grown on demand
        cap = (w * bh * 3 + (1 << 20)) // 16 * 16
        s = (C.c_int32 * 3)(*[int(v) for v in seed])
        hp = None if hist is None else np.ascontiguousarray(hist, np.uint64).ctypes.data_as(_lib.u64p)
        for _ in range(2):
            if self.raw is None or self.raw.numel() < cap:
                self.raw = self.torch.empty(cap, dtype=self.torch.uint8, device=self.dev)
            cap = self.raw.numel() // 16 * 16
            nbits, tail = C.c_uint64(), C.c_uint32()
            rc = self.lib.pixo_b200_jpeg_band_entropy_dev(
                self.ctx.handle, self._p(self.d_y), self._p(self.d_cb), self._p(self.d_cr), *self.geo, s, hp,
                int(self.raw.data_ptr()), cap, C.byref(nbits), C.byref(tail))
            if rc == _lib.ERR_OUTPUT_TOO_SMALL:
                cap = ((nbits.value + 7) // 8 + 4096) // 16 * 16
                continue
            _lib.check(self.ctx.handle, rc)
            return int(nbits.value), int(tail.value)
        _lib.check(self.ctx.handle, rc)

    def splice(self, nbits, start_bit, tail_in, is_last):
        """-> uint8 tensor (device) of this band's finished scan bytes."""
        cap = (nbits + 7) // 8 * 2 + 64     # worst case: every byte stuffed
        if self.out is None or self.out.numel() < cap:
            self.out = self.torch.empty(cap, dtype=self.torch.uint8, device=self.dev)
        n = C.c_uint64()
        _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_splice_dev(
            self.ctx.handle, self._p(self.raw) if self.raw is not None else None, nbits, start_bit, tail_in,
            int(is_last), int(self.out.data_ptr()), self.out.numel(), C.byref(n)))
        return self.out[: n.value]


class HostBandCoder:
    """The same stages from host arrays through the library's host twins (no device): the CPU-only
    world_size-2 tests run the collective logic with it."""

    def __init__(self, y, cb, cr, width, band_height, color_type, subsampling):
        import torch
        self.lib, self.torch = _lib.load(), torch
        self.y = np.ascontiguousarray(y, np.int16).reshape(-1, 64)
        self.cb = np.ascontiguousarray(cb, np.int16).reshape(-1, 64)
        self.cr = np.ascontiguousarray(cr, np.int16).reshape(-1, 64)
        self.geo = (int(width), int(band_height), int(color_type), int(subsampling))
        self.ny = self.y.shape[0]
        self.dev = torch.device("cpu")
        self.raw = None

    def _ptrs(self):
        z = np.zeros((1, 64), np.int16)
        cb = self.cb if len(self.cb) else z
        cr = self.cr if len(self.cr) else z
        self._keep = (cb, cr)
        return self.y.ctypes.data, cb.ctypes.data, cr.ctypes.data

    def last_dc(self) -> np.ndarray:
        v = [int(a[-1, 0]) if len(a) else 0 for a in (self.y, self.cb, self.cr)]
        return np.array(v, np.int32)

    def histogram(self, seed):
        hist = np.zeros(536, np.uint64)
        if self.ny:
            s = (C.c_int32 * 3)(*[int(v) for v in seed])
            _lib.check(None, self.lib.pixo_b200_jpeg_band_histogram(*self._ptrs(), *self.geo, s,
                                                                    hist.ctypes.data_as(_lib.u64p)))
        return self.torch.from_numpy(hist.astype(np.int64))

    def entropy(self, seed, hist):
        if not self.ny:
            return 0, 0
        cap = self.y.size * 4 + self.cb.size * 8 + 4096
        self.raw = np.zeros(cap, np.uint8)
        s = (C.c_int32 * 3)(*[int(v) for v in seed])
        hp = None if hist is None else np.ascontiguousarray(hist, np.uint64).ctypes.data_as(_lib.u64p)
        nbits, tail = C.c_uint64(), C.c_uint32()
        _lib.check(None, self.lib.pixo_b200_jpeg_band_entropy(*self._ptrs(), *self.geo, s, hp, self.raw.ctypes.data,
                                                              cap, C.byref(nbits), C.byref(tail)))
        return int(nbits.value), int(tail.value)

    def splice(self, nbits, start_bit, tail_in, is_last):
        cap = (nbits + 7) // 8 * 2 + 64
        out = np.zeros(cap, np.uint8)
        n = C.c_size_t()
        _lib.check(None, self.lib.pixo_b200_jpeg_band_splice(self.raw.ctypes.data if self.raw is not None else None,
                                                             nbits, start_bit, tail_in, int(is_last), out.ctypes.data,
                                                             cap, C.byref(n)))
        return self.torch.from_numpy(out[: n.value])


def write_headers(width, height, color_type, quality, subsampling, hist=None) -> bytes:
    buf = np.zeros(2048, np.uint8)
    n = C.c_size_t()
    hp = None if hist is None else np.ascontiguousarray(hist, np.uint64).ctypes.data_as(_lib.u64p)
    _lib.check(None, _lib.load().pixo_b200_jpeg_write_headers(int(width), int(height), int(color_type), int(quality),
                                                              int(subsampling), 0, hp, buf.ctypes.data, buf.size,
                                                              C.byref(n)))
    return buf[: n.value].tobytes()


def encode_tiled(coder, width: int, height: int, color_type: int, quality: int, subsampling: int,
                 optimize_huffman: bool, rank: int, world: int, dst: int = 0):
    """Distributed entropy stage of one tiled frame: the complete JPEG on `dst`, None elsewhere."""
    parts, hist = tiled_scan_parts(coder, optimize_huffman, rank, world, dst)
    if rank != dst:
        return None
    return assemble_tiled(parts, hist, width, height, color_type, quality, subsampling)


def assemble_tiled(parts, hist, width, height, color_type, quality, subsampling) -> bytes:
    """Host side of the last step: headers + the bands' scan bytes (device or host tensors) + EOI."""
    import torch
    scan = torch.cat([p.cpu() for p in parts]).numpy().tobytes() if parts else b""
    return write_headers(width, height, color_type, quality, subsampling, hist) + scan + b"\xff\xd9"


def tiled_scan_parts(coder, optimize_huffman: bool, rank: int, world: int, dst: int = 0):
    """The device part of `encode_tiled`.  `coder` holds this rank's band (coefficients already
    computed).  Returns (the bands' finished scan bytes in band order as tensors on dst's device -
    None on the other ranks -, the summed histogram or None).  Collectives: all_gather of 4 ints (DC
    predictors), [all_reduce of 536 counters], all_gather of 2 ints (bits, tail), all_gather of 1 int
    (byte counts), gather of the scan bytes (only dst receives)."""
    import torch
    import torch.distributed as dist
    dev = coder.dev

    def all_gather_ints(vals):
        t = torch.tensor(vals, dtype=torch.int64, device=dev)
        if world == 1:
            return t.reshape(1, -1).cpu().numpy()
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t)
        return torch.stack(out).cpu().numpy()

    ld = coder.last_dc()
    g = all_gather_ints([int(ld[0]), int(ld[1]), int(ld[2]), int(coder.ny > 0)])
    seed = dc_seeds(g[:, :3], [bool(v) for v in g[:, 3]], rank)
    hist = None
    if optimize_huffman:
        h = coder.histogram(seed)
        if world > 1:
            dist.all_reduce(h, op=dist.ReduceOp.SUM)
        hist = h.cpu().numpy().astype(np.uint64)
    nbits, tail = coder.entropy(seed, hist)
    g = all_gather_ints([nbits, tail])
    start, tail_in, is_last = bit_offsets([int(v) for v in g[:, 0]], [int(v) for v in g[:, 1]], rank)
    if nbits == 0:
        is_last = False          # an empty band owns nothing; the last NON-empty band pads
    body = coder.splice(nbits, start, tail_in, is_last) if nbits else torch.empty(0, dtype=torch.uint8, device=dev)
    sizes = all_gather_ints([int(body.numel())])[:, 0]
    if world == 1:
        parts = [body]
    else:
        mx = int(max(sizes.max(), 1))
        pad = torch.zeros(mx, dtype=torch.uint8, device=dev)
        pad[: body.numel()] = body
        bufs = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
        dist.gather(pad, bufs, dst=dst)      # every rank sends its (padded) bytes, only dst receives
        parts = [bufs[r][: int(sizes[r])] for r in range(world)] if rank == dst else None
    return (parts if rank == dst else None), hist


class ThreadComm:
    """all_gather / gather among `world` THREADS of one process (one band per thread, every band with
    a context of its own on the same GPU): lets the multi-rank flow run - collectives included - where
    there is only one device.  Device work is synchronised before tensors change hands."""

    def __init__(self, world: int):
        import threading
        self.world = world
        self.slots = [None] * world
        self.barrier = threading.Barrier(world)

    def all_gather(self, rank, t):
        import torch
        torch.cuda.current_stream().synchronize()
        self.slots[rank] = t
        self.barrier.wait()
        out = torch.stack([x.clone() for x in self.slots])
        torch.cuda.current_stream().synchronize()
        self.barrier.wait()
        return out

    def gather(self, rank, t, dst):
        allv = self.all_gather(rank, t)
        return [allv[r] for r in range(self.world)] if rank == dst else None

    def all_reduce_sum(self, rank, t):
        return self.all_gather(rank, t).sum(0)


class _DistComm:
    def __init__(self, world):
        self.world = world

    def all_gather(self, rank, t):
        import torch
        import torch.distributed as dist
        if self.world == 1:
            return t.reshape(1, *t.shape)
        out = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(out, t)
        return torch.stack(out)

    def gather(self, rank, t, dst):
        import torch
        import torch.distributed as dist
        if self.world == 1:
            return [t]
        bufs = [torch.empty_like(t) for _ in range(self.world)] if rank == dst else None
        dist.gather(t, bufs, dst=dst)
        return bufs

    def all_reduce_sum(self, rank, t):
        import torch.distributed as dist
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return t


def tiled_scan_parts_async(coder, nonempty: list[bool], rank: int, world: int, dst: int = 0, comm=None):
    """`tiled_scan_parts` without host round trips: every value that crosses a band boundary stays
    on the device (pixo_b200_jpeg_band_*_async), the collectives are queued on the same stream as the
    kernels, and the host waits once - for the byte counts it needs to size the final gather.
    Standard Huffman tables only (optimised tables need the all-reduced statistics on the host).
    `coder` is a DeviceBandCoder whose context runs on torch's current stream; nonempty[r] = band r
    holds at least one MCU (known from the band plan)."""
    import torch
    dev, lib, ctx = coder.dev, coder.lib, coder.ctx
    i64 = torch.int64
    comm = comm or _DistComm(world)
    all_gather = lambda t: comm.all_gather(rank, t)

    prev = next((r for r in range(rank - 1, -1, -1) if nonempty[r]), None)
    is_last = coder.ny > 0 and not any(nonempty[rank + 1:])
    # 1. DC predictors: the last DC of every band's three arrays
    if coder.ny:
        ld = torch.stack([coder.d_y[coder.ny - 1, 0], coder.d_cb[coder.nc - 1, 0] if coder.nc else coder.d_y[0, 0] * 0,
                          coder.d_cr[coder.nc - 1, 0] if coder.nc else coder.d_y[0, 0] * 0]).to(torch.int32)
    else:
        ld = torch.zeros(3, dtype=torch.int32, device=dev)
    g = all_gather(ld)
    seed = (g[prev] if prev is not None else torch.zeros(3, dtype=torch.int32, device=dev)).contiguous()
    # 2. this band's code as a raw bit string
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    bits_tail = torch.zeros(2, dtype=i64, device=dev)
    if coder.ny:
        w, bh = coder.geo[0], coder.geo[1]
        cap = (w * bh * 3 + (1 << 20)) // 16 * 16
        if coder.raw is None or coder.raw.numel() < cap:
            coder.raw = torch.empty(cap, dtype=torch.uint8, device=dev)
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_band_entropy_dev_async(
            ctx.handle, coder._p(coder.d_y), coder._p(coder.d_cb), coder._p(coder.d_cr), *coder.geo, int(seed.data_ptr()),
            None, int(coder.raw.data_ptr()), coder.raw.numel() // 16 * 16, int(bits_tail.data_ptr()), int(flags.data_ptr())))
    # 3. bit offsets: bits of all bands before this one; the previous non-empty band's last 7 bits
    bt = all_gather(bits_tail)
    start = bt[:rank, 0].sum() if rank else torch.zeros((), dtype=i64, device=dev)
    tail_prev = bt[prev, 1] if prev is not None else torch.zeros((), dtype=i64, device=dev)
    offset = torch.stack([start, tail_prev, torch.full((), int(is_last), dtype=i64, device=dev)]).contiguous()
    # 4. splice
    out_len = torch.zeros(1, dtype=i64, device=dev)
    if coder.ny:
        cap = coder.raw.numel() * 2 + 64
        if coder.out is None or coder.out.numel() < cap:
            coder.out = torch.empty(cap, dtype=torch.uint8, device=dev)
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_band_splice_dev_async(
            ctx.handle, int(coder.raw.data_ptr()), int(offset.data_ptr()), int(coder.out.data_ptr()), coder.out.numel(),
            int(out_len.data_ptr()), int(flags.data_ptr())))
    # 5. the one host wait: byte counts (and flags) of all bands
    info = all_gather(torch.cat([out_len, flags.to(i64)])).cpu().numpy()
    if int(info[:, 1].max()):
        raise _lib.PixoError(_lib.ERR_CUDA, f"band entropy stage reported flags {info[:, 1].tolist()}")
    sizes = info[:, 0]
    body = coder.out[: int(sizes[rank])] if coder.ny else torch.empty(0, dtype=torch.uint8, device=dev)
    if world == 1:
        return [body], None
    mx = int(max(sizes.max(), 1))
    pad = torch.zeros(mx, dtype=torch.uint8, device=dev)
    pad[: body.numel()] = body
    bufs = comm.gather(rank, pad, dst)
    return ([bufs[r][: int(sizes[r])] for r in range(world)] if rank == dst else None), None


def encode_tiled_local(coders: list, width: int, height: int, color_type: int, quality: int, subsampling: int,
                       optimize_huffman: bool = False) -> bytes:
    """The same stage sequence with every band in THIS process (one GPU context, or the host
    twins): what `encode_tiled` does across ranks, minus the collectives.  Used at world size 1
    (bench.py's C4 line on one GPU, the single-device tests)."""
    parts, hist = tiled_scan_parts_local(coders, optimize_huffman)
    return assemble_tiled(parts, hist, width, height, color_type, quality, subsampling)


def tiled_scan_parts_local(coders: list, optimize_huffman: bool = False):
    import torch
    world = len(coders)
    last = np.stack([c.last_dc() for c in coders])
    nonempty = [c.ny > 0 for c in coders]
    seeds = [dc_seeds(last, nonempty, r) for r in range(world)]
    hist = None
    if optimize_huffman:
        hist = sum(c.histogram(seeds[r]).cpu().numpy().astype(np.uint64) for r, c in enumerate(coders))
    coded = [c.entropy(seeds[r], hist) for r, c in enumerate(coders)]
    nbits = [n for n, _ in coded]
    tails = [t for _, t in coded]
    parts = []
    for r, c in enumerate(coders):
        if not nbits[r]:
            continue
        start, tail_in, is_last = bit_offsets(nbits, tails, r)
        parts.append(c.splice(nbits[r], start, tail_in, is_last))
    return parts, hist


# ---- the progressive scans of one tiled frame (pixo's max preset) -------------------------------------
# A band of whole MCU rows is a contiguous range of every component's array (4:2:0 Y in MCU order too), so each of
# the 7 scans of simple_progressive_script codes the band's range on its own once three things cross in from the
# bands before it: the DC predictors (DC scans), the EOB run pending at the band's start (AC scans) and the bit
# offset in the scan's stream.  Each rank codes its band into 7 raw strings (pixo_b200_jpeg_band_dev_progressive),
# splices every scan at its offset (k_seg_*), and dst writes the file with the segments in scan-major order.

PROG_SCANS = 7
PROG_SCAN_COMP = (0, 1, 2, 0, 0, 1, 2)   # the component of each scan: Y DC, Cb DC, Cr DC, Y 1-10, Y 11-63, Cb, Cr


def prog_dc_seeds(last_dcs, counts, rank: int) -> np.ndarray:
    """DC predictors band `rank` starts from, per component: the last DC of the nearest earlier band that has
    blocks of that component (0 for none; pixo never resets them).  last_dcs, counts: [world, 3] (blocks of Y, Cb,
    Cr)."""
    seed = np.zeros(3, np.int32)
    for c in range(3):
        for r in range(rank - 1, -1, -1):
            if int(counts[r][c]):
                seed[c] = int(last_dcs[r][c])
                break
    return seed


def ac_carries(last_encs, rank: int) -> np.ndarray:
    """The EOB-run carry of band `rank` in each AC scan (Y 1-10, Y 11-63, Cb, Cr): the largest
    ((frame index + 1) << 1 | init) over the earlier bands' last non-empty blocks, 0 for none.  last_encs: [world, 4]
    (pixo_b200_jpeg_band_dev_progressive_summary's last_enc of every band)."""
    out = np.zeros(4, np.uint32)
    for r in range(rank):
        out = np.maximum(out, np.asarray(last_encs[r], np.uint32))
    return out


def scan_bit_offsets(nbits, tails, rank: int) -> tuple[int, int, bool]:
    """(start_bit, tail_in, is_last) of band `rank` in ONE scan's stream: `bit_offsets` for bands that may write fewer
    than 7 bits of a scan (a tail then holds all of its band's bits), so the bits inherited in the first byte can
    come from several bands.  is_last: the band writes the scan's last bit (and 1-pads it)."""
    start = int(sum(int(n) for n in nbits[:rank]))
    need = start & 7
    tail_in = have = 0
    for r in range(rank - 1, -1, -1):
        if have >= need:
            break
        take = min(int(nbits[r]), need - have)
        tail_in |= (int(tails[r]) & ((1 << take) - 1)) << have
        have += take
    is_last = bool(int(nbits[rank])) and not any(int(n) for n in nbits[rank + 1:])
    return start, tail_in, is_last


def band_bases(bands: list[Band], rank: int) -> tuple[int, int]:
    """Frame index of band `rank`'s first Y block and first chroma block."""
    return sum(b.y_blocks for b in bands[:rank]), sum(b.c_blocks for b in bands[:rank])


class ProgressiveBandCoder:
    """One rank's band of a progressive frame on its device (pixo_b200_jpeg_band_dev_progressive*).  coded: the band's
    (y, cb, cr) int16 device arrays to code (natural order, the trellis arrays under trellis_quant); plain: the
    plain-rounded arrays the optimised tables are counted from (None: the coded ones).  ny / nc: the band's blocks,
    y_base / c_base the frame index of its first ones, frame_ny / frame_nc the frame's (frame_nc 0: gray).
    geometry (width, band_height, color_type, subsampling) is needed for the table statistics only."""

    def __init__(self, ctx, coded, ny, nc, y_base, c_base, frame_ny, frame_nc, plain=None, geometry=None):
        import torch
        self.ctx, self.lib, self.torch = ctx, _lib.load(), torch
        self.coded = tuple(coded)
        self.plain = tuple(plain) if plain is not None else None
        self.ny, self.nc = int(ny), int(nc)
        self.y_base, self.c_base = int(y_base), int(c_base)
        self.frame_ny, self.frame_nc = int(frame_ny), int(frame_nc)
        self.geometry = geometry
        self.dev = self.coded[0].device
        self.raw = None
        self.dht = torch.empty(1088, dtype=torch.uint8, device=self.dev)

    @staticmethod
    def _p(t):
        return None if t is None else int(t.data_ptr())

    def _arrays(self, arrs):
        y, cb, cr = arrs
        return self._p(y), self._p(cb) if self.nc else None, self._p(cr) if self.nc else None

    def summary(self) -> list[int]:
        """[plain last DC x 3, coded last DC x 3, last_enc x 4, ny, nc]: what the later bands need from this one."""
        dc, enc = (C.c_int32 * 3)(), (C.c_uint32 * 4)()
        _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_dev_progressive_summary(
            self.ctx.handle, *self._arrays(self.coded), self.ny, self.nc, self.y_base, self.c_base, dc, enc))
        plain = list(dc)
        if self.plain is not None:
            pdc = (C.c_int32 * 3)()
            _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_last_dc(
                self.ctx.handle, *self._arrays(self.plain), self.ny, self.nc, pdc))
            plain = list(pdc)
        return plain + list(dc) + list(enc) + [self.ny, self.nc]

    def histogram(self, seed):
        """536 baseline counters of the plain arrays from DC predictors `seed` (torch int64 on the device)."""
        hist = self.torch.zeros(536, dtype=self.torch.int64, device=self.dev)
        if self.ny:
            if self.geometry is None:
                raise _lib.PixoError(_lib.ERR_INVALID_ARGUMENT, "optimised tables need the band's geometry")
            self.torch.cuda.current_stream(self.dev).synchronize()
            s = (C.c_int32 * 3)(*[int(v) for v in seed])
            _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_histogram_dev(
                self.ctx.handle, *self._arrays(self.plain or self.coded), *[int(v) for v in self.geometry], s,
                int(hist.data_ptr())))
            self.ctx.sync()
        return hist

    def code(self, seed, carry, hist=None) -> tuple[list[int], list[int]]:
        """The band's 7 raw strings from DC predictors `seed`, EOB-run carries `carry` and the frame's summed
        statistics `hist` (device int64 [536]; None: standard tables) -> (bits, tails) per scan.  self.dht then
        holds the tables."""
        if hist is not None:
            self.torch.cuda.current_stream(self.dev).synchronize()   # (an all-reduce on torch's stream)
        s = (C.c_int32 * 3)(*[int(v) for v in seed])
        cy = (C.c_uint32 * 4)(*[int(v) for v in carry])
        need, nbits, tails = C.c_size_t(), (C.c_uint64 * 7)(), (C.c_uint32 * 7)()
        if self.raw is None and (self.ny or self.nc):
            self.raw = self.torch.empty(((self.ny + 2 * self.nc) * 48 + 7 * 4096) // 16 * 16, dtype=self.torch.uint8,
                                        device=self.dev)
        for _ in range(2):
            rc = self.lib.pixo_b200_jpeg_band_dev_progressive(
                self.ctx.handle, *self._arrays(self.coded), self.ny, self.nc, self.y_base, self.c_base, self.frame_ny,
                self.frame_nc, s, cy, self._p(hist), self._p(self.dht), self._p(self.raw),
                0 if self.raw is None else self.raw.numel(), C.byref(need), nbits, tails)
            if rc != _lib.ERR_OUTPUT_TOO_SMALL:
                break
            self.raw = self.torch.empty(need.value, dtype=self.torch.uint8, device=self.dev)
        _lib.check(self.ctx.handle, rc)
        return list(nbits), list(tails)

    def splice(self, scan, nbits, start_bit, tail_in, is_last):
        """-> uint8 device tensor: this band's finished bytes of scan `scan`."""
        out = self.torch.empty((nbits + 7) // 8 * 2 + 64, dtype=self.torch.uint8, device=self.dev)
        n = C.c_uint64()
        _lib.check(self.ctx.handle, self.lib.pixo_b200_jpeg_band_dev_progressive_splice(
            self.ctx.handle, self._p(self.raw), int(scan), int(nbits), int(start_bit), int(tail_in), int(is_last),
            int(out.data_ptr()), out.numel(), C.byref(n)))
        return out[: n.value]


def band_coefficients(ctx, d_pixels, width: int, band_height: int, color_type: int, subsampling: int, quality: int,
                      trellis: bool):
    """The band's coefficient arrays from its pixel rows (device uint8, band_height x width x bpp): (plain, coded),
    each (y, cb, cr) int16 device tensors [max(n, 1), 64] - plain-rounded, and COEF_TRELLIS ones when `trellis`
    (coded is plain otherwise)."""
    import torch
    from . import jpeg
    lib = _lib.load()
    dev = d_pixels.device
    ny, nc = jpeg.block_counts(width, band_height, color_type, subsampling) if band_height else (0, 0)
    _, _, lq, cq = jpeg.quant_tables(quality)

    def arrays(flags):
        a = [torch.empty((max(n, 1), 64), dtype=torch.int16, device=dev) for n in (ny, nc, nc)]
        if ny:
            torch.cuda.current_stream(dev).synchronize()   # torch's stream is not the context's
            _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
                ctx.handle, int(d_pixels.data_ptr()), d_pixels.numel(), 1, width, band_height, color_type, subsampling,
                lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p), int(a[0].data_ptr()), ny * 64,
                int(a[1].data_ptr()), int(a[2].data_ptr()), nc * 64, flags, None))
            ctx.sync()
        return tuple(a)

    plain = arrays(0)
    return plain, (arrays(2) if trellis else plain)   # 2: COEF_TRELLIS


def progressive_band_coder(ctx, d_pixels, width: int, height: int, color_type: int, subsampling: int, quality: int,
                           trellis: bool, bands: list[Band], rank: int) -> ProgressiveBandCoder:
    """Band `rank` of plan_bands(width, height, ...) from its pixel rows on its device: transform (and trellis),
    then its coder."""
    b = bands[rank]
    bh = b.px_row1 - b.px_row0
    plain, coded = band_coefficients(ctx, d_pixels, width, bh, color_type, subsampling, quality, trellis)
    yb, cb = band_bases(bands, rank)
    return ProgressiveBandCoder(ctx, coded, b.y_blocks, b.c_blocks, yb, cb, sum(x.y_blocks for x in bands),
                                sum(x.c_blocks for x in bands), plain if trellis else None,
                                (width, max(bh, 1), color_type, subsampling))


def _check_progressive_options(options):
    from . import jpeg
    if jpeg._restart(options):
        raise _lib.PixoError(_lib.ERR_UNSUPPORTED, "a restart interval on a tiled progressive frame")


def tiled_progressive_parts(coder, optimize_huffman: bool, rank: int, world: int, dst: int = 0, comm=None):
    """The progressive scans of one tiled frame, this rank's band in `coder` (ProgressiveBandCoder).  Returns, on
    dst, (the 7 segments back to back as a uint8 tensor on dst's device, their 7 lengths, the tables as 1088 bytes)
    and None elsewhere.  Collectives (through `comm`: torch.distributed by default, or ThreadComm): all-gather of
    the summaries, [all-reduce of the 536 counters], all-gather of 7 x (bits, tail), all-gather of 7 byte counts,
    gather of the bytes to dst."""
    import torch
    comm = comm or _DistComm(world)
    dev = coder.dev

    def all_gather(vals):
        return comm.all_gather(rank, torch.tensor([int(v) for v in vals], dtype=torch.int64, device=dev)).cpu().numpy()

    s = all_gather(coder.summary())
    counts = s[:, [10, 11, 11]]
    hist = None
    if optimize_huffman:
        hist = comm.all_reduce_sum(rank, coder.histogram(prog_dc_seeds(s[:, 0:3], counts, rank)))
    nbits, tails = coder.code(prog_dc_seeds(s[:, 3:6], counts, rank), ac_carries(s[:, 6:10], rank), hist)
    bt = all_gather(nbits + tails).reshape(world, 2, PROG_SCANS)
    bodies = []
    for k in range(PROG_SCANS):
        start, tail_in, is_last = scan_bit_offsets(bt[:, 0, k], bt[:, 1, k], rank)
        bodies.append(coder.splice(k, nbits[k], start, tail_in, is_last))
    sizes = all_gather([b.numel() for b in bodies])            # [world, 7]
    pad = torch.zeros(max(int(sizes.sum(1).max()), 1), dtype=torch.uint8, device=dev)
    body = torch.cat(bodies)
    pad[: body.numel()] = body
    bufs = comm.gather(rank, pad, dst)
    if rank != dst:
        return None
    segs = []
    for k in range(PROG_SCANS):                                 # scan-major: every band's bytes of scan k
        for r in range(world):
            off = int(sizes[r, :k].sum())
            segs.append(bufs[r][off: off + int(sizes[r, k])])
    return torch.cat(segs), [int(v) for v in sizes.sum(0)], coder.dht.cpu().numpy()


def encode_progressive_tiled(coder, options, rank: int, world: int, dst: int = 0, comm=None):
    """One frame tiled over `world` ranks as the progressive file pixo writes for `options` (JpegOptions; its
    geometry, quality and optimize_huffman; trellis_quant decides the coder's arrays): the file on dst, None
    elsewhere.  A restart interval raises ERR_UNSUPPORTED."""
    from . import jpeg
    _check_progressive_options(options)
    parts = tiled_progressive_parts(coder, bool(options.optimize_huffman), rank, world, dst, comm)
    if parts is None:
        return None
    seg, lens, dht = parts
    return jpeg.progressive_file(options, dht, seg.cpu().numpy(), lens)


def tiled_progressive_parts_local(coders: list, optimize_huffman: bool = False):
    """tiled_progressive_parts with every band in THIS process (one device): (segments, lengths, tables)."""
    import torch
    world = len(coders)
    s = np.array([c.summary() for c in coders], np.int64)
    counts = s[:, [10, 11, 11]]
    hist = None
    if optimize_huffman:
        hist = sum(c.histogram(prog_dc_seeds(s[:, 0:3], counts, r)) for r, c in enumerate(coders))
    coded = [c.code(prog_dc_seeds(s[:, 3:6], counts, r), ac_carries(s[:, 6:10], r), hist) for r, c in enumerate(coders)]
    nb = np.array([n for n, _ in coded], np.int64)
    tl = np.array([t for _, t in coded], np.int64)
    segs, lens = [], [0] * PROG_SCANS
    for k in range(PROG_SCANS):
        for r, c in enumerate(coders):
            start, tail_in, is_last = scan_bit_offsets(nb[:, k], tl[:, k], r)
            part = c.splice(k, int(nb[r, k]), start, tail_in, is_last)
            segs.append(part)
            lens[k] += part.numel()
    dev = coders[0].dev
    return torch.cat(segs) if segs else torch.empty(0, dtype=torch.uint8, device=dev), lens, coders[0].dht.cpu().numpy()


def encode_progressive_tiled_local(coders: list, options) -> bytes:
    """encode_progressive_tiled with every band in this process."""
    from . import jpeg
    _check_progressive_options(options)
    seg, lens, dht = tiled_progressive_parts_local(coders, bool(options.optimize_huffman))
    return jpeg.progressive_file(options, dht, seg.cpu().numpy(), lens)


# ---- Adler-32 of a stream held in pieces (PNG filter stage in row bands) ----------------------------

ADLER_MOD = 65521


def adler32_combine(parts: list[tuple[int, int]]) -> int:
    """Combine per-piece Adler-32 values, in stream order.  parts: (adler32 of the piece computed
    from the initial state s1=1,s2=0 as compress::adler32::adler32 does - src/compress/adler32.rs:26-47 -,
    piece length).  For pieces A then B:  s1 = s1A + s1B - 1,  s2 = s2A + s2B + lenB * (s1A - 1)  (mod 65521)."""
    s1, s2 = 1, 0
    for ad, ln in parts:
        b1, b2 = ad & 0xFFFF, (ad >> 16) & 0xFFFF
        s2 = (s2 + b2 + (ln % ADLER_MOD) * (s1 - 1)) % ADLER_MOD
        s1 = (s1 + b1 - 1) % ADLER_MOD
    return (s2 << 16) | s1
