"""The encode paths hand the entropy stage coefficient records: zig-zag blocks whose 32-byte sectors
past the last non-zero coefficient are never written, plus a per-block extent (sectors written).
Every reader must take a block's extent from the extent array, so these tests encode in an order that leaves stale
coefficients in the context's buffer - q=100 noise (every sector written), then smooth frames (one
sector), then noise again - and compare every result with the CPU oracle byte for byte."""
import numpy as np
import pytest

import pixo_b200
from pixo_b200 import ColorType, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling

pytestmark = pytest.mark.gpu

W, H = 320, 256
PATHS = [(2, 1), (2, 0), (0, 0)]   # (colour type, subsampling): 4:2:0, 4:4:4, gray
ZZ_NAT = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20,
                   13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52,
                   45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


def _extents(blocks):
    """zig-zag position of each block's last non-zero coefficient (-1: none)"""
    nz = blocks[:, ZZ_NAT] != 0
    return np.where(nz.any(1), 63 - np.argmax(nz[:, ::-1], 1), -1)


def _frames(po, ct):
    """name -> frame of the path's channel count (3: RGB, 1: gray)"""
    ch = 3 if ct == 2 else 1
    yy, xx = np.mgrid[0:H, 0:W]
    # a flat frame with one hard edge, under weak texture that grows from left to right: its blocks
    # end at every zig-zag position, among them both sides of the sector borders 15/16 and 31/32
    k = (1 + xx * 16 // W)[..., None]
    edge = np.full((H, W, 3), 60, np.int32)
    edge[xx + 2 * yy > 200] = 200
    edge = np.clip(edge + po.gen_noise(W, H, 3, 77).reshape(H, W, 3) % (2 * k + 1) - k, 0, 255).astype(np.uint8)
    grad = po.gen_gradient_rgb(W, H).reshape(H, W, 3)
    pick = (lambda a: a.reshape(-1)) if ch == 3 else (lambda a: np.ascontiguousarray(a.reshape(H, W, 3)[..., 0]).reshape(-1))
    return {
        "noise": po.gen_noise(W, H, ch, 5),
        "gradient": pick(grad),
        "flat": np.full(W * H * ch, 117, np.uint8),
        "edge": pick(edge),
        "noise2": po.gen_noise(W, H, ch, 6),
    }


# q=100 noise first: every sector of every block is written; the smooth frames after it write one
SEQUENCE = [("noise", 100), ("gradient", 80), ("flat", 80), ("edge", 80), ("noise2", 80), ("gradient", 90)]


def _scan(jpg: bytes) -> bytes:
    """entropy-coded segment of a baseline file: after the SOS header, before EOI"""
    i = 2
    while True:
        ln = int.from_bytes(jpg[i + 2:i + 4], "big")
        if jpg[i + 1] == 0xDA:
            return jpg[i + 2 + ln:-2]
        i += 2 + ln


def test_edge_frame_reaches_the_sector_borders(po):
    """The edge frame really has blocks that end on both sides of zig-zag positions 16 and 32."""
    for ct, ss in PATHS:
        img = _frames(po, ct)["edge"]
        ext = np.concatenate([_extents(a) for a in po.jpeg_coefficients(img, W, H, ct, ss, 80) if len(a)])
        for p in (15, 16, 31, 32):
            assert (ext == p).any(), (ct, ss, p)


@pytest.mark.parametrize("ct,ss", PATHS)
@pytest.mark.parametrize("ri,opt", [(0, False), (5, False), (0, True), (3, True)])
def test_encode_over_stale_records(po, ct, ss, ri, opt):
    frames = _frames(po, ct)
    with pixo_b200.Context(0) as ctx:
        for name, q in SEQUENCE:
            o = JpegOptions(W, H, ColorType(ct), q, Subsampling(ss), ri or None, opt)
            got = jpeg.encode(frames[name], o, ctx=ctx)
            assert got == po.jpeg_encode(frames[name], W, H, ct, q, ss, ri, opt), (name, q)
        assert ctx.host_fallbacks == 0


@pytest.mark.parametrize("ct,ss", PATHS)
def test_encode_batch_over_stale_records(po, ct, ss):
    frames = _frames(po, ct)
    order = ["noise", "gradient", "flat", "edge", "noise2"]
    with pixo_b200.Context(0) as ctx:
        for q in (100, 80):
            for opt in (False, True):
                batch = np.stack([frames[n] for n in (order if q == 100 else order[::-1])])
                o = JpegOptions(W, H, ColorType(ct), q, Subsampling(ss), None, opt)
                got = jpeg.encode_batch(batch, o, ctx=ctx)
                for k in range(len(batch)):
                    assert got[k] == po.jpeg_encode(batch[k], W, H, ct, q, ss, 0, opt), (q, opt, k)
        assert ctx.host_fallbacks == 0


@pytest.mark.parametrize("ct,ss", PATHS)
def test_segmented_single_frame_over_stale_records(po, ct, ss, monkeypatch):
    """one frame cut into segments (k_huff<RAW> + splice) reads the records too"""
    monkeypatch.setenv("PIXO_B200_SEGMENTS", "5")
    frames = _frames(po, ct)
    with pixo_b200.Context(0) as ctx:
        for name, q in SEQUENCE:
            got = jpeg.encode(frames[name], JpegOptions(W, H, ColorType(ct), q, Subsampling(ss)), ctx=ctx)
            assert got == po.jpeg_encode(frames[name], W, H, ct, q, ss), (name, q)
        assert ctx.host_fallbacks == 0


def test_encode_dev_over_stale_records(po):
    """pixo_b200_jpeg_encode_dev, the device-resident path, on the same sequence (4:2:0 and 4:4:4)"""
    import torch
    from pixo_b200 import _lib
    lib = _lib.load()
    frames = _frames(po, 2)
    cap = jpeg.output_capacity(W, H) // 256 * 256
    for ss in (1, 0):
        with pixo_b200.Context(0) as ctx:
            for name, q in SEQUENCE:
                d_px = torch.from_numpy(frames[name]).cuda()
                d_scan = torch.zeros(cap, dtype=torch.uint8, device="cuda")
                d_len = torch.zeros(1, dtype=torch.int64, device="cuda")
                d_ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                _lib.check(ctx.handle, lib.pixo_b200_jpeg_encode_dev(ctx.handle, d_px.data_ptr(), W * H * 3, 1, W, H, 2, q,
                                                                     ss, d_scan.data_ptr(), cap, d_len.data_ptr(),
                                                                     d_ovf.data_ptr()))
                ctx.sync()
                assert int(d_ovf.cpu()[0]) == 0
                got = d_scan[: int(d_len.cpu()[0])].cpu().numpy().tobytes()
                assert got == _scan(po.jpeg_encode(frames[name], W, H, 2, q, ss)), (ss, name, q)


def test_host_fallback_reads_records(po):
    """the last-resort host coder gets dense arrays from the records: q=100 noise leaves every sector
    of the buffer written, then shorter records are finished by the host coder (retry off, a scan
    buffer too small for them)"""
    frames = _frames(po, 2)
    with pixo_b200.Context(0) as ctx:
        o = JpegOptions(W, H, ColorType.Rgb, 100, Subsampling.S420)
        assert jpeg.encode(frames["noise"], o, ctx=ctx) == po.jpeg_encode(frames["noise"], W, H, 2, 100, 1)
        ctx.set_scan_capacity(1024, gpu_retry=False)
        for name in ("edge", "noise2"):
            ref = po.jpeg_encode(frames[name], W, H, 2, 80, 1)
            assert len(ref) > 4096
            assert jpeg.encode(frames[name], JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420), ctx=ctx) == ref, name
        assert ctx.host_fallbacks == 2
        ctx.set_scan_capacity(0)
