"""The host encode calls over three groups of frames.  A batch is cut into groups (8 frames of 2048x2048 RGB:
about 96 MB of input per group, at least two groups per call), and a group's pixels and coefficient records
reuse the slots of the group two before it.  These batches have 20 frames, so the third group reuses both
slots.  Its q=100 noise frames outgrow the device scan buffer and are coded a second time from their
coefficients in the reused slot.  Every file is compared byte for byte with the CPU oracle."""
import numpy as np
import pytest

import pixo_b200
from pixo_b200 import ColorType, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling

pytestmark = pytest.mark.gpu

W = H = 2048
N = 20              # groups of 8, 8 and 4 frames
NOISE = (17, 19)    # in the third group, among gradients
Q = 100


@pytest.fixture(scope="module")
def frames(po):
    grad = po.gen_gradient_rgb(W, H).reshape(H, W, 3)
    out = [po.gen_noise(W, H, 3, 40 + k) if k in NOISE else np.roll(grad, 37 * k, axis=1).reshape(-1) for k in range(N)]
    assert len(po.jpeg_encode(out[NOISE[0]], W, H, 2, Q, 1)) > (W * H * 3 // 2 + 65536) * 9 // 8   # beyond the heuristic
    return np.stack(out)


def _header_len(jpg: bytes) -> int:
    """bytes of a baseline file before its entropy-coded segment"""
    i = 2
    while True:
        ln = int.from_bytes(jpg[i + 2:i + 4], "big")
        if jpg[i + 1] == 0xDA:
            return i + 2 + ln
        i += 2 + ln


@pytest.mark.parametrize("ri,opt", [(None, False), (4, True)])
def test_encode_batch_over_three_groups(po, frames, ri, opt):
    o = JpegOptions(W, H, ColorType.Rgb, Q, Subsampling.S420, ri, opt)
    with pixo_b200.Context(0) as ctx:
        got = jpeg.encode_batch(frames, o, ctx=ctx)
        assert ctx.host_fallbacks == 0
    for k in range(N):
        assert got[k] == po.jpeg_encode(frames[k], W, H, 2, Q, 1, ri or 0, opt), k


def test_host_fallback_over_three_groups(po, frames):
    """a scan buffer too small for every frame and no GPU retry: the host coder finishes each frame, from the
    records of its group's slot and, with optimised tables, from the frame's tables as the device built them"""
    for ri, opt in ((None, False), (4, True)):
        with pixo_b200.Context(0) as ctx:
            ctx.set_scan_capacity(4096, gpu_retry=False)
            got = jpeg.encode_batch(frames, JpegOptions(W, H, ColorType.Rgb, Q, Subsampling.S420, ri, opt), ctx=ctx)
            assert ctx.host_fallbacks == N, (ri, opt)
        for k in range(N):
            assert got[k] == po.jpeg_encode(frames[k], W, H, 2, Q, 1, ri or 0, opt), (ri, opt, k)


def test_progressive_batch_over_three_groups(frames):
    o = JpegOptions.max(W, H, 90)
    with pixo_b200.Context(0) as ctx:
        got = jpeg.encode_progressive_batch(frames, o, ctx=ctx)
        for k in range(N):
            assert got[k] == jpeg.encode_progressive(frames[k], o, ctx=ctx), k
        assert ctx.host_fallbacks == 0


def test_encode_dev_matches_encode_batch(frames):
    """pixo_b200_jpeg_encode_dev on the same frames: headers + scan + EOI are the encode_batch files"""
    import torch
    from pixo_b200 import _lib
    cap = 9 << 20
    with pixo_b200.Context(0) as ctx:
        files = jpeg.encode_batch(frames, JpegOptions(W, H, ColorType.Rgb, Q, Subsampling.S420), ctx=ctx)
        d_px = torch.from_numpy(frames).cuda()
        d_scan = torch.zeros((N, cap), dtype=torch.uint8, device="cuda")
        d_len = torch.zeros(N, dtype=torch.int64, device="cuda")
        d_ovf = torch.ones(N, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        _lib.check(ctx.handle, _lib.load().pixo_b200_jpeg_encode_dev(
            ctx.handle, d_px.data_ptr(), W * H * 3, N, W, H, 2, Q, 1, d_scan.data_ptr(), cap, d_len.data_ptr(),
            d_ovf.data_ptr()))
        ctx.sync()
        lens, ovf = d_len.cpu().numpy(), d_ovf.cpu().numpy()
        for k in range(N):
            assert ovf[k] == 0, k
            scan = d_scan[k, :int(lens[k])].cpu().numpy().tobytes()
            assert files[k][:_header_len(files[k])] + scan + b"\xff\xd9" == files[k], k
