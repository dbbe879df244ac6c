"""GPU parity: CUDA transform path (through the C ABI) vs the CPU oracle — bit-exact int16
coefficients and byte-identical JPEG streams."""
import hashlib

import numpy as np
import pytest

import pixo_b200
from pixo_b200 import ColorType, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from util import EDGE_CASE_DIMENSIONS, images

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    """Every test in this file must be served by the GPU entropy stage: the host coder may only
    run where a test forces it (and resets the expectation itself)."""
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was silently finished by the host entropy coder"


def _check_coeffs(po, ctx, img, w, h, ct, ss, q):
    y, cb, cr = jpeg.compute_all_coefficients(img, w, h, ColorType(ct), Subsampling(ss), q, ctx=ctx)
    ry, rcb, rcr = po.jpeg_coefficients(img, w, h, ct, ss, q)
    assert np.array_equal(y, ry), f"Y mismatch {w}x{h} ct={ct} ss={ss} q={q}: {(y != ry).sum()} coeffs"
    assert np.array_equal(cb, rcb), f"Cb mismatch {w}x{h} ss={ss} q={q}: {(cb != rcb).sum()}"
    assert np.array_equal(cr, rcr), f"Cr mismatch {w}x{h} ss={ss} q={q}: {(cr != rcr).sum()}"


@pytest.mark.parametrize("w,h", EDGE_CASE_DIMENSIONS)
def test_coefficients_edge_case_dimensions(po, gpu_ctx, w, h):
    for name, img in images(po, w, h, 3).items():
        for ss in (0, 1):
            _check_coeffs(po, gpu_ctx, img, w, h, 2, ss, 80)
    gray = po.gen_noise(w, h, 1, 11)
    _check_coeffs(po, gpu_ctx, gray, w, h, 0, 0, 80)


@pytest.mark.parametrize("q", [1, 10, 50, 75, 80, 95, 100])
def test_coefficients_all_qualities(po, gpu_ctx, q):
    w, h = 253, 131   # not MCU aligned, pitch not 16-byte aligned
    for img in images(po, w, h, 3).values():
        for ss in (0, 1):
            _check_coeffs(po, gpu_ctx, img, w, h, 2, ss, q)


@pytest.mark.parametrize("w,h", [(512, 16), (513, 16), (528, 33), (1040, 17), (31, 257), (3840, 32)])
def test_coefficients_tile_boundaries(po, gpu_ctx, w, h):
    # widths around the 32-MCU (512 px) tile and the 64-block tile of the 4:4:4 / gray kernels
    img = po.gen_noise(w, h, 3, 5)
    for ss in (0, 1):
        _check_coeffs(po, gpu_ctx, img, w, h, 2, ss, 90)
    _check_coeffs(po, gpu_ctx, po.gen_noise(w, h, 1, 6), w, h, 0, 0, 90)


def test_c1_256_full_bitstream(po, gpu_ctx):
    """BASELINE config C1: 256x256 RGB -> JPEG q=80, byte-identical files."""
    w = h = 256
    for img in images(po, w, h, 3).values():
        for ss in (Subsampling.S420, Subsampling.S444):
            for opt in (False, True):
                for ri in (None, 5):
                    o = JpegOptions(w, h, ColorType.Rgb, 80, ss, ri, opt)
                    got = jpeg.encode(img, o, ctx=gpu_ctx)
                    ref = po.jpeg_encode(img, w, h, 2, 80, int(ss), ri or 0, opt)
                    assert got == ref


def test_gray_full_bitstream(po, gpu_ctx):
    w, h = 100, 75
    img = po.gen_noise(w, h, 1, 2)
    for q in (50, 95):
        o = JpegOptions(w, h, ColorType.Gray, q, Subsampling.S444, None, True)
        assert jpeg.encode(img, o, ctx=gpu_ctx) == po.jpeg_encode(img, w, h, 0, q, 0, 0, True)


def test_c2_4k_coefficients_and_bitstream(po, gpu_ctx):
    """BASELINE config C2 at full size: 3840x2160 q=80 4:2:0."""
    w, h = 3840, 2160
    for img in (po.gen_gradient_rgb(w, h), po.gen_noise(w, h, 3, 42)):
        _check_coeffs(po, gpu_ctx, img, w, h, 2, 1, 80)
        o = JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420)
        got = jpeg.encode(img, o, ctx=gpu_ctx)
        ref = po.jpeg_encode(img, w, h, 2, 80, 1)
        assert hashlib.sha256(got).digest() == hashlib.sha256(ref).digest()


def test_c3_1080p_batch_qualities(po, gpu_ctx):
    """BASELINE config C3 (a slice of it): 1920x1080 frames, q in {50,80,95}; height 1080 is
    not a multiple of 16, so the last MCU row replicates."""
    w, h, n = 1920, 1080, 6
    frames = np.stack([po.gen_noise(w, h, 3, 42 + k) if k % 2 else np.roll(po.gen_gradient_rgb(w, h), k * w * 3)
                       for k in range(n)])
    for q in (50, 80, 95):
        o = JpegOptions(w, h, ColorType.Rgb, q, Subsampling.S420)
        got = jpeg.encode_batch(frames, o, ctx=gpu_ctx)
        for k in range(n):
            assert got[k] == po.jpeg_encode(frames[k], w, h, 2, q, 1), (q, k)
    o = JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420, None, True)
    got = jpeg.encode_batch(frames[:3], o, ctx=gpu_ctx)
    for k in range(3):
        assert got[k] == po.jpeg_encode(frames[k], w, h, 2, 80, 1, 0, True)


def test_zigzag_flag_and_histograms(po, gpu_ctx):
    w, h = 333, 222
    img = po.gen_noise(w, h, 3, 8)
    for ss in (0, 1):
        y, cb, cr, hist = jpeg.compute_all_coefficients(img, w, h, ColorType.Rgb, Subsampling(ss), 80,
                                                        zigzag=True, histograms=True, ctx=gpu_ctx)
        ry, rcb, rcr = po.jpeg_coefficients(img, w, h, 2, ss, 80)
        zz = np.array([int(v) for v in po.zigzag_reorder(np.arange(64, dtype=np.int16))])
        assert np.array_equal(y, ry[:, zz]) and np.array_equal(cb, rcb[:, zz]) and np.array_equal(cr, rcr[:, zz])
        assert np.array_equal(hist, po.jpeg_histograms(ry, rcb, rcr, w, h, 2, ss))
        _, _, _, hist2 = jpeg.compute_all_coefficients(img, w, h, ColorType.Rgb, Subsampling(ss), 80,
                                                       histograms=True, ctx=gpu_ctx)
        assert np.array_equal(hist2, hist)


def test_custom_quant_tables_and_rejection(po, gpu_ctx):
    w, h = 64, 64
    img = po.gen_noise(w, h, 3, 1)
    rng = np.random.default_rng(0)
    lq = rng.integers(1, 256, 64).astype(np.float32); cq = rng.integers(1, 256, 64).astype(np.float32)
    y, cb, cr = jpeg.compute_all_coefficients(img, w, h, lum_q=lq, chr_q=cq, ctx=gpu_ctx)
    ry, rcb, rcr = po.jpeg_coefficients(img, w, h, 2, 1, lum_q=lq, chr_q=cq)
    assert np.array_equal(y, ry) and np.array_equal(cb, rcb) and np.array_equal(cr, rcr)
    lq[3] = 0.5
    with pytest.raises(pixo_b200.PixoError):
        jpeg.compute_all_coefficients(img, w, h, lum_q=lq, chr_q=cq, ctx=gpu_ctx)


def test_error_behaviour_matches_reference(gpu_ctx):
    # tests/jpeg_conformance.rs:242-292
    E = pixo_b200._lib
    for q in (0, 101):
        with pytest.raises(pixo_b200.PixoError) as e:
            jpeg.encode(bytes(3), JpegOptions(1, 1, ColorType.Rgb, q), ctx=gpu_ctx)
        assert e.value.code == E.ERR_INVALID_QUALITY
    with pytest.raises(pixo_b200.PixoError) as e:
        jpeg.encode(bytes(3), JpegOptions(0, 1, ColorType.Rgb, 80), ctx=gpu_ctx)
    assert e.value.code == E.ERR_INVALID_DIMENSIONS
    with pytest.raises(pixo_b200.PixoError) as e:
        jpeg.encode(bytes(4), JpegOptions(1, 1, ColorType.Rgba, 80), ctx=gpu_ctx)
    assert e.value.code == E.ERR_UNSUPPORTED_COLOR
    with pytest.raises(pixo_b200.PixoError) as e:
        jpeg.encode(bytes(5), JpegOptions(1, 1, ColorType.Rgb, 80), ctx=gpu_ctx)
    assert e.value.code == E.ERR_INVALID_DATA_LENGTH
    with pytest.raises(pixo_b200.PixoError) as e:
        jpeg.encode(bytes(3), JpegOptions(1, 1, ColorType.Rgb, 80, restart_interval=0), ctx=gpu_ctx)
    assert e.value.code == E.ERR_INVALID_RESTART
    with pytest.raises(pixo_b200.PixoError) as e:
        jpeg.encode(bytes(3), JpegOptions(1, 1, ColorType.Rgb, 80, progressive=True), ctx=gpu_ctx)
    assert e.value.code == E.ERR_UNSUPPORTED


def test_determinism_and_decoder_acceptance(po, gpu_ctx):
    import io
    from PIL import Image
    w, h = 200, 120
    img = po.gen_gradient_rgb(w, h)
    o = JpegOptions(w, h, ColorType.Rgb, 85, Subsampling.S420)
    a = jpeg.encode(img, o, ctx=gpu_ctx)
    assert a == jpeg.encode(img, o, ctx=gpu_ctx)
    im = Image.open(io.BytesIO(a)); im.load()
    assert im.size == (w, h)
    sizes = [len(jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, q, Subsampling.S420), ctx=gpu_ctx))
             for q in (10, 50, 90)]
    assert sizes[0] < sizes[1] < sizes[2]   # tests/jpeg_conformance.rs:84


def _scan_bytes(jpg: bytes) -> bytes:
    """entropy-coded segment of a baseline file: after the SOS header, before EOI"""
    i = 2
    while True:
        assert jpg[i] == 0xFF
        ln = int.from_bytes(jpg[i + 2:i + 4], "big")
        if jpg[i + 1] == 0xDA:
            return jpg[i + 2 + ln:-2]
        i += 2 + ln


@pytest.mark.parametrize("w,h,ct,ss", [(640, 480, 2, 1), (333, 222, 2, 0), (257, 129, 0, 0)])
def test_entropy_stage_dense_blocks(po, gpu_ctx, w, h, ct, ss):
    """Noise at q 97-100: blocks longer than the 768-bit shared-memory slot (local-memory
    words), chunks that need several assembly windows, frequent 0xFF bytes; optimised tables."""
    img = po.gen_noise(w, h, 3 if ct == 2 else 1, 7)
    for q in (100, 97):
        for opt in (False, True):
            o = JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), None, opt)
            assert jpeg.encode(img, o, ctx=gpu_ctx) == po.jpeg_encode(img, w, h, ct, q, ss, 0, opt), (q, opt)


def test_dense_frames_are_recoded_on_the_gpu_not_the_host(po):
    """q=100 noise outgrows the heuristic device scan buffer (half the raw frame): the frame is
    coded a second time by k_huff with the exact size; the host coder stays idle.  With the retry
    switched off and a tiny buffer the host coder must take over - and be counted."""
    w, h = 640, 480
    img = po.gen_noise(w, h, 3, 7)
    ref = po.jpeg_encode(img, w, h, 2, 100, 1)
    assert len(ref) > (w * h * 3 // 2 + 65536) * 9 // 8   # really beyond the heuristic
    with pixo_b200.Context(0) as ctx:
        o = JpegOptions(w, h, ColorType.Rgb, 100, Subsampling.S420)
        l0 = ctx.launch_count
        assert jpeg.encode(img, o, ctx=ctx) == ref
        assert ctx.host_fallbacks == 0
        assert ctx.launch_count - l0 >= 3          # K1, entropy stage (overflow), entropy stage again with the exact size
        batch = np.stack([img, po.gen_gradient_rgb(w, h), img])
        got = jpeg.encode_batch(batch, o, ctx=ctx, capacity_each=jpeg.output_capacity(w, h))
        assert got[0] == ref and got[2] == ref and got[1] == po.jpeg_encode(batch[1], w, h, 2, 100, 1)
        assert ctx.host_fallbacks == 0
        ctx.set_scan_capacity(4096, gpu_retry=False)
        assert jpeg.encode(img, o, ctx=ctx) == ref
        assert ctx.host_fallbacks == 1
        ctx.set_scan_capacity(4096, gpu_retry=True)      # tiny first buffer, GPU retry on
        assert jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420), ctx=ctx) == \
            po.jpeg_encode(img, w, h, 2, 80, 1)
        assert ctx.host_fallbacks == 1
        ctx.set_scan_capacity(0)


def test_batch_optimize_many_small_frames_fresh_context(po):
    """ADVICE r1: per-image optimised tables run one k_huff pass per image, each with its own
    scratch region - 20 small frames on a context that has never grown its scratch."""
    w, h, n = 256, 256, 20
    frames = np.stack([po.gen_noise(w, h, 3, 100 + k) if k % 3 else po.gen_gradient_rgb(w, h) for k in range(n)])
    with pixo_b200.Context(0) as ctx:
        for ri in (None, 3):
            o = JpegOptions(w, h, ColorType.Rgb, 85, Subsampling.S420, ri, True)
            got = jpeg.encode_batch(frames, o, ctx=ctx)
            for k in range(n):
                assert got[k] == po.jpeg_encode(frames[k], w, h, 2, 85, 1, ri or 0, True), (ri, k)
        assert ctx.host_fallbacks == 0


def test_restart_streams_decode_like_the_plain_stream(po, gpu_ctx):
    """Independent pin for restart intervals (the reference's wasm API cannot produce them): a
    conforming decoder (libjpeg via PIL) must reconstruct exactly the same pixels from the
    restart and the non-restart encodes of the same frame, and see the DRI/RSTn structure."""
    import io
    from PIL import Image
    w, h = 333, 222
    for img in (po.gen_noise(w, h, 3, 9), po.gen_gradient_rgb(w, h)):
        for ss in (Subsampling.S420, Subsampling.S444):
            plain = jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, 85, ss), ctx=gpu_ctx)
            want = np.asarray(Image.open(io.BytesIO(plain)).convert("RGB"))
            for ri in (1, 4, 37):
                rst = jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, 85, ss, ri), ctx=gpu_ctx)
                assert b"\xff\xdd\x00\x04" + ri.to_bytes(2, "big") in rst[:700]     # DRI
                got = np.asarray(Image.open(io.BytesIO(rst)).convert("RGB"))
                assert np.array_equal(got, want), (ss, ri)


def test_encode_dev_device_resident(po, gpu_ctx):
    """pixo_b200_jpeg_encode_dev: device RGB in, device scan bytes + lengths out; a capacity that
    is too small is reported (needed size in the length) and nothing is written past it."""
    import torch
    from pixo_b200 import _lib
    lib = _lib.load()
    w, h, n = 1000, 600, 3
    frames = np.stack([po.gen_noise(w, h, 3, 5), po.gen_gradient_rgb(w, h), po.gen_noise(w, h, 3, 6)])
    stride = w * h * 3
    d_px = torch.from_numpy(frames.reshape(n, -1)).cuda()
    refs = [_scan_bytes(po.jpeg_encode(frames[k].reshape(-1), w, h, 2, 80, 1)) for k in range(n)]
    for cap in (1 << 20, 4096):
        d_scan = torch.full((n, cap + 256), 0xA5, dtype=torch.uint8, device="cuda")
        d_len = torch.zeros(n, dtype=torch.int64, device="cuda")
        d_ovf = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        rc = lib.pixo_b200_jpeg_encode_dev(gpu_ctx.handle, d_px.data_ptr(), stride, n, w, h, 2, 80, 1,
                                           d_scan.data_ptr(), cap + 256, d_len.data_ptr(), d_ovf.data_ptr())
        _lib.check(gpu_ctx.handle, rc)
        gpu_ctx.sync()
        lens, ovf, scan = d_len.cpu().numpy(), d_ovf.cpu().numpy(), d_scan.cpu().numpy()
        for k in range(n):
            assert lens[k] == len(refs[k]), k
            if len(refs[k]) <= cap + 256:
                assert ovf[k] == 0 and scan[k, :lens[k]].tobytes() == refs[k]
            else:
                assert ovf[k] != 0


def _upload_coefficients(po, img, w, h, ct, ss, q):
    """The oracle's coefficients, and the same arrays as int16 device tensors (None for absent chroma)."""
    import torch
    host = po.jpeg_coefficients(img, w, h, ct, ss, q)
    dev = [torch.from_numpy(a).cuda() if len(a) else None for a in host]
    torch.cuda.synchronize()
    return host, dev


@pytest.mark.parametrize("w,h,ct,ss", [(333, 222, 2, 1), (333, 222, 2, 0), (257, 129, 0, 0)])
def test_entropy_encode_dev_matches_oracle(po, gpu_ctx, w, h, ct, ss):
    """pixo_b200_jpeg_entropy_encode_dev on device coefficients: standard and optimised tables,
    with and without a restart interval, 4:2:0 / 4:4:4 / gray."""
    grad = po.gen_gradient_rgb(w, h)
    for img in (po.gen_noise(w, h, 3 if ct == 2 else 1, 4), grad if ct == 2 else grad[::3].copy()):
        (y, cb, cr), d = _upload_coefficients(po, img, w, h, ct, ss, 80)
        for ri in (0, 7):
            for opt in (False, True):
                o = JpegOptions(w, h, ColorType(ct), 80, Subsampling(ss), ri or None, opt)
                ref = po.jpeg_encode_from_coefficients(y, cb, cr, w, h, ct, 80, ss, ri, opt)
                assert jpeg.entropy_encode_dev(*d, o, ctx=gpu_ctx) == ref, (ri, opt)


def test_entropy_encode_dev_recodes_on_the_gpu(po, monkeypatch):
    """A scan that outgrows the first pass's device buffer is coded again with the size the kernel
    reported: unsegmented (q=100 noise beyond the heuristic), after a segmented first pass, and after
    a segmented first pass into a tiny buffer.  An output that holds the headers but not the scan is
    reported as too small, and nothing is written past it."""
    import ctypes as C
    from pixo_b200 import _lib
    w, h = 640, 480
    img = po.gen_noise(w, h, 3, 7)
    with pixo_b200.Context(0) as ctx:
        for q, segments, cap in ((100, None, 0), (80, "5", 0), (80, "5", 4096)):
            if segments:
                monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
            ctx.set_scan_capacity(cap)
            (y, cb, cr), d = _upload_coefficients(po, img, w, h, 2, 1, q)
            ref = po.jpeg_encode_from_coefficients(y, cb, cr, w, h, 2, q, 1)
            if q == 100:
                assert len(ref) > (w * h * 3 // 2 + 65536) * 9 // 8   # really beyond the heuristic
            l0 = ctx.launch_count
            assert jpeg.entropy_encode_dev(*d, JpegOptions(w, h, ColorType.Rgb, q, Subsampling.S420), ctx=ctx) == ref
            # two k_huff passes unsegmented; one k_huff<RAW> + four splice kernels per segmented pass
            assert ctx.launch_count - l0 >= (2 if not segments else 5 if not cap else 10), (q, segments, cap)
        ctx.set_scan_capacity(0)
        monkeypatch.delenv("PIXO_B200_SEGMENTS")
        out_cap = 4096
        buf = np.full(out_cap + 256, 0xA5, np.uint8)
        n = C.c_size_t(0)
        rc = _lib.load().pixo_b200_jpeg_entropy_encode_dev(
            ctx.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), w, h, 2, 80, 1, 0, 0,
            buf.ctypes.data, out_cap, C.byref(n))
        assert rc == _lib.ERR_OUTPUT_TOO_SMALL
        assert (buf[out_cap:] == 0xA5).all()


def test_large_pageable_input_takes_the_staged_copy(po, gpu_ctx):
    """Sources of 64 MB and more (ordinary, pageable memory) are pushed through the pinned slot
    ring by several host threads; the pieces must land exactly where a single copy would put them."""
    w, h = 6000, 4000     # 72 MB of RGB
    rng = np.random.default_rng(11)
    img = np.roll(po.gen_gradient_rgb(w, h).reshape(h, w * 3), 7, axis=0).reshape(-1).copy()
    img[rng.integers(0, img.size, 200000)] ^= 0x5A     # break the regularity at random places
    for ss in (Subsampling.S420, Subsampling.S444):
        o = JpegOptions(w, h, ColorType.Rgb, 80, ss)
        got = jpeg.encode(img, o, ctx=gpu_ctx)
        ref = po.jpeg_encode(img, w, h, 2, 80, int(ss))
        assert hashlib.sha256(got).digest() == hashlib.sha256(ref).digest()


@pytest.mark.parametrize("w,h,ss,ri", [(256, 256, 1, 1), (256, 256, 1, 5), (333, 222, 0, 7), (640, 480, 1, 40),
                                       (640, 480, 0, 33), (100, 75, 1, 65535), (1000, 600, 1, 63)])
def test_restart_intervals_on_the_gpu_coder(po, gpu_ctx, w, h, ss, ri):
    """handle_restart (src/jpeg/mod.rs:1423-1445): per-interval 1-padding, RSTn markers (not
    stuffed, none before EOI), DC predictors reset - intervals shorter, equal to and longer than a
    32-block chunk, not dividing the MCU count, and larger than the image."""
    for img in (po.gen_noise(w, h, 3, 3), po.gen_gradient_rgb(w, h)):
        for q, opt in ((80, False), (97, True)):
            o = JpegOptions(w, h, ColorType.Rgb, q, Subsampling(ss), ri, opt)
            assert jpeg.encode(img, o, ctx=gpu_ctx) == po.jpeg_encode(img, w, h, 2, q, ss, ri, opt), (q, opt)
    g = po.gen_noise(w, h, 1, 5)
    o = JpegOptions(w, h, ColorType.Gray, 85, Subsampling.S444, ri)
    assert jpeg.encode(g, o, ctx=gpu_ctx) == po.jpeg_encode(g, w, h, 0, 85, 0, ri, False)


@pytest.mark.parametrize("segments", [2, 5, 64])
def test_segmented_entropy_coding_forced(po, gpu_ctx, monkeypatch, segments):
    """Large single frames are cut into runs of MCUs that are Huffman-coded as independent bit
    strings and spliced on the device (k_huff<RAW> + k_seg_*).  The size threshold keeps small frames
    on the single-pass kernel, so force the segment count here: ragged last segments, segments
    shorter than a chunk, DC prediction across segment borders, optimised tables, dense q=100 noise
    (0xFF stuffing across the borders), gray / 4:4:4 / 4:2:0."""
    monkeypatch.setenv("PIXO_B200_SEGMENTS", str(segments))
    for (w, h, ct, ss) in ((640, 480, 2, 1), (333, 222, 2, 0), (257, 129, 0, 0), (48, 32, 2, 1)):
        img = po.gen_noise(w, h, 3 if ct == 2 else 1, 7)
        for q, opt in ((80, False), (100, False), (55, True)):
            o = JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), None, opt)
            assert jpeg.encode(img, o, ctx=gpu_ctx) == po.jpeg_encode(img, w, h, ct, q, ss, 0, opt), (w, h, q, opt)
    frames = np.stack([po.gen_noise(512, 256, 3, s) for s in (1, 2, 3)])
    got = jpeg.encode_batch(frames, JpegOptions(512, 256, ColorType.Rgb, 90, Subsampling.S420), ctx=gpu_ctx)
    for k in range(3):
        assert got[k] == po.jpeg_encode(frames[k], 512, 256, 2, 90, 1), k
