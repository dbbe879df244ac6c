"""k_trellis on the GPU: PIXO_B200_COEF_TRELLIS (pixo's compute_all_coefficients with use_trellis = true,
host and device entry points) and pixo_b200_jpeg_trellis_quantize_dev against the C oracle
(oracle/jpeg_trellis.c), on images and on constructed blocks, plus the error paths."""
import ctypes as C

import numpy as np
import pytest

from golden_inputs import make_input
from oracle import jpeg_trellis as jt
import trellis_ref as tr

pytestmark = pytest.mark.gpu

COEF_ZIGZAG, COEF_TRELLIS = 1, 2
ZZ = np.array(tr.ZIGZAG)


@pytest.fixture(scope="module", autouse=True)
def oracle_built():
    jt.build()


@pytest.fixture(autouse=True)
def no_host_fallback(gpu_ctx):
    """No frame of this file is finished by host code."""
    from pixo_b200 import _lib
    yield
    assert _lib.load().pixo_b200_ctx_host_fallbacks(gpu_ctx.handle) == 0


def _img(kind, w, h, ct, seed):
    if ct == 0 and kind == "gradient":   # the RGB gradient has no gray form
        kind = "vgrad"
    return make_input(kind, w, h, 1 if ct == 0 else 3, seed)


def _host(ctx, img, w, h, ct, ss, q, zigzag=False):
    from pixo_b200 import ColorType, jpeg
    return jpeg.compute_all_coefficients(img, w, h, ColorType(ct), jpeg.Subsampling(ss), q, zigzag=zigzag,
                                         use_trellis=True, ctx=ctx)


def _want(img, w, h, ct, ss, q, zigzag=False):
    y, cb, cr = jt.jpeg_coefficients(img, w, h, ct, ss, q)
    if zigzag:
        y, cb, cr = y[:, ZZ], cb[:, ZZ], cr[:, ZZ]
    return y, cb, cr


def _same(got, want):
    for g, w_ in zip(got, want):
        assert g.shape == w_.shape
        bad = np.nonzero((g != w_).any(1))[0]
        assert bad.size == 0, f"{bad.size} blocks differ, first {bad[0]}: {g[bad[0]]} vs {w_[bad[0]]}"


CASES = [(w, h) for w, h in [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 15), (33, 17), (70, 45), (255, 257),
                             (256, 8), (257, 16)]]


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
@pytest.mark.parametrize("w,h", CASES)
def test_coef_trellis_host(gpu_ctx, ct, ss, w, h):
    for i, (kind, q) in enumerate([("noise", 80), ("smooth", 50), ("primaries", 95), ("gradient", 25)]):
        img = _img(kind, w, h, ct, 100 + i)
        _same(_host(gpu_ctx, img, w, h, ct, ss, q), _want(img, w, h, ct, ss, q))


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
@pytest.mark.parametrize("q", [1, 50, 75, 100])
def test_coef_trellis_host_zigzag_qualities(gpu_ctx, ct, ss, q):
    w, h = 123, 77
    img = _img("noise", w, h, ct, q)
    _same(_host(gpu_ctx, img, w, h, ct, ss, q, zigzag=True), _want(img, w, h, ct, ss, q, zigzag=True))


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
@pytest.mark.parametrize("zigzag", [False, True])
def test_coef_trellis_dev_batch(gpu_ctx, lib, ct, ss, zigzag):
    """A device batch of frames with their own strides; tile edges (4:2:0 units are 256 px wide, 4:4:4
    units 256 px, gray tiles 512 px) fall inside the frame."""
    import torch
    from pixo_b200 import jpeg
    w, h, n, qual = 530, 41, 3, 85
    bpp = 1 if ct == 0 else 3
    frames = np.stack([_img(["noise", "smooth", "primaries"][i], w, h, ct, 7 + i).reshape(-1) for i in range(n)])
    px = torch.from_numpy(frames).cuda()
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    ys, cs = ny * 64 + 64, max(nc, 1) * 64 + 128
    dy = torch.zeros(n * ys, dtype=torch.int16, device="cuda")
    dcb = torch.zeros(n * cs, dtype=torch.int16, device="cuda")
    dcr = torch.zeros(n * cs, dtype=torch.int16, device="cuda")
    _, _, lq, cq = jpeg.quant_tables(qual)
    rc = lib.pixo_b200_jpeg_coefficients_dev(
        gpu_ctx.handle, px.data_ptr(), w * h * bpp, n, w, h, ct, ss, lq.ctypes.data_as(C.POINTER(C.c_float)),
        cq.ctypes.data_as(C.POINTER(C.c_float)), dy.data_ptr(), ys, dcb.data_ptr(), dcr.data_ptr(), cs,
        COEF_TRELLIS | (COEF_ZIGZAG if zigzag else 0), None)
    assert rc == 0, lib.pixo_b200_last_error(gpu_ctx.handle)
    y, cb, cr = dy.cpu().numpy(), dcb.cpu().numpy(), dcr.cpu().numpy()
    for i in range(n):
        got = (y[i * ys:i * ys + ny * 64].reshape(ny, 64), cb[i * cs:i * cs + nc * 64].reshape(nc, 64),
               cr[i * cs:i * cs + nc * 64].reshape(nc, 64))
        _same(got, _want(frames[i], w, h, ct, ss, qual, zigzag))


def test_coef_trellis_1024(gpu_ctx):
    w = h = 1024
    img = _img("smooth", w, h, 2, 5)
    _same(_host(gpu_ctx, img, w, h, 2, 1, 80), _want(img, w, h, 2, 1, 80))


def test_batch_32x4k_sampled(gpu_ctx, lib):
    """32 4K frames in one call (several groups of f32 scratch); four frames checked against the oracle."""
    import torch
    from pixo_b200 import jpeg
    w, h, n, qual = 3840, 2160, 32, 80
    g = torch.Generator(device="cuda").manual_seed(3)
    base = torch.randint(0, 256, (n, h // 8, w // 8, 3), dtype=torch.uint8, device="cuda", generator=g)
    px = base.repeat_interleave(8, 1).repeat_interleave(8, 2).contiguous()   # blocky: a mix of flat and busy
    px[:, ::3] ^= torch.randint(0, 8, (n, (h + 2) // 3, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    torch.cuda.synchronize()   # the library works on its own stream
    ny, nc = jpeg.block_counts(w, h, 2, 1)
    dy = torch.empty(n * ny * 64, dtype=torch.int16, device="cuda")
    dcb = torch.empty(n * nc * 64, dtype=torch.int16, device="cuda")
    dcr = torch.empty(n * nc * 64, dtype=torch.int16, device="cuda")
    _, _, lq, cq = jpeg.quant_tables(qual)
    rc = lib.pixo_b200_jpeg_coefficients_dev(
        gpu_ctx.handle, px.data_ptr(), w * h * 3, n, w, h, 2, 1, lq.ctypes.data_as(C.POINTER(C.c_float)),
        cq.ctypes.data_as(C.POINTER(C.c_float)), dy.data_ptr(), ny * 64, dcb.data_ptr(), dcr.data_ptr(), nc * 64,
        COEF_TRELLIS, None)
    assert rc == 0, lib.pixo_b200_last_error(gpu_ctx.handle)
    for i in (0, 5, 17, 31):
        frame = px[i].cpu().numpy().reshape(-1)
        got = (dy[i * ny * 64:(i + 1) * ny * 64].cpu().numpy().reshape(ny, 64),
               dcb[i * nc * 64:(i + 1) * nc * 64].cpu().numpy().reshape(nc, 64),
               dcr[i * nc * 64:(i + 1) * nc * 64].cpu().numpy().reshape(nc, 64))
        _same(got, _want(frame, w, h, 2, 1, qual))


def _dev_quant(ctx, d, q, lam, zigzag=False):
    import torch
    from pixo_b200 import jpeg
    out = jpeg.trellis_quantize_dev(torch.from_numpy(np.ascontiguousarray(d)).cuda(), q, lam, zigzag=zigzag, ctx=ctx)
    return out.cpu().numpy()


@pytest.mark.parametrize("lam", [None, 0.1, 0.5, 2.0, 10.0] + [tr.adaptive_lambda(q) for q in (1, 30, 50, 79, 80, 95, 100)])
def test_trellis_quantize_dev_constructed(gpu_ctx, lam):
    d, qs = tr.constructed_blocks(11, 300)
    for q in np.unique(qs, axis=0):   # one call per table, many blocks each
        sel = (qs == q).all(1)
        got = _dev_quant(gpu_ctx, d[sel], q, lam)
        want = jt.trellis_quantize_blocks(d[sel], q, lam)
        assert np.array_equal(got, want)


def test_trellis_quantize_dev_zigzag_and_many(gpu_ctx):
    rng = np.random.default_rng(4)
    d = (rng.laplace(0, 30, (20000, 64)) * (rng.random((20000, 64)) < 0.5)).astype(np.float32)
    q = rng.integers(1, 120, 64).astype(np.float32)
    want = jt.trellis_quantize_blocks(d, q, 1.0)
    assert np.array_equal(_dev_quant(gpu_ctx, d, q, None), want)
    assert np.array_equal(_dev_quant(gpu_ctx, d, q, None, zigzag=True), want[:, ZZ])


def test_trellis_quantize_host_and_adaptive(gpu_ctx):
    from pixo_b200 import jpeg
    d, qs = tr.constructed_blocks(5, 20)
    q = qs[-1]
    assert np.array_equal(jpeg.trellis_quantize(d, q, ctx=gpu_ctx), jt.trellis_quantize_blocks(d, q))
    for qual in (10, 60, 90):
        assert np.array_equal(jpeg.trellis_quantize_adaptive(d[3], q, qual, ctx=gpu_ctx),
                              jt.trellis_quantize(d[3], q, jt.trellis_lambda(qual)))


@pytest.mark.parametrize("bad", ["nan", "inf", "fq_high", "fq_low", "dc_high", "tiny"])
def test_trellis_rejects_input(gpu_ctx, bad):
    from pixo_b200 import _lib
    d = np.zeros((130, 64), np.float32)
    q = np.full(64, 2.0, np.float32)
    v = {"nan": np.nan, "inf": np.inf, "fq_high": 65533.0, "fq_low": -65534.0, "dc_high": 70000.0, "tiny": 1e-38}[bad]
    d[77, 0 if bad == "dc_high" else 9] = v
    with pytest.raises(_lib.PixoError) as e:
        _dev_quant(gpu_ctx, d, q, None)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    d[77] = 0.0
    d[5, 9] = 65532.0   # |fq| = 32766: the largest accepted
    assert np.array_equal(_dev_quant(gpu_ctx, d, q, None), jt.trellis_quantize_blocks(d, q))


def test_trellis_rejects_arguments(gpu_ctx):
    from pixo_b200 import _lib
    d = np.zeros((4, 64), np.float32)
    for q, lam in [(np.full(64, 0.5), None), (np.full(64, 256.0), None), (np.full(64, 2.0), float("nan"))]:
        with pytest.raises(_lib.PixoError) as e:
            _dev_quant(gpu_ctx, d, q, lam)
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT


def test_coef_trellis_rejects_histogram(gpu_ctx, lib):
    from pixo_b200 import _lib, jpeg
    img = _img("noise", 16, 16, 2, 1)
    with pytest.raises(_lib.PixoError) as e:
        jpeg.compute_all_coefficients(img, 16, 16, quality=80, histograms=True, use_trellis=True, ctx=gpu_ctx)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    import torch
    px = torch.from_numpy(img).cuda()
    buf = torch.zeros(4096, dtype=torch.int16, device="cuda")
    hist = torch.zeros(536, dtype=torch.int64, device="cuda")
    _, _, lq, cq = jpeg.quant_tables(80)
    rc = lib.pixo_b200_jpeg_coefficients_dev(gpu_ctx.handle, px.data_ptr(), 768, 1, 16, 16, 2, 1,
                                             lq.ctypes.data_as(C.POINTER(C.c_float)),
                                             cq.ctypes.data_as(C.POINTER(C.c_float)), buf.data_ptr(), 1024,
                                             buf[2048:].data_ptr(), buf[3072:].data_ptr(), 512, COEF_TRELLIS,
                                             hist.data_ptr())
    assert rc == _lib.ERR_INVALID_ARGUMENT


def test_plain_coefficients_unchanged_beside_trellis(gpu_ctx, po):
    """A plain call after trellis calls on the same context still returns quantize_block's output."""
    from pixo_b200 import jpeg
    img = _img("noise", 70, 45, 2, 9)
    _host(gpu_ctx, img, 70, 45, 2, 1, 80)
    got = jpeg.compute_all_coefficients(img, 70, 45, quality=80, ctx=gpu_ctx)
    want = po.jpeg_coefficients(img, 70, 45, po.RGB, po.S420, 80)
    for g, w_ in zip(got, want):
        assert np.array_equal(g, w_)


@pytest.mark.parametrize("ss", [0, 1])
def test_encode_ignores_trellis_quant(gpu_ctx, po, ss):
    """Baseline encode_scan ignores use_trellis: trellis_quant = 1 gives the same bytes."""
    from pixo_b200 import ColorType, jpeg
    w, h = 100, 75
    img = _img("smooth", w, h, 2, 3)
    a = jpeg.encode(img, jpeg.JpegOptions(w, h, ColorType.Rgb, 80, jpeg.Subsampling(ss), None, True, False, True),
                    ctx=gpu_ctx)
    b = jpeg.encode(img, jpeg.JpegOptions(w, h, ColorType.Rgb, 80, jpeg.Subsampling(ss), None, True, False, False),
                    ctx=gpu_ctx)
    assert a == b == po.jpeg_encode(img, w, h, po.RGB, 80, po.S420 if ss else po.S444, 0, True)


@pytest.mark.parametrize("c", __import__("test_jpeg_trellis").FIXTURES, ids=__import__("test_jpeg_trellis").FIXTURE_IDS)
def test_fixture_reencoded_from_gpu(gpu_ctx, c):
    """The GPU's trellis coefficients, re-encoded by pixo's progressive scan writer, reproduce every scan
    of a real max-preset file byte for byte (no oracle in between)."""
    import jpeg_progressive_scans as ps
    from test_jpeg_trellis import fixture_case
    img, ss, want, tables = fixture_case(c)
    got = ps.encode_scans(*_host(gpu_ctx, img, c["w"], c["h"], c["ct"], ss, c["q"]), tables)
    assert [g == w_ for g, w_ in zip(got, want)] == [True] * 7


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
@pytest.mark.parametrize("w,h,q", [(1297, 35, 90), (2063, 19, 80), (1100, 48, 95)])
def test_coef_trellis_wide_ragged(gpu_ctx, ct, ss, w, h, q):
    """Frames several transform units wide (256 px; gray tiles 512 px) with a ragged last unit."""
    for kind in ("noise", "smooth", "primaries"):
        img = _img(kind, w, h, ct, w + q)
        _same(_host(gpu_ctx, img, w, h, ct, ss, q), _want(img, w, h, ct, ss, q))


@pytest.mark.parametrize("ct,ss,w,h", [(2, 1, 16384, 8200), (0, 0, 16000, 16384)], ids=["420", "gray"])
def test_coef_trellis_large_frame_in_bands(gpu_ctx, lib, ct, ss, w, h):
    """A frame whose f32 DCT exceeds the 256 MiB scratch bound is done in bands of MCU rows.  A block's
    coefficients depend only on its own pixels away from the bottom edge, so crops of whole MCU rows
    around the band borders (and the frame's last rows) are checked against the oracle on the crop."""
    import torch
    from pixo_b200 import jpeg
    bpp, mcu = (1, 8) if ct == 0 else (3, 16 if ss else 8)
    g = torch.Generator(device="cuda").manual_seed(9)
    base = torch.randint(0, 256, ((h + 7) // 8, (w + 7) // 8, bpp), dtype=torch.uint8, device="cuda", generator=g)
    px = base.repeat_interleave(8, 0).repeat_interleave(8, 1)[:h, :w].contiguous()
    px[::3] ^= torch.randint(0, 16, px[::3].shape, dtype=torch.uint8, device="cuda", generator=g)
    torch.cuda.synchronize()   # the library works on its own stream
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    dy = torch.empty(ny * 64, dtype=torch.int16, device="cuda")
    dcb = torch.empty(max(nc, 1) * 64, dtype=torch.int16, device="cuda")
    dcr = torch.empty(max(nc, 1) * 64, dtype=torch.int16, device="cuda")
    _, _, lq, cq = jpeg.quant_tables(80)
    fp = C.POINTER(C.c_float)
    rc = lib.pixo_b200_jpeg_coefficients_dev(gpu_ctx.handle, px.data_ptr(), px.numel(), 1, w, h, ct, ss,
                                             lq.ctypes.data_as(fp), cq.ctypes.data_as(fp), dy.data_ptr(), ny * 64,
                                             dcb.data_ptr(), dcr.data_ptr(), nc * 64, COEF_TRELLIS, None)
    assert rc == 0, lib.pixo_b200_last_error(gpu_ctx.handle)
    mx, my = (w + mcu - 1) // mcu, (h + mcu - 1) // mcu
    ypm = 4 if mcu == 16 else 1
    row_bytes = mx * (ypm + (2 if ct else 0)) * 256
    assert row_bytes * my > 256 << 20
    band = (256 << 20) // row_bytes
    img = px.cpu().numpy()
    for m0 in sorted({band - 1, 2 * band - 2, my - 2}):
        crop = np.ascontiguousarray(img[m0 * mcu:min(h, (m0 + 2) * mcu)])
        ch = crop.shape[0]
        want = jt.jpeg_coefficients(crop.reshape(-1), w, ch, ct, ss, 80)
        got = (dy[m0 * mx * ypm * 64:(m0 * mx * ypm + len(want[0])) * 64].cpu().numpy().reshape(-1, 64),
               dcb[m0 * mx * 64:(m0 * mx + len(want[1])) * 64].cpu().numpy().reshape(-1, 64),
               dcr[m0 * mx * 64:(m0 * mx + len(want[2])) * 64].cpu().numpy().reshape(-1, 64))
        _same(got[:3 if ct else 1], want[:3 if ct else 1])
