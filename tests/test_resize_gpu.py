"""The CUDA resizers (pixo_b200_resize / pixo_b200_resize_dev) against real pixo output (tests/golden/resize/)
and against oracle/resize.c: an option matrix, full-size batches, the largest frames and sides pixo takes,
the layouts device callers pass, and the device output fed straight into the JPEG and PNG device paths."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

from oracle import resize as rz
from pixo_b200 import ColorType, _lib
from pixo_b200 import resize as pr
from pixo_b200.resize import ResizeAlgorithm, ResizeOptions
from test_dev_layouts_gpu import GUARD8, assert_guard, guarded, noise_poison, placed, run, scan_bytes
from test_resize import CASES, ERRORS, case_input, fixture

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_host_fallback(gpu_ctx):
    yield
    assert gpu_ctx.host_fallbacks == 0


def opts(sw, sh, dw, dh, ct, alg):
    return ResizeOptions.builder(sw, sh).dst(dw, dh).color_type(ColorType(ct)).algorithm(ResizeAlgorithm(alg)).build()


def frame(sw, sh, ct, seed, kind="noise"):
    rng = np.random.default_rng(seed)
    bpp = ct + 1
    if kind == "noise":
        return rng.integers(0, 256, sw * sh * bpp, dtype=np.uint8)
    y, x = np.mgrid[0:sh, 0:sw]
    img = ((((x // 5) + (y // 3)) % 2) * 255).astype(np.uint8)
    img = np.repeat(img[:, :, None], bpp, axis=2)
    img[:, :, 0] ^= rng.integers(0, 2, (sh, sw), dtype=np.uint8) * 0x3C
    return img.reshape(-1)


def resize_dev(ctx, frames, sw, sh, dw, dh, ct, alg, off=0, pad=0, out_off=64, out_pad=0):
    """pixo_b200_resize_dev on `frames` at element offset `off` and stride flen + pad (random poison around),
    into slots at `out_off` with stride dlen + out_pad inside a guarded buffer; returns the frames' outputs."""
    n, flen, dlen = len(frames), frames[0].size, dw * dh * (ct + 1)
    src = placed(frames, off, flen + pad, noise_poison(n + off))
    dstride = dlen + out_pad
    out = guarded(n * dstride, np.uint8, GUARD8, base=out_off)
    run(ctx, _lib.load().pixo_b200_resize_dev, src.ptr(off), flen + pad, n, sw, sh, dw, dh, ct, alg,
        out.ptr(out_off), dstride)
    o = out.get()
    assert_guard(o, [(out_off + i * dstride, dlen) for i in range(n)], GUARD8, "resize output")
    return [o[out_off + i * dstride: out_off + i * dstride + dlen] for i in range(n)]


@pytest.mark.parametrize("k", range(len(CASES)))
def test_reproduces_pixo(gpu_ctx, k):
    c = CASES[k]
    got = pr.resize(case_input(c), opts(c["sw"], c["sh"], c["dw"], c["dh"], c["ct"], c["alg"]), ctx=gpu_ctx)
    assert np.array_equal(got, fixture(c))


GEOMS = [(1, 1, 1, 1), (1, 1, 5, 3), (5, 3, 1, 1), (1297, 35, 640, 71), (35, 1297, 97, 600), (200, 100, 333, 77),
         (64, 64, 31, 17), (97, 61, 257, 251), (13, 11, 1297, 35)]


@pytest.mark.parametrize("alg", range(3))
@pytest.mark.parametrize("ct", range(4))
def test_option_matrix_equals_oracle(gpu_ctx, ct, alg):
    """Three frames of each geometry in one device batch (odd offsets and strides, so the RGBA and
    GrayAlpha nearest copies take the byte path), and the first through the host entry point."""
    for gi, (sw, sh, dw, dh) in enumerate(GEOMS):
        frames = [frame(sw, sh, ct, 100 * gi + i, ("noise", "edges")[i % 2]) for i in range(3)]
        want = [rz.resize(f, sw, sh, dw, dh, ct, alg) for f in frames]
        for off, pad in ((0, 0), (1, 3)):
            got = resize_dev(gpu_ctx, frames, sw, sh, dw, dh, ct, alg, off, pad, out_off=64 + off, out_pad=pad)
            for i in range(3):
                assert np.array_equal(got[i], want[i]), (sw, sh, dw, dh, off, i)
        assert np.array_equal(pr.resize(frames[0], opts(sw, sh, dw, dh, ct, alg), ctx=gpu_ctx), want[0])


@pytest.mark.parametrize("alg", range(3))
def test_4k_batch_to_1080p(gpu_ctx, alg):
    n, sw, sh, dw, dh = 32, 3840, 2160, 1920, 1080
    rng = np.random.default_rng(alg)
    base = rng.integers(0, 256, (sh, sw, 4), dtype=np.uint8)
    frames = [np.roll(base, 7 * i, axis=1).reshape(-1) if i % 3 else frame(sw, sh, 3, i, "edges") for i in range(n)]
    src = torch.from_numpy(np.stack(frames)).cuda()
    dst = torch.empty((n, dw * dh * 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    pr.resize_dev(src, sw * sh * 4, n, opts(sw, sh, dw, dh, 3, alg), dst, dw * dh * 4, ctx=gpu_ctx)
    gpu_ctx.sync()
    got = dst.cpu().numpy()
    for i in (0, 1, 17, 31):
        assert np.array_equal(got[i], rz.resize(frames[i], sw, sh, dw, dh, 3, alg)), i


@pytest.mark.parametrize("alg", range(3))
def test_16k_frame_over_the_band_cap(gpu_ctx, alg):
    """16 384^2 RGBA -> 12 000 x 16 384: Lanczos3's intermediate (786 MB) is done in bands."""
    sw = sh = 16384
    dw, dh = 12000, 16384
    img = np.random.default_rng(5).integers(0, 256, sw * sh * 4, dtype=np.uint8)
    img[: sw * 4 * 64] = frame(sw, 64, 3, 9, "edges")
    src = torch.from_numpy(img).cuda()
    dst = torch.empty(dw * dh * 4, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    pr.resize_dev(src, 0, 1, opts(sw, sh, dw, dh, 3, alg), dst, 0, ctx=gpu_ctx)
    gpu_ctx.sync()
    got = hashlib.sha256(dst.cpu().numpy().tobytes()).hexdigest()
    del src, dst
    assert got == hashlib.sha256(rz.resize(img, sw, sh, dw, dh, 3, alg).tobytes()).hexdigest()


@pytest.mark.parametrize("alg", range(3))
@pytest.mark.parametrize("sw,sh,dw,dh", [(1 << 24, 1, 4099, 3), (1, 1 << 24, 3, 4099), (4099, 1, 1 << 24, 1),
                                         (1, 3, 2, 1 << 24)])
def test_longest_sides(gpu_ctx, sw, sh, dw, dh, alg):
    """Sides of 2^24, where f32 index arithmetic is at its edge."""
    img = frame(sw, sh, 0, sw + sh)
    got = pr.resize(img, opts(sw, sh, dw, dh, 0, alg), ctx=gpu_ctx)
    assert np.array_equal(got, rz.resize(img, sw, sh, dw, dh, 0, alg))


@pytest.mark.parametrize("alg", range(3))
def test_frames_beyond_4gib_and_the_65535_split(gpu_ctx, alg):
    """65 537 tiny frames in one call (grid.z passes), and a frame at a byte offset above 2^32."""
    n, sw, sh, dw, dh = 65537, 5, 3, 4, 7
    frames = np.random.default_rng(alg).integers(0, 256, (n, sw * sh * 2), dtype=np.uint8)
    got = resize_dev(gpu_ctx, list(frames), sw, sh, dw, dh, 1, alg, off=3, pad=1, out_off=5, out_pad=2)
    for i in (0, 1, 65534, 65535, 65536):
        assert np.array_equal(got[i], rz.resize(frames[i], sw, sh, dw, dh, 1, alg)), i
    big = torch.full(((1 << 32) + 32768,), 0x5A, dtype=torch.uint8, device="cuda")
    f = frame(97, 61, 3, 1, "edges")
    off = (1 << 32) + 1
    big[off:off + f.size] = torch.from_numpy(f).cuda()
    out = torch.full((64 + 40 * 30 * 4 + 64,), GUARD8, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _lib.check(gpu_ctx.handle, _lib.load().pixo_b200_resize_dev(gpu_ctx.handle, big.data_ptr() + off, 0, 1, 97, 61,
                                                                40, 30, 3, alg, out.data_ptr() + 63, 0))
    gpu_ctx.sync()
    o = out.cpu().numpy()
    assert np.array_equal(o[63:63 + 4800], rz.resize(f, 97, 61, 40, 30, 3, alg))
    assert (o[:63] == GUARD8).all() and (o[63 + 4800:] == GUARD8).all()


@pytest.mark.parametrize("args,status", ERRORS)
def test_errors_match_pixo_order(gpu_ctx, args, status):
    sw, sh, dw, dh, ct, alg = args
    n = sw * sh * (ct + 1) if status != 5 and ct <= 3 and sw <= 1 << 24 else 3
    data = np.zeros(max(n, 1), np.uint8)
    out = np.zeros(64, np.uint8)
    got = C.c_size_t(0)
    rc = _lib.load().pixo_b200_resize(gpu_ctx.handle, data.ctypes.data, n, sw, sh, dw, dh, ct, alg, out.ctypes.data,
                                      out.size, C.byref(got))
    assert rc == status


def test_output_too_small_and_refused_layouts(gpu_ctx):
    lib = _lib.load()
    img = frame(20, 10, 2, 1)
    out = np.zeros(599, np.uint8)
    got = C.c_size_t(0)
    assert lib.pixo_b200_resize(gpu_ctx.handle, img.ctypes.data, img.size, 20, 10, 10, 20, 2, 2, out.ctypes.data,
                                out.size, C.byref(got)) == _lib.ERR_OUTPUT_TOO_SMALL
    assert got.value == 600
    src = torch.zeros(2 * img.size, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(2 * 600, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launch_count
    assert lib.pixo_b200_resize_dev(gpu_ctx.handle, src.data_ptr(), img.size - 1, 2, 20, 10, 10, 20, 2, 2,
                                    dst.data_ptr(), 600) == _lib.ERR_INVALID_DATA_LENGTH
    assert lib.pixo_b200_resize_dev(gpu_ctx.handle, src.data_ptr(), img.size, 2, 20, 10, 10, 20, 2, 2,
                                    dst.data_ptr(), 599) == _lib.ERR_OUTPUT_TOO_SMALL
    assert lib.pixo_b200_resize_dev(gpu_ctx.handle, src.data_ptr(), img.size, 2, 20, 10, 10, 20, 2, 3,
                                    dst.data_ptr(), 600) == _lib.ERR_INVALID_ARGUMENT
    assert gpu_ctx.launch_count == before


def test_resize_dev_into_jpeg_encode_dev(po, gpu_ctx):
    """A resized batch straight into the device JPEG path equals the oracle's resize then encode."""
    n, sw, sh, dw, dh = 3, 640, 480, 333, 251
    frames = [frame(sw, sh, 2, i, ("noise", "edges")[i % 2]) for i in range(n)]
    src = torch.from_numpy(np.stack(frames)).cuda()
    dlen = dw * dh * 3
    mid = torch.empty(n * dlen, dtype=torch.uint8, device="cuda")
    cap = (dlen + 65536 + 15) // 16 * 16   # scan slots: 16-byte aligned
    scan = torch.empty(n * cap, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(n, dtype=torch.int64, device="cuda")
    ovf = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    lib = _lib.load()
    _lib.check(gpu_ctx.handle, lib.pixo_b200_resize_dev(gpu_ctx.handle, src.data_ptr(), sw * sh * 3, n, sw, sh, dw, dh,
                                                        2, 2, mid.data_ptr(), dlen))
    _lib.check(gpu_ctx.handle, lib.pixo_b200_jpeg_encode_dev(gpu_ctx.handle, mid.data_ptr(), dlen, n, dw, dh, 2, 80, 1,
                                                             scan.data_ptr(), cap, lens.data_ptr(), ovf.data_ptr()))
    gpu_ctx.sync()
    s, ln = scan.cpu().numpy(), lens.cpu().numpy()
    assert not ovf.cpu().numpy().any()
    for i in range(n):
        want = scan_bytes(po.jpeg_encode(rz.resize(frames[i], sw, sh, dw, dh, 2, 2), dw, dh, 2, 80, 1))
        assert s[i * cap:i * cap + ln[i]].tobytes() == want, i


@pytest.mark.parametrize("ct", range(4))
def test_resize_dev_into_png_filter_dev(po, gpu_ctx, ct):
    n, sw, sh, dw, dh, bpp = 2, 301, 199, 150, 97, ct + 1
    frames = [frame(sw, sh, ct, 50 + i) for i in range(n)]
    src = torch.from_numpy(np.stack(frames)).cuda()
    dlen, flen = dw * dh * bpp, dh * (dw * bpp + 1)
    mid = torch.empty(n * dlen, dtype=torch.uint8, device="cuda")
    out = torch.empty(n * flen, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    lib = _lib.load()
    _lib.check(gpu_ctx.handle, lib.pixo_b200_resize_dev(gpu_ctx.handle, src.data_ptr(), sw * sh * bpp, n, sw, sh, dw,
                                                        dh, ct, 1, mid.data_ptr(), dlen))
    _lib.check(gpu_ctx.handle, lib.pixo_b200_png_filter_dev(gpu_ctx.handle, mid.data_ptr(), dlen, n, dw, dh, dw * bpp,
                                                            bpp, 6, out.data_ptr(), flen, None))
    gpu_ctx.sync()
    o = out.cpu().numpy()
    for i in range(n):
        want = po.apply_filters(rz.resize(frames[i], sw, sh, dw, dh, ct, 1), dw, dh, bpp, 6)
        assert np.array_equal(o[i * flen:(i + 1) * flen], want), i
