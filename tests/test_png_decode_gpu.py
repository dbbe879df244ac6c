"""The GPU PNG decoder (pixo_b200.decode, png_decode.cu) against the C oracle (oracle/png_decode.c): pixels, geometry,
colour type, status code and the single-file message on the real-pixo goldens and the constructed corpus; mixed
batches with guard bytes; full-size frames against their source bytes; a batch over several passes; launches per
pass; and a PNG -> resize -> JPEG transcode that stays on the device."""
import glob
import hashlib
import os
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import pixo_b200
from pixo_b200 import ColorType, _lib, decode, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from oracle import png_decode as pd
from oracle import pyoracle as po
from png_decode_corpus import bit_flips, corpus, png, truncations
from test_png_decode import sparse_files

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STATUS = {pd.INVALID: _lib.ERR_INVALID_DECODE, pd.UNSUPPORTED: _lib.ERR_UNSUPPORTED_DECODE,
          pd.DIMENSIONS: _lib.ERR_INVALID_DIMENSIONS, pd.TOO_LARGE: _lib.ERR_IMAGE_TOO_LARGE}


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = pixo_b200.Context(0)
    yield c
    assert c.host_fallbacks == 0
    c.close()


def goldens():
    files = sorted(glob.glob(os.path.join(GOLD, "p*.png")) + glob.glob(os.path.join(GOLD, "reduce", "*.png")) +
                   glob.glob(os.path.join(GOLD, "quantize", "*.png")))
    assert len(files) == 225
    return [open(p, "rb").read() for p in files]


def check_single(data, ctx):
    want = pd.decode(data)
    if want.kind != pd.OK:
        with pytest.raises(pixo_b200.PixoError) as e:
            decode.decode_png(data, ctx=ctx)
        assert e.value.code == STATUS[want.kind] and want.message in str(e.value), (want.message, str(e.value))
        return
    img = decode.decode_png(data, ctx=ctx)
    assert (img.width, img.height, int(img.color_type)) == (want.width, want.height, want.color_type)
    assert np.array_equal(img.pixels, want.pixels)


def check_batch(files, ctx):
    """decode_png_batch_dev on `files` equals the oracle on every file: the pixels, or pixo's error code."""
    got = decode.decode_png_batch_dev(files, ctx=ctx)
    ctx.sync()
    host = got.frames.cpu().numpy()
    for i, f in enumerate(files):
        want = pd.decode(f)
        if want.kind != pd.OK:
            assert got.geometries[i] is None and got.errors[i] is not None, i
            assert got.errors[i].code == STATUS[want.kind], (i, want.message, got.errors[i])
            continue
        w, h, ct = got.geometries[i]
        assert (w, h, int(ct)) == (want.width, want.height, want.color_type), i
        n = want.pixels.size
        assert np.array_equal(host[got.offsets[i]:got.offsets[i] + n], want.pixels), i
    return got


def test_goldens(ctx):
    files = goldens()
    for f in files:
        check_single(f, ctx)
    check_batch(files, ctx)


def test_corpus_single_and_batch(ctx):
    files = [f for _, f in corpus()]
    for f in files:
        check_single(f, ctx)
    check_batch(files, ctx)


def test_truncations_and_bit_flips(ctx):
    g = goldens()
    files = []
    for k in (0, 5, 70, 120, 200):
        files += truncations(g[k]) + bit_flips(g[k], 40, k)
    for f in files[::7]:
        check_single(f, ctx)
    check_batch(files, ctx)


def test_mixed_batch_guards_and_launches(ctx):
    """Failing files interleaved with good ones: nothing is written for them, and the guard bytes around every frame
    stay intact.  One pass makes 4 launches when it holds files that need expanding, 3 when it does not."""
    g = goldens()
    bad = [f for n, f in corpus() if pd.decode(f, pixels=False).kind != pd.OK]
    files = [g[i % len(g)] if i % 3 else bad[i % len(bad)] for i in range(120)]
    want = [pd.decode(f) for f in files]
    sizes = [w.pixels.size if w.kind == pd.OK else 64 for w in want]
    offs, o = [], 64
    for s in sizes:
        offs.append(o)
        o += s + 64
    buf = torch.full((o,), 0xA5, dtype=torch.uint8, device="cuda")
    import ctypes as C
    n = len(files)
    ptrs = (C.c_char_p * n)(*files)
    lens = (C.c_size_t * n)(*[len(f) for f in files])
    co = (C.c_size_t * n)(*offs)
    status = (C.c_int32 * n)()
    before = ctx.launch_count
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_decode_to_device(ctx.handle, C.cast(ptrs, C.c_void_p), lens, n,
                                                                      buf.data_ptr(), co, status))
    assert ctx.launch_count - before == 4   # k_png_crc, k_png_inflate, k_png_unfilter, k_png_expand
    ctx.sync()
    host = buf.cpu().numpy()
    mask = np.ones(o, bool)
    for i, w in enumerate(want):
        if w.kind == pd.OK:
            assert status[i] == 0 and np.array_equal(host[offs[i]:offs[i] + sizes[i]], w.pixels), i
            mask[offs[i]:offs[i] + sizes[i]] = False
        else:
            assert status[i] == STATUS[w.kind], (i, w.message, status[i])
    assert (host[mask] == 0xA5).all()
    rgb8 = [f for f in g if f[24] == 8 and f[25] in (0, 2, 4, 6)][:3]   # IHDR: 8-bit, not indexed
    direct = [png(5, 4, 8, 2, zlib.compress(bytes([0] + list(range(15))) * 4))] + rgb8
    before = ctx.launch_count
    check_batch(direct, ctx)
    assert ctx.launch_count - before == 3


def _png_of(img: np.ndarray, w: int, h: int, ch: int, level: int = 1) -> bytes:
    ct = {1: 0, 2: 4, 3: 2, 4: 6}[ch]
    rows = np.concatenate([np.zeros((h, 1), np.uint8), img.reshape(h, w * ch)], axis=1)
    return png(w, h, 8, ct, zlib.compress(rows.tobytes(), level))


def test_full_size_batches(ctx):
    for (w, h, ch, n) in ((3840, 2160, 4, 32), (1920, 1080, 3, 256)):
        src = [po.gen_noise(w, h, ch, s) for s in range(4)]
        enc = [_png_of(s, w, h, ch) for s in src]
        files = [enc[i % 4] for i in range(n)]
        got = decode.decode_png_batch_dev(files, ctx=ctx)
        ctx.sync()
        for i in range(n):
            assert got.errors[i] is None, (i, got.errors[i])
            frame = got.frames[got.offsets[i]:got.offsets[i] + w * h * ch].cpu().numpy()
            assert np.array_equal(frame, src[i % 4]), i


def periodic_16k():
    """A 16 384^2 RGB frame whose rows repeat with a period of 999 bytes, each row shifted from the one above, with
    filters Up and None: the stream is mostly long matches, so inflating its 805 MB stays quick."""
    w = h = 16384
    base = np.tile(np.random.default_rng(3).integers(0, 256, 999, dtype=np.uint8), w * 3 // 999 + 2)
    img = np.lib.stride_tricks.sliding_window_view(base, w * 3)[(np.arange(h) * 7) % 999]
    rows = np.empty((h, w * 3 + 1), np.uint8)
    rows[:, 0] = 2   # Up
    rows[0, 1:] = img[0]
    rows[1:, 1:] = img[1:] - img[:-1]
    rows[::3, 0] = 0
    rows[::3, 1:] = img[::3]
    return png(w, h, 8, 2, zlib.compress(rows.tobytes(), 1)), img


def test_16k_frame(ctx):
    """One 16 384^2 RGB file goes alone; the unfilter wavefront runs over 512 row groups."""
    f, img = periodic_16k()
    out = decode.decode_png(f, ctx=ctx)
    assert hashlib.sha256(out.pixels.tobytes()).hexdigest() == hashlib.sha256(img.tobytes()).hexdigest()


def test_batch_over_several_passes(ctx):
    """More files than one pass holds (65 536): the second pass decodes the rest."""
    small = [png(2, 1, 8, 0, zlib.compress(bytes([0, k & 255, 3]))) for k in range(300)]
    files = [small[i % 300] for i in range(65536 + 37)]
    before = ctx.launch_count
    got = decode.decode_png_batch_dev(files, ctx=ctx)
    assert ctx.launch_count - before == 6   # two passes of k_png_crc, k_png_inflate, k_png_unfilter
    host = got.frames.cpu().numpy()
    for i in list(range(0, len(files), 997)) + [len(files) - 1]:
        assert got.errors[i] is None and host[got.offsets[i]:got.offsets[i] + 2].tolist() == [(i % 300) & 255, 3], i


def test_transcode_on_device(ctx):
    """decode_png_batch_dev -> resize_dev -> encode_dev with no host copy of pixels, against the oracle chain."""
    from oracle import resize as rz
    from pixo_b200.resize import ResizeAlgorithm, ResizeOptions
    w, h, dw, dh, n = 64, 48, 40, 30, 4
    src = [po.gen_noise(w, h, 3, s) for s in range(n)]
    files = [_png_of(s, w, h, 3, 6) for s in src]
    got = decode.decode_png_batch_dev(files, ctx=ctx)
    assert got.offsets == [i * w * h * 3 for i in range(n)]
    ro = ResizeOptions.builder(w, h).dst(dw, dh).color_type(ColorType.Rgb).algorithm(ResizeAlgorithm.Lanczos3).build()
    small = torch.empty(n * dw * dh * 3, dtype=torch.uint8, device="cuda")
    pixo_b200.resize.resize_dev(got.frames, w * h * 3, n, ro, small, dw * dh * 3, ctx=ctx)
    cap = 1 << 16
    scan = torch.empty(n * cap, dtype=torch.uint8, device="cuda")
    lens = torch.empty(n, dtype=torch.int64, device="cuda")
    ovf = torch.empty(n, dtype=torch.int32, device="cuda")
    jpeg.encode_dev(small, dw * dh * 3, n, JpegOptions(dw, dh, ColorType.Rgb, 80, Subsampling.S420), scan, cap, lens,
                    ovf, ctx=ctx)
    ctx.sync()
    for i, f in enumerate(files):
        px = pd.decode(f).pixels
        want = po.jpeg_encode(rz.resize(px, w, h, dw, dh, 2, 2), dw, dh, po.RGB, 80, po.S420)
        assert int(ovf[i]) == 0
        body = scan[i * cap:i * cap + int(lens[i])].cpu().numpy().tobytes()
        assert want.endswith(body + b"\xff\xd9") and len(body) > 0, i


def test_sparse_files_get_their_own_slots(ctx):
    """Bilevel and palette files whose frames are far larger than their streams decode into slots of their own, the
    last one too: the frames tensor holds every frame, and a guarded call writes nothing past any frame."""
    g = goldens()
    files = [g[0]] + sparse_files() + [dict(corpus())["huge_claim_small_idat"]] + sparse_files()[:1]
    got = check_batch(files, ctx)
    for i, f in enumerate(files):
        if got.geometries[i]:
            w, h, ct = got.geometries[i]
            assert got.offsets[i] + w * h * ct.bytes_per_pixel() <= got.frames.numel(), i
    want = [pd.decode(f) for f in files]
    sizes = [w.pixels.size if w.kind == pd.OK else 0 for w in want]
    offs = list(np.cumsum([64] + [s + 64 for s in sizes[:-1]]))
    total = offs[-1] + sizes[-1] + 64
    buf = torch.full((total,), 0xA5, dtype=torch.uint8, device="cuda")
    import ctypes as C
    n = len(files)
    status = (C.c_int32 * n)()
    _lib.check(ctx.handle, _lib.load().pixo_b200_png_decode_to_device(
        ctx.handle, C.cast((C.c_char_p * n)(*files), C.c_void_p), (C.c_size_t * n)(*map(len, files)), n,
        buf.data_ptr(), (C.c_size_t * n)(*map(int, offs)), status))
    host = buf.cpu().numpy()
    mask = np.ones(total, bool)
    for i, w in enumerate(want):
        assert (status[i] == 0) == (w.kind == pd.OK), i
        if w.kind == pd.OK:
            assert np.array_equal(host[offs[i]:offs[i] + sizes[i]], w.pixels), i
            mask[offs[i]:offs[i] + sizes[i]] = False
    assert (host[mask] == 0xA5).all()
    for f in sparse_files():
        check_single(f, ctx)
