"""The GPU baseline JPEG decoder (pixo_b200.decode, jpeg_decode.cu) against the C oracle (oracle/jpeg_decode.c), byte
for byte: real pixo files, files from the GPU encoder over its options, constructed corrupt and hostile files, mixed
batches, full-size frames, a device transcode, and the batch call's ordering on a caller's stream."""
import glob
import hashlib
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import pixo_b200
from pixo_b200 import ColorType, decode, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from oracle import jpeg_decode as jd
from oracle import pyoracle as po
from jpeg_decode_corpus import constructed, corrupted, truncations

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = pixo_b200.Context(0)
    yield c
    c.close()


def check_batch(files, ctx):
    """decode_jpeg_batch_dev on `files` equals the oracle on every file: the pixels, or pixo's error."""
    got = decode.decode_jpeg_batch_dev(files, ctx=ctx)
    ctx.sync()
    host = got.frames.cpu().numpy()
    for i, f in enumerate(files):
        want = jd.decode(f, coefs=False)
        if want.status != jd.OK:
            assert got.geometries[i] is None and got.errors[i] is not None, i
            assert want.message in str(got.errors[i]), (i, want.message, str(got.errors[i]))
            continue
        w, h, ct = got.geometries[i]
        assert (w, h, int(ct)) == (want.width, want.height, want.color_type), i
        n = want.pixels.size
        assert np.array_equal(host[got.offsets[i]:got.offsets[i] + n], want.pixels), i
    return got


def test_goldens_direct(ctx):
    files = sorted(glob.glob(os.path.join(GOLD, "j*.jpg")))
    assert len(files) == 71
    for p in files:
        data = open(p, "rb").read()
        img = decode.decode_jpeg(data, ctx=ctx)
        want = jd.decode(data, coefs=False)
        assert (img.width, img.height, int(img.color_type)) == (want.width, want.height, want.color_type), p
        assert np.array_equal(img.pixels, want.pixels), p
    check_batch([open(p, "rb").read() for p in files], ctx)


def test_progressive_files_are_refused(ctx):
    for p in sorted(glob.glob(os.path.join(GOLD, "trellis", "*.jpg")))[:8]:
        with pytest.raises(pixo_b200.PixoError) as e:
            decode.decode_jpeg(open(p, "rb").read(), ctx=ctx)
        assert e.value.code == pixo_b200._lib.ERR_UNSUPPORTED_DECODE
        assert str(e.value) == "Unsupported: progressive JPEG not supported"


def _encoded_matrix(ctx):
    files = []
    for (w, h) in ((1, 1), (7, 9), (64, 48), (1297, 35)):
        for ct, ss in ((ColorType.Gray, Subsampling.S444), (ColorType.Rgb, Subsampling.S444),
                       (ColorType.Rgb, Subsampling.S420)):
            img = po.gen_noise(w, h, 1 if ct == ColorType.Gray else 3, w * 7 + h)
            for q in (1, 50, 80, 95, 100):
                for opt in (False, True):
                    for ri in (None, 1, 5):
                        files.append(jpeg.encode(img, JpegOptions(w, h, ct, q, ss, ri, opt), ctx=ctx))
    return files


def test_gpu_encoded_matrix(ctx):
    files = _encoded_matrix(ctx)
    assert len(files) == 360
    got = check_batch(files, ctx)
    assert all(e is None for e in got.errors)


def test_constructed_corpus(ctx):
    files = [constructed(s) for s in range(400)]
    small = jpeg.encode(po.gen_noise(19, 11, 3, 5), JpegOptions(19, 11, ColorType.Rgb, 90, Subsampling.S420, 1),
                        ctx=ctx)
    files += truncations(small) + corrupted(small, 1, 100)
    files += [b"", b"\xff\xd8", b"not a jpeg", open(os.path.join(GOLD, "trellis", "t000.jpg"), "rb").read()]
    check_batch(files, ctx)


def test_mixed_batch_and_launches(ctx):
    golds = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "j*.jpg")))]
    files = [golds[i % len(golds)] if i % 3 else constructed(1000 + i) for i in range(90)]
    before = ctx.launch_count
    check_batch(files, ctx)
    assert ctx.launch_count - before == 3   # one pass: k_jdec_scan, k_jdec_idct, k_jdec_color


def _big(ctx, w, h, n, ss=Subsampling.S420, q=80):
    fr = np.stack([po.gen_noise(w, h, 3, s) if s % 2 else np.asarray(po.gen_gradient_rgb(w, h)).reshape(-1)
                   for s in range(min(n, 4))])
    files = jpeg.encode_batch(fr, JpegOptions(w, h, ColorType.Rgb, q, ss), ctx=ctx)
    return [files[i % len(files)] for i in range(n)]


def test_full_size_batches(ctx):
    check_batch(_big(ctx, 1920, 1080, 256), ctx)
    check_batch(_big(ctx, 3840, 2160, 32), ctx)


def test_16k_frame(ctx):
    f = _big(ctx, 16384, 16384, 1)[0]
    img = decode.decode_jpeg(f, ctx=ctx)
    want = jd.decode(f, coefs=False)
    assert hashlib.sha256(img.pixels.tobytes()).hexdigest() == hashlib.sha256(want.pixels.tobytes()).hexdigest()


def test_transcode_on_device(ctx):
    """decode_jpeg_batch_dev -> resize_dev -> encode_dev with no host copy of pixels, against the oracle
    composition."""
    from oracle import resize as rz
    from pixo_b200.resize import ResizeAlgorithm, ResizeOptions
    w, h, dw, dh, n = 64, 48, 40, 30, 4   # 64 * 48 * 3 is a multiple of 256: the frames are back to back
    files = [jpeg.encode(po.gen_noise(w, h, 3, s), JpegOptions(w, h, ColorType.Rgb, 85, Subsampling.S420), ctx=ctx)
             for s in range(n)]
    got = decode.decode_jpeg_batch_dev(files, ctx=ctx)
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
        px = jd.decode(f, coefs=False).pixels
        want = po.jpeg_encode(rz.resize(px, w, h, dw, dh, 2, 2), dw, dh, po.RGB, 80, po.S420)
        assert int(ovf[i]) == 0
        body = scan[i * cap:i * cap + int(lens[i])].cpu().numpy().tobytes()
        assert want.endswith(body + b"\xff\xd9") and len(body) > 0, i


def test_batch_is_ordered_on_the_callers_stream(ctx):
    """The batch call returns with its work queued on the context's stream: work queued before it on that stream
    runs first, and a read queued after it sees the frames, with no host synchronisation in between."""
    golds = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(GOLD, "j*.jpg")))][:20]
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            torch.cuda._sleep(50_000_000)   # holds the stream while the call queues its work
            got = decode.decode_jpeg_batch_dev(golds, ctx=ctx)
            copy = got.frames.clone()
        assert not s.query()   # the call did not wait for the stream
        s.synchronize()
        host = copy.cpu().numpy()
        for i, f in enumerate(golds):
            want = jd.decode(f, coefs=False).pixels
            assert np.array_equal(host[got.offsets[i]:got.offsets[i] + want.size], want), i
    finally:
        ctx.set_stream(None)
