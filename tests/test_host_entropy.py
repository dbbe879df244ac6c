"""Host half of the product (headers, Huffman tables, multi-threaded entropy coder, argument
validation) against the oracle.  CPU only."""
import numpy as np
import pytest

import pixo_b200
from pixo_b200 import ColorType
from pixo_b200.jpeg import JpegOptions, Subsampling, entropy_encode


@pytest.mark.parametrize("w,h", [(1, 1), (17, 15), (70, 45), (256, 256), (640, 483)])
@pytest.mark.parametrize("ct", [0, 2])
def test_entropy_stage_is_byte_identical(po, w, h, ct):
    ch = 3 if ct == 2 else 1
    img = po.gen_noise(w, h, ch, 7) if (w + h) % 2 else po.gen_noise(w, h, ch, 1) // 3
    for ss in (0, 1):
        for q in (1, 50, 80, 95, 100):
            y, cb, cr = po.jpeg_coefficients(img, w, h, ct, ss, q)
            for ri in (0, 1, 7, 100):
                for opt in (False, True):
                    ref = po.jpeg_encode(img, w, h, ct, q, ss, ri, opt)
                    o = JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), ri or None, opt)
                    assert entropy_encode(y, cb, cr, o) == ref, (ss, q, ri, opt)


def test_entropy_thread_count_does_not_change_bytes(po):
    w, h = 1920, 1080
    img = po.gen_gradient_rgb(w, h)
    y, cb, cr = po.jpeg_coefficients(img, w, h, 2, 1, 80)
    ref = po.jpeg_encode_from_coefficients(y, cb, cr, w, h, 2, 80, 1)
    o = JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420)
    assert entropy_encode(y, cb, cr, o) == ref
    o.restart_interval = 120
    assert entropy_encode(y, cb, cr, o) == po.jpeg_encode_from_coefficients(y, cb, cr, w, h, 2, 80, 1, 120)


def test_all_ff_stuffing(po):
    """Coefficients chosen to emit long runs of 1 bits (0xFF bytes) at every alignment."""
    w, h = 64, 64
    rng = np.random.default_rng(3)
    y = np.zeros((64, 64), np.int16); y[:, :] = rng.choice([-1023, 1023, 511, -511], size=(64, 64))
    cb = np.zeros((0, 64), np.int16)
    ref = po.jpeg_encode_from_coefficients(y, cb, cb, w, h, 0, 80, 0)
    assert ref.count(b"\xff\x00") > 10
    o = JpegOptions(w, h, ColorType.Gray, 80, Subsampling.S444)
    assert entropy_encode(y, cb, cb, o) == ref


def test_quant_tables_match_oracle(po):
    from pixo_b200 import jpeg
    for q in list(range(1, 101)):
        a = jpeg.quant_tables(q); b = po.quant_tables(q)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_entropy_validation_errors():
    y = np.zeros((1, 64), np.int16)
    for q in (0, 101):
        with pytest.raises(pixo_b200.PixoError) as e:
            entropy_encode(y, y, y, JpegOptions(1, 1, ColorType.Rgb, q))
        assert e.value.code == pixo_b200._lib.ERR_INVALID_QUALITY
    with pytest.raises(pixo_b200.PixoError) as e:
        entropy_encode(y, y, y, JpegOptions(0, 1, ColorType.Rgb, 80))
    assert e.value.code == pixo_b200._lib.ERR_INVALID_DIMENSIONS
    with pytest.raises(pixo_b200.PixoError) as e:
        entropy_encode(y, y, y, JpegOptions(70000, 1, ColorType.Rgb, 80))
    assert e.value.code == pixo_b200._lib.ERR_IMAGE_TOO_LARGE
    with pytest.raises(pixo_b200.PixoError) as e:
        entropy_encode(y, y, y, JpegOptions(1, 1, ColorType.Rgba, 80))
    assert e.value.code == pixo_b200._lib.ERR_UNSUPPORTED_COLOR


def test_entropy_rejects_uncodable_coefficients_and_bad_restart():
    """ADVICE r1: the standard tables have no code for AC category > 10 / DC-difference category
    > 11, and the DRI field is 16 bits - reject instead of reading past the tables."""
    E = pixo_b200._lib
    o = JpegOptions(8, 8, ColorType.Gray, 80, Subsampling.S444)
    z = np.zeros((0, 64), np.int16)
    for pos, val in ((5, 1024), (5, -1024), (0, 2048), (0, -2048)):
        y = np.zeros((1, 64), np.int16); y[0, pos] = val
        with pytest.raises(pixo_b200.PixoError) as e:
            entropy_encode(y, z, z, o)
        assert e.value.code == E.ERR_INVALID_ARGUMENT
    y = np.zeros((1, 64), np.int16); y[0, 0] = 2047; y[0, 5] = -1023
    assert entropy_encode(y, z, z, o)[:2] == b"\xff\xd8"
    with pytest.raises(pixo_b200.PixoError) as e:
        entropy_encode(y, z, z, JpegOptions(8, 8, ColorType.Gray, 80, Subsampling.S444, 70000))
    assert e.value.code == E.ERR_INVALID_RESTART
    from pixo_b200 import jpeg
    for fn in (lambda: entropy_encode(y, z, z, JpegOptions(8, 8, ColorType.Gray, 80, Subsampling.S444, 0)),
               lambda: jpeg.encode_batch(np.zeros((1, 64), np.uint8), JpegOptions(8, 8, ColorType.Gray, 80, restart_interval=0))):
        with pytest.raises(pixo_b200.PixoError) as e:
            fn()
        assert e.value.code == E.ERR_INVALID_RESTART
    # -32768 after 15 zeros in Cr (its category would index one past the chroma AC statistics), and a
    # DC difference that is out of range only because the restart interval resets the predictor
    c = np.zeros((1, 64), np.int16)
    cr = c.copy(); cr[0, 12] = -32768          # natural 12 = zig-zag 16: 15 zeros before it
    y2 = np.zeros((2, 64), np.int16); y2[:, 0] = (2047, 4000)
    for args, opts in (((c, c, cr), JpegOptions(8, 8, ColorType.Rgb, 80, Subsampling.S444)),
                       ((y2, z, z), JpegOptions(16, 8, ColorType.Gray, 80, Subsampling.S444, 1))):
        with pytest.raises(pixo_b200.PixoError) as e:
            entropy_encode(*args, opts)
        assert e.value.code == E.ERR_INVALID_ARGUMENT
    assert entropy_encode(y2, z, z, JpegOptions(16, 8, ColorType.Gray, 80, Subsampling.S444))[:2] == b"\xff\xd8"
    # the band twins check the same rules, with the seed as the first predictor
    _band_twins_reject_out_of_range()


def _band_twins_reject_out_of_range():
    import ctypes as C
    E = pixo_b200._lib
    lib = E.load()
    z = np.zeros((1, 64), np.int16)

    def both(y, cb, cr, ct, seed):
        s = (C.c_int32 * 3)(*seed)
        hist = np.full(537, 7, np.uint64)
        raw = np.zeros(1 << 16, np.uint8)
        nbits, tail = C.c_uint64(), C.c_uint32()
        rh = lib.pixo_b200_jpeg_band_histogram(y.ctypes.data, cb.ctypes.data, cr.ctypes.data, 8, 8, ct, 0, s,
                                               hist.ctypes.data_as(E.u64p))
        assert hist[536] == 7
        re = lib.pixo_b200_jpeg_band_entropy(y.ctypes.data, cb.ctypes.data, cr.ctypes.data, 8, 8, ct, 0, s, None,
                                             raw.ctypes.data, raw.size, C.byref(nbits), C.byref(tail))
        return rh, re

    ac = z.copy(); ac[0, 1] = 1024
    assert both(ac, z, z, 0, (0, 0, 0)) == (E.ERR_INVALID_ARGUMENT,) * 2
    ok = z.copy(); ok[0, 0] = -1
    assert both(ok, z, z, 0, (2047, 0, 0)) == (E.ERR_INVALID_ARGUMENT,) * 2     # -1 - 2047: the seed counts
    assert both(ok, z, z, 0, (2046, 0, 0)) == (0, 0)
    assert both(z, z, ok, 2, (0, 0, 2047)) == (E.ERR_INVALID_ARGUMENT,) * 2      # Cr's own seed
    assert both(z, z, ok, 2, (0, 2047, 0)) == (0, 0)
    for nat in (12, 63):                                                          # run 15 / run 62
        cr = z.copy(); cr[0, nat] = -32768
        assert both(z, z, cr, 2, (0, 0, 0)) == (E.ERR_INVALID_ARGUMENT,) * 2
