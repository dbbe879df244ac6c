"""The baseline JPEG decoder's contract on the CPU: pixo's own decoder tests restated against the C oracle
(oracle/jpeg_decode.c) and the host-only pixo_b200_jpeg_decode_info; the oracle's entropy stage against real pixo
files; and the oracle against an independent pure-Python restatement (tests/jpeg_decode_ref.py)."""
import glob
import io
import json
import os

import numpy as np
import pytest

import pixo_b200
from pixo_b200 import ColorType, decode
from oracle import jpeg_decode as jd
from oracle import pyoracle as po
from golden_inputs import make_input
from jpeg_decode_corpus import constructed, corrupted, seg, sof0, truncations
import jpeg_decode_ref as ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MANIFEST = json.load(open(os.path.join(GOLD, "manifest.json")))["jpeg"]
ZZ = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
      21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
      61, 54, 47, 55, 62, 63]
KIND = {jd.INVALID: "invalid", jd.UNSUPPORTED: "unsupported", jd.PANIC: "panic"}

DQT = seg(0xDB, b"\x00" + bytes([16] * 64))
SOF_8x8 = bytes([0xFF, 0xC0, 0x00, 0x0B, 0x08, 0x00, 0x08, 0x00, 0x08, 0x01, 0x01, 0x11, 0x00])
DHT_DC = bytes([0xFF, 0xC4, 0x00, 0x14, 0x00]) + bytes([0, 1] + [0] * 14) + b"\x00"
SOI, EOI = b"\xFF\xD8", b"\xFF\xD9"


def err(data):
    r = jd.decode(data)
    assert r.status != jd.OK
    return r.status, r.message


def both_refuse(data, kind, text):
    """the oracle, the Python restatement and pixo_b200_jpeg_decode_info refuse `data` alike"""
    st, msg = err(data)
    assert st == kind and text in msg, (st, msg)
    assert ref.decode(data) == (KIND[st], msg)
    with pytest.raises(pixo_b200.PixoError) as e:
        decode.jpeg_info(data)
    want = {jd.UNSUPPORTED: pixo_b200._lib.ERR_UNSUPPORTED_DECODE}.get(st, pixo_b200._lib.ERR_INVALID_DECODE)
    assert e.value.code == want
    assert str(e.value) == ("Unsupported: " if st == jd.UNSUPPORTED else "Decode error: ") + msg


# ---- pixo's decoder tests (src/decode/jpeg.rs:745-1273) ----

I, U = jd.INVALID, jd.UNSUPPORTED


@pytest.mark.parametrize("data,kind,text", [
    (b"not a jpeg", I, "not a JPEG file"), (b"", I, "not a JPEG file"), (SOI, I, "unexpected end of file"),
    (b"\xFF\xD9\xFF\xD8", I, "not a JPEG file"),
    (SOI + b"\xFF\xDB\x00\x43", I, "invalid marker length"),                       # truncated DQT
    (SOI + b"\xFF\xC0\x00\x0B\x08", I, "invalid marker length"),                   # truncated SOF
    (SOI + DQT + bytes([0xFF, 0xC0, 0x00, 0x0B, 0x08, 0, 0, 0, 8, 1, 1, 0x11, 0]) + EOI, I, "no image data found"),
    (SOI + b"\xFF\x01", I, "truncated marker"),
    (SOI + DQT + DHT_DC + b"\xFF\xDA\x00\x08\x01\x01\x00\x00\x3F\x00" + EOI, I, "SOS component count mismatch"),
    (SOI + DQT + bytes([0xFF, 0xC0, 0x00, 0x08, 0x08, 0, 8, 0, 8, 0]) + EOI, I, "invalid SOF0 length"),
    (SOI + seg(0xC0, bytes([8, 0, 8, 0, 8, 0, 0, 0])) + EOI, U, "0 components not supported"),
    (SOI + seg(0xE0, b"JFIF\x00" + bytes([1, 1, 0, 0, 1, 0, 1, 0, 0])) + EOI, I, "no image data found"),
    (SOI + seg(0xFE, b"test") + EOI, I, "no image data found"),
    (SOI + SOF_8x8[:11] + b"\x00\x00" + EOI, I, "invalid sampling factors 0x0 for component 1"),
    (SOI + SOF_8x8[:12] + b"\x05" + EOI, I, "invalid quantization table ID 5 for component 1"),
    (SOI + DQT + SOF_8x8 + DHT_DC + b"\xFF\xDA\x00\x08\x01\x01\x50\x00\x3F\x00" + EOI,
     I, "invalid DC Huffman table ID 5 for component 1"),
    (SOI + DQT + SOF_8x8 + DHT_DC + b"\xFF\xDA\x00\x08\x01\x01\x07\x00\x3F\x00" + EOI,
     I, "invalid AC Huffman table ID 7 for component 1"),
    (SOI + seg(0xC4, b"\x05" + bytes(16)), I, "invalid Huffman table ID"),
    (SOI + seg(0xC4, b"\x00" + bytes([0, 2] + [0] * 14) + b"\x00"), I, "truncated DHT values"),
    (SOI + seg(0xDD, b"\x00"), I, "invalid DRI length"),
    (SOI + seg(0xC0, bytes([12, 0, 8, 0, 8, 1, 1, 0x11, 0])), U, "12-bit precision not supported"),
    (SOI + seg(0xDA, b""), I, "empty SOS segment"),
], ids=lambda v: v if isinstance(v, str) else None)
def test_pixo_refusals(data, kind, text):
    both_refuse(data, kind, text)


def test_sof2_is_unsupported():
    data = SOI + DQT + bytes([0xFF, 0xC2, 0x00, 0x0B, 0x08, 0, 8, 0, 8, 1, 1, 0x11, 0]) + EOI
    both_refuse(data, jd.UNSUPPORTED, "progressive JPEG not supported")


def test_sos_without_components_is_refused():
    """pixo panics here (ycbcr_to_rgb indexes components[1]); the decoder refuses the file instead"""
    both_refuse(SOI + seg(0xDA, b"\x00\x00\x3F\x00") + EOI, jd.PANIC, "SOS with no frame components")


def test_missing_dht_decodes_to_a_zero_image():
    data = SOI + DQT + SOF_8x8 + b"\xFF\xDA\x00\x08\x01\x01\x00\x00\x3F\x00" + EOI
    r = jd.decode(data)
    assert (r.status, r.width, r.height, r.stored) == (jd.OK, 8, 8, 0)
    assert not r.pixels.any()
    assert decode.jpeg_info(data) == (8, 8, ColorType.Gray)
    assert ref.decode(data) == ("ok", 8, 8, 0, bytes(64))


def test_zero_height_with_a_scan_is_an_empty_image():
    data = SOI + DQT + bytes([0xFF, 0xC0, 0x00, 0x0B, 0x08, 0, 0, 0, 8, 1, 1, 0x11, 0]) + DHT_DC + \
        b"\xFF\xDA\x00\x08\x01\x01\x00\x00\x3F\x00" + EOI
    r = jd.decode(data)
    assert (r.status, r.width, r.height, r.pixels.size) == (jd.OK, 8, 0, 0)


@pytest.mark.parametrize("data,end", [
    (b"\x12\x34\xFF\xD9", 2), (b"\x12\xFF\x00\x34\xFF\xD9", 4), (b"\x12\xFF\xD0\x34\xFF\xD9", 4),
    (b"\xFF\x00\xFF\x00\xFF\xD9", 4), (b"\x12\x34\x56\x78", 4), (b"", 0), (b"\xFF", 1), (b"\x12", 1),
])
def test_find_entropy_end(data, end):
    assert jd.find_entropy_end(data) == end == ref.entropy_end(data)


def test_read_amplitude_and_tables():
    r = ref.Bits(bytes([0b01101111]))
    assert [ref.amplitude(r, 1), ref.amplitude(r, 2), ref.amplitude(r, 3)] == [-1, 3, -4]
    t = ref.Table([0, 2, 1] + [0] * 13, b"\x00\x01\x02")
    assert (t.maxcode[2], t.maxcode[3]) == (1, 4)
    assert ref.Table([0] * 16, b"").maxcode[1] == -1


def test_bit_reader():
    """bit_reader.rs's MsbBitReader tests, and the RSTn quirk: an 8-bit peek that fetches the byte after RSTn
    clears the bits still unread"""
    r = ref.Bits(bytes([0xFF, 0x00, 0xAB]))
    assert (r.read(8), r.read(8)) == (0xFF, 0xAB)
    r = ref.Bits(bytes([0xAB, 0xFF, 0xD0, 0xCD]))
    assert (r.read(4), r.read(8)) == (0b1010, 0xCD)
    r = ref.Bits(bytes([0x12, 0x34, 0xFF, 0xD1, 0xAB]))
    assert (r.read(16), r.read(8)) == (0x1234, 0xAB)
    r = ref.Bits(bytes([0x12, 0x34, 0x56, 0x78, 0x9A]))
    r.peek(25)
    r.consume(0)
    assert r.peek(8) == 0x12
    r = ref.Bits(b"")
    with pytest.raises(ref.Bits.End):
        r.read(1)


def test_idct():
    q = np.ones(64, np.uint16)
    assert (jd.idct_block(np.zeros(64, np.int16), q) == 128).all()
    c = np.zeros(64, np.int16)
    c[0] = 1000
    out = jd.idct_block(c, q)
    assert (out == out[0]).all() and out[0] == 253
    rng = np.random.default_rng(3)
    for _ in range(200):
        c = rng.integers(-32768, 32768, 64).astype(np.int16)
        q = rng.integers(0, 65536, 64).astype(np.uint16)
        assert list(jd.idct_block(c, q)) == ref.idct([int(x) for x in c], [int(x) for x in q])


# ---- the entropy stage against real pixo ----

@pytest.mark.parametrize("c", MANIFEST, ids=lambda c: c["file"])
def test_golden_coefficients_equal_the_encoders(c):
    r = jd.decode(open(os.path.join(GOLD, c["file"]), "rb").read())
    assert r.status == jd.OK and r.stored == r.blocks
    img = make_input(c["kind"], c["w"], c["h"], 1 if c["ct"] == 0 else 3, c["seed"])
    y, cb, cr = po.jpeg_coefficients(img, c["w"], c["h"], c["ct"], c["s420"], c["q"])
    nat = np.zeros_like(r.coefs)
    nat[:, ZZ] = r.coefs
    if c["ct"] == 0:
        want = y
    else:
        bpm = 4 if c["s420"] else 1
        want = np.concatenate([np.concatenate([y[i * bpm:(i + 1) * bpm], cb[i:i + 1], cr[i:i + 1]])
                               for i in range(len(y) // bpm)])
    assert np.array_equal(nat, want)


def test_progressive_goldens_are_refused():
    files = sorted(glob.glob(os.path.join(GOLD, "trellis", "*.jpg")) + glob.glob(os.path.join(GOLD, "progressive", "*.jpg")))
    assert len(files) == 55   # 51 trellis and 4 progressive real-pixo files
    for p in files:
        assert err(open(p, "rb").read()) == (jd.UNSUPPORTED, "progressive JPEG not supported"), p


def test_plausible_against_pil():
    """A plausibility floor only: pixo's IDCT scales its odd part down by 2^13, so its pixels are far from a
    conforming decoder's; the largest difference is recorded, not pinned."""
    Image = pytest.importorskip("PIL.Image")
    worst, maxdiff = 99.0, 0
    for c in MANIFEST:
        data = open(os.path.join(GOLD, c["file"]), "rb").read()
        r = jd.decode(data, coefs=False)
        im = np.asarray(Image.open(io.BytesIO(data)).convert("L" if r.color_type == 0 else "RGB")).reshape(-1)
        d = im.astype(float) - r.pixels
        worst = min(worst, 10 * np.log10(255 ** 2 / max((d ** 2).mean(), 1e-9)))
        maxdiff = max(maxdiff, int(np.abs(d).max()))
    assert worst > 6.0, worst
    print(f"worst PSNR {worst:.1f} dB, max difference {maxdiff}")


# ---- two restatements agree ----

def _agree(data):
    r = jd.decode(data, coefs=False)
    got = ref.decode(data)
    if r.status != jd.OK:
        assert got == (KIND[r.status], r.message)
    else:
        assert got == ("ok", r.width, r.height, r.color_type, r.pixels.tobytes())


@pytest.mark.parametrize("seed", range(60))
def test_constructed_files_agree(seed):
    _agree(constructed(seed))


@pytest.mark.parametrize("first,second", [
    (b"\x01\x44\x00\x02\x11\x00\x03\x11\x00", b"\x01\x11\x00"),                         # gray after 4x4 colour
    (b"\x01\xFF\x00\x02\x11\x00\x03\x11\x00", b"\x01\x11\x00"),                         # gray after 15x15
    (b"\x01\x44\x00\x02\x11\x00\x03\x11\x00", b"\x01\x11\x00\x02\x11\x00\x03\x11\x00"),  # colour after colour
])
def test_a_second_sof0_keeps_the_first_ones_maxima(first, second):
    """pixo never resets max_h / max_v_sampling, so the planes of the second SOF0 are sized by the first one's MCUs
    and can be smaller than the frame: pixels past a plane read 0 (Y) or 128 (Cb, Cr)"""
    dht = seg(0xC4, b"\x00" + bytes([0, 1] + [0] * 14) + b"\x00") + seg(0xC4, b"\x10" + bytes([0, 1] + [0] * 14) + b"\x00")
    nc = len(second) // 3
    sos = seg(0xDA, bytes([nc]) + b"".join(bytes([c + 1, 0]) for c in range(nc)) + b"\x00\x3F\x00")
    data = SOI + DQT + sof0(64, 64, first) + sof0(64, 64, second) + dht + sos + bytes(200) + EOI
    r = jd.decode(data, coefs=False)
    assert r.status == jd.OK and r.pixels.size == 64 * 64 * (1 if nc == 1 else 3)
    _agree(data)
    if nc == 1:
        assert r.pixels.reshape(64, 64)[63, 63] == 0   # past the 4 x 8-row plane


def test_truncations_and_corruptions_agree():
    small = po.jpeg_encode(po.gen_noise(11, 9, 3, 4), 11, 9, po.RGB, 90, po.S420, 1)
    for f in truncations(small) + corrupted(small, 2, 40):
        _agree(f)


def test_restart_quirk_is_reproduced():
    """a file with restart interval 1 decodes fully; the C oracle and the restatement agree on it and on its
    RSTn-less twin, whose scan runs on past each interval's padding"""
    f = po.jpeg_encode(po.gen_noise(24, 16, 3, 9), 24, 16, po.RGB, 75, po.S444, 1)
    r = jd.decode(f)
    assert r.status == jd.OK and r.stored == r.blocks
    _agree(f)
    stripped = bytearray()
    i = 0
    while i < len(f):
        if f[i] == 0xFF and i + 1 < len(f) and 0xD0 <= f[i + 1] <= 0xD7:
            i += 2
            continue
        stripped.append(f[i])
        i += 1
    _agree(bytes(stripped))


def test_info_matches_oracle_geometry():
    for s in range(40):
        f = constructed(s)
        r = jd.decode(f, pixels=False, coefs=False)
        assert decode.jpeg_info(f) == (r.width, r.height, ColorType(r.color_type))
