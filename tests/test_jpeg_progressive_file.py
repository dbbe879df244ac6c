"""pixo_b200_jpeg_progressive_file: a whole progressive file from one frame's tables and its 7 segments (what
pixo_b200_jpeg_encode_dev_progressive leaves in a slot).  Every real-pixo max-preset file and progressive fixture,
and oracle files over the colour modes and restart intervals, come back byte for byte from their own DHT and
segments.  Host-only: no GPU needed."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import jpeg_progressive_scans as ps
from oracle import jpeg_progressive as jp
from pixo_b200 import ColorType, _lib, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from progressive_inputs import make_progressive_input
from trellis_inputs import make_trellis_input

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _manifest(sub):
    with open(os.path.join(GOLD, sub, "manifest.json")) as f:
        return json.load(f)["jpeg"]


def _read(sub, name):
    with open(os.path.join(GOLD, sub, name), "rb") as f:
        return f.read()


def parts(data: bytes):
    """A progressive file's DHT block, its 7 segments back to back and their lengths."""
    sc = ps.scans(data)
    assert [(c, ss, se) for c, ss, se, _, _, _ in sc] == [([c], ss, se) for c, ss, se in ps.SCRIPT]
    segs = [s[5] for s in sc]
    return jpeg.dht_array(ps.dht(data)), b"".join(segs), [len(s) for s in segs]


def rebuild(data: bytes, o: JpegOptions) -> bytes:
    return jpeg.progressive_file(o, *parts(data))


def opts(w, h, ct, ss, q, ri=0):
    return JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), ri or None, True, True, True)


@pytest.mark.parametrize("e", _manifest("trellis"), ids=lambda e: e["file"])
def test_rebuilds_pixo_max_files(lib, e):
    data = _read("trellis", e["file"])
    assert rebuild(data, opts(e["w"], e["h"], e["ct"], e["s420"], e["q"])) == data


@pytest.mark.parametrize("e", _manifest("progressive"), ids=lambda e: e["file"])
def test_rebuilds_progressive_fixtures(lib, e):
    data = _read("progressive", e["file"])
    assert rebuild(data, opts(e["w"], e["h"], e["ct"], e["s420"], e["q"])) == data


@pytest.mark.parametrize("ri", [0, 5])
@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
def test_rebuilds_oracle_files(lib, ct, ss, ri):
    jp.build()
    for i, (w, h) in enumerate([(1, 1), (17, 9), (64, 33)]):
        for trellis, optimize in ((True, True), (False, False), (False, True)):
            img = make_trellis_input(["noise", "smooth", "hifreq"][i], w, h, 1 if ct == 0 else 3, i)
            data = jp.encode(img, w, h, ct, ss, 80, ri, optimize, trellis)
            assert rebuild(data, opts(w, h, ct, ss, 80, ri)) == data, (w, h, trellis, optimize)


def test_standard_tables_when_dht_is_none(lib):
    jp.build()
    img = make_trellis_input("smooth", 40, 33, 3, 7)
    data = jp.encode(img, 40, 33, 2, 1, 75, 0, False, False)
    _, segs, lens = parts(data)
    assert jpeg.progressive_file(opts(40, 33, 2, 1, 75), None, segs, lens) == data


def _call(o, dht, segs, lens, cap):
    d = np.ascontiguousarray(dht, np.uint8).reshape(-1)
    s = np.frombuffer(segs, np.uint8) if segs else np.zeros(1, np.uint8)
    ln = np.ascontiguousarray(lens, np.uint64)
    out = np.zeros(max(cap, 1), np.uint8)
    n = C.c_size_t(12345)
    rc = _lib.load().pixo_b200_jpeg_progressive_file(
        int(o.width), int(o.height), int(o.color_type), int(o.quality), int(o.subsampling),
        int(o.restart_interval or 0), d.ctypes.data, s.ctypes.data, ln.ctypes.data_as(_lib.u64p), out.ctypes.data,
        cap, C.byref(n))
    return rc, out, n.value


def test_refuses_short_output_malformed_tables_and_bad_options(lib):
    e = _manifest("progressive")[2]
    data = _read("progressive", e["file"])
    o = opts(e["w"], e["h"], e["ct"], e["s420"], e["q"])
    dht, segs, lens = parts(data)
    rc, out, n = _call(o, dht, segs, lens, len(data))
    assert rc == 0 and n == len(data) and out[:n].tobytes() == data
    rc, out, n = _call(o, dht, segs, lens, len(data) - 1)
    assert rc == _lib.ERR_OUTPUT_TOO_SMALL and n == 12345 and not out.any()
    bad = dht.copy()
    bad[2, :16] = 0
    bad[2, 8] = 255
    bad[2, 9] = 255                               # 510 values
    assert _call(o, bad, segs, lens, len(data) + 1024)[0] == _lib.ERR_INVALID_ARGUMENT
    bad = dht.copy()
    bad[0, :16] = 0
    bad[0, 0] = 3                                 # three 1-bit codes
    assert _call(o, bad, segs, lens, len(data) + 1024)[0] == _lib.ERR_INVALID_ARGUMENT
    for o2, code in ((opts(e["w"], e["h"], e["ct"], e["s420"], 0), _lib.ERR_INVALID_QUALITY),
                     (opts(e["w"], e["h"], e["ct"], e["s420"], e["q"], 70000), _lib.ERR_INVALID_RESTART),
                     (opts(0, e["h"], e["ct"], e["s420"], e["q"]), _lib.ERR_INVALID_DIMENSIONS),
                     (opts(e["w"], 70000, e["ct"], e["s420"], e["q"]), _lib.ERR_IMAGE_TOO_LARGE),
                     (JpegOptions(e["w"], e["h"], ColorType.Rgba, e["q"], Subsampling.S444), _lib.ERR_UNSUPPORTED_COLOR)):
        rc, out, n = _call(o2, dht, segs, lens, len(data) + 1024)
        assert rc == code and not out.any(), (o2, rc)
    with pytest.raises(_lib.PixoError):
        jpeg.progressive_file(o, dht, segs, lens[:6])
