"""The builders of tests/decode_inputs.py are right, so the full-size GPU decoder tests built on them test the
decoders: the vectorised filter equals the per-byte one, large PNGs decode through zlib and the C oracle to their
source rows, every JPEG the coefficient writer makes decodes in the oracle to exactly the written coefficients, and the
committed libjpeg-turbo files decode in the oracle (or are refused with pixo's messages)."""
import io
import json
import os
import zlib

import numpy as np
import pytest

from oracle import jpeg_decode as jd
from oracle import png_decode as pd
from decode_inputs import (RestartTail, expand_source, filter_rows_np, geometry, jfif, png_image, qtable,
                           dense_coefs, safe_tails, sparse_coefs)
from png_decode_corpus import DEPTHS, filter_bpp, filter_rows, row_bytes
import jpeg_decode_ref as ref

LIBJPEG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "libjpeg")


@pytest.mark.parametrize("bpp", range(1, 9))
def test_filter_rows_np_equals_filter_rows(bpp):
    rng = np.random.default_rng(bpp)
    raw = rng.integers(0, 256, (9, bpp * 7 + 3), dtype=np.uint8)
    for filters in ((0,), (1,), (2,), (3,), (4,), (4, 3, 2, 1, 0), (3, 5, 4)):
        assert filter_rows_np(raw, filters, bpp) == filter_rows(raw, filters, bpp), filters
    smooth = np.cumsum(rng.integers(0, 3, raw.shape), axis=1).astype(np.uint8)
    assert filter_rows_np(smooth, (4, 3), bpp) == filter_rows(smooth, (4, 3), bpp)


@pytest.mark.parametrize("ct,depth", [(ct, d) for ct, ds in DEPTHS.items() for d in ds])
def test_png_image_decodes_to_its_rows(ct, depth):
    """A tall file with random per-row filters: zlib gives back the filtered rows, and the oracle gives the frame
    the source rows make."""
    w = {1: 515, 2: 333, 4: 129, 8: 97, 16: 61}[depth]
    f, raw = png_image(w, 301, depth, ct, 7, filters="random", idat_chunks=[1, 4095, 4096, 4097, 65539])
    assert raw.shape == (301, row_bytes(w, depth, ct))
    filters = np.random.default_rng(8).integers(0, 5, 301)
    r = pd.decode(f)
    assert r.kind == pd.OK and (r.width, r.height) == (w, 301)
    assert np.array_equal(r.pixels, expand_source(raw, w, depth, ct, 7))
    stream = b"".join(f[o + 8:o + 8 + int.from_bytes(f[o:o + 4], "big")] for o in _idats(f))
    assert zlib.decompress(stream) == filter_rows_np(raw, filters, filter_bpp(depth, ct))


def _idats(f):
    o, out = 8, []
    while o < len(f):
        n = int.from_bytes(f[o:o + 4], "big")
        if f[o + 4:o + 8] == b"IDAT":
            out.append(o)
        o += 12 + n
    return out


def test_png_image_at_4k():
    f, raw = png_image(3840, 2160, 8, 6, 3, filters="random", level=1)
    r = pd.decode(f)
    assert r.kind == pd.OK and np.array_equal(r.pixels, raw.reshape(-1))


SAMPLINGS = [
    [(1, 1)], [(2, 3)], [(4, 1)],
    [(1, 1), (1, 1), (1, 1)], [(2, 2), (1, 1), (1, 1)], [(2, 1), (1, 1), (1, 1)], [(1, 2), (1, 1), (1, 1)],
    [(4, 1), (2, 1), (1, 1)], [(3, 2), (1, 1), (2, 1)], [(1, 1), (2, 2), (1, 1)], [(2, 3), (3, 2), (1, 4)],
    [(4, 4), (4, 4), (3, 3)],
]


@pytest.mark.parametrize("sampling", SAMPLINGS, ids=lambda s: "_".join(f"{h}x{v}" for h, v in s))
@pytest.mark.parametrize("restart", [0, 1, 7, "row", "over"])
@pytest.mark.parametrize("tables", ["standard", "optimal"])
def test_jfif_decodes_to_its_coefficients(sampling, restart, tables):
    """The oracle decodes every block the writer wrote, to exactly its coefficients, in decode order; on the smaller
    files the pure-Python restatement agrees with the oracle's pixels."""
    w, h = 8 * 4 * max(s[0] for s in sampling) + 3, 8 * 3 * max(s[1] for s in sampling) - 5
    mw, mh, bpm = geometry(w, h, [(a, b, None) for a, b in sampling])
    rs = {"row": mw, "over": mw * mh + 5}.get(restart, restart)
    for kind in ("sparse", "dense"):
        seed = len(sampling) * 100 + bpm + (restart if isinstance(restart, int) else 50) + (kind == "dense")
        big = tables == "optimal" and kind == "dense"
        comps = [(a, b, qtable(seed + c, 65535 if kind == "dense" else 255)) for c, (a, b) in enumerate(sampling)]
        C = sparse_coefs(mw * mh * bpm, seed) if kind == "sparse" else \
            dense_coefs(mw * mh * bpm, seed, 15 if big else 10, 16 if big else 11)
        C = safe_tails(C, bpm, rs, mw * mh, seed)
        data = jfif(w, h, comps, C, restart=rs, tables=tables)
        r = jd.decode(data)
        assert r.status == jd.OK and r.stored == r.blocks == C.n, (r.status, r.message, r.stored, C.n)
        assert np.array_equal(r.coefs, C.dense())
        if C.n <= 200:
            assert ref.decode(data) == ("ok", w, h, r.color_type, r.pixels.tobytes())


def test_jfif_16bit_dqt_wraps_the_idct():
    """Dense blocks times a 16-bit table overflow the IDCT's i32: the oracle and the restatement wrap alike."""
    comps = [(1, 1, [65535] * 64)]
    C = dense_coefs(4, 1, 10, 11, density=1.0)
    data = jfif(16, 16, comps, C)
    assert data[data.index(b"\xFF\xDB") + 4] == 0x10   # a 16-bit DQT
    r = jd.decode(data)
    assert r.status == jd.OK and np.array_equal(r.coefs, C.dense())
    assert ref.decode(data) == ("ok", 16, 16, 0, r.pixels.tobytes())
    c = C.dense()[0].astype(np.int64)
    assert (np.abs(c) * 65535 << 13).max() >= 1 << 31


def test_jfif_refuses_a_restart_tail_pixos_reader_would_drop():
    """An interval that ends on a short EOB is a file pixo decodes wrongly: the writer refuses it unless
    safe_tails ends each interval on a long code."""
    comps = [(1, 1, [1] * 64)]
    C = sparse_coefs(16, 2, nac=0)
    with pytest.raises(RestartTail):
        jfif(32, 32, comps, C, restart=1)
    data = jfif(32, 32, comps, safe_tails(C, 1, 1, 16), restart=1)
    assert data.count(b"\xFF\xD0") == 2 and data.count(b"\xFF\xD7") == 1
    assert jd.decode(data).stored == 16


def test_jfif_stuffs_ff():
    comps = [(1, 1, [1] * 64)]
    C = dense_coefs(64, 3)
    data = jfif(64, 64, comps, C)
    scan = data[data.index(b"\xFF\xDA") + 2 + 10:-2]
    assert scan.count(b"\xFF\x00") > 0 and scan.count(b"\xFF") == scan.count(b"\xFF\x00")
    assert np.array_equal(jd.decode(data).coefs, C.dense())


def libjpeg_files():
    m = json.load(open(os.path.join(LIBJPEG, "manifest.json")))
    return [(c, open(os.path.join(LIBJPEG, c["file"]), "rb").read()) for c in m]


def test_libjpeg_fixtures_decode_in_the_oracle():
    files = libjpeg_files()
    assert len(files) == 48 and sum(len(d) for _, d in files) < 400_000
    for c, data in files:
        r = jd.decode(data, coefs=False)
        if c["file"] == "refused_cmyk.jpg":
            assert (r.status, r.message) == (jd.UNSUPPORTED, "4 components not supported")
        elif c["file"] == "refused_progressive.jpg":
            assert (r.status, r.message) == (jd.UNSUPPORTED, "progressive JPEG not supported")
        else:
            assert r.status == jd.OK and (r.width, r.height) == (c["w"], c["h"]), c["file"]
            assert r.color_type == (0 if c["sub"] == "gray" else 2)


def test_libjpeg_fixtures_plausible_against_pil():
    """The PSNR floor of test_jpeg_decode.test_plausible_against_pil.  Files with restart markers are left out:
    pixo's reader clears its bit buffer at each RSTn, so it drops bits libjpeg-turbo's intervals end on."""
    Image = pytest.importorskip("PIL.Image")
    worst = 99.0
    for c, data in libjpeg_files():
        if c["refused"] or c["restart"]:
            continue
        r = jd.decode(data, coefs=False)
        im = np.asarray(Image.open(io.BytesIO(data)).convert("L" if r.color_type == 0 else "RGB")).reshape(-1)
        d = im.astype(float) - r.pixels
        worst = min(worst, 10 * np.log10(255 ** 2 / max((d ** 2).mean(), 1e-9)))
    assert worst > 6.0, worst
