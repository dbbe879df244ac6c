"""pixo_b200_jpeg_write_headers_dht: the headers of a file written from the tables a scan was coded with
(the DHT blocks pixo_b200_jpeg_encode_dev_opts hands back).  Host-only: no GPU needed."""
import ctypes as C

import numpy as np
import pytest

from pixo_b200 import ColorType, _lib, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling


def dht_from_oracle(t) -> np.ndarray:
    """The oracle's po_huff_tables as a 4 x 272 DHT block (16 counts, then the values, zero-padded)."""
    a = np.zeros((4, 272), np.uint8)
    for k in range(4):
        a[k, :16] = list(t.bits[k])
        a[k, 16:16 + t.nvals[k]] = list(t.vals[k])[:t.nvals[k]]
    return a


def oracle_tables(po, hist, has_chroma):
    """pixo's tables for a histogram (standard ones when optimized_from_counts gives None) and whether
    they are the optimised ones."""
    t = po.HuffTables()
    ok = po.lib().po_huff_optimized(np.ascontiguousarray(hist, np.uint64).ctypes.data_as(po.u64p),
                                    int(has_chroma), C.byref(t))
    if not ok:
        po.lib().po_huff_standard(C.byref(t))
    return t, bool(ok)


def headers_hist(w, h, ct, q, ss, ri, hist):
    buf = np.zeros(2048, np.uint8)
    n = C.c_size_t()
    hp = None if hist is None else np.ascontiguousarray(hist, np.uint64).ctypes.data_as(_lib.u64p)
    _lib.check(None, _lib.load().pixo_b200_jpeg_write_headers(w, h, ct, q, ss, ri, hp, buf.ctypes.data, buf.size,
                                                              C.byref(n)))
    return buf[:n.value].tobytes()


def options(w, h, ct, q, ss, ri):
    return JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), ri or None, True)


@pytest.mark.parametrize("ct,ss", [(0, 0), (2, 1), (2, 0)])
@pytest.mark.parametrize("ri", [0, 3])
def test_standard_tables_give_write_headers_without_statistics(po, ct, ss, ri):
    t = po.HuffTables()
    po.lib().po_huff_standard(C.byref(t))
    got = jpeg.write_headers_dht(options(37, 19, ct, 80, ss, ri), dht_from_oracle(t))
    assert got == headers_hist(37, 19, ct, 80, ss, ri, None)


@pytest.mark.parametrize("ct,ss", [(0, 0), (2, 1), (2, 0)])
@pytest.mark.parametrize("ri", [0, 3])
@pytest.mark.parametrize("w,h,kind,seed", [(64, 48, "noise", 1), (97, 33, "smooth", 2), (16, 16, "noise", 3)])
def test_optimised_tables_give_write_headers_from_statistics(po, ct, ss, ri, w, h, kind, seed):
    ch = 3 if ct == 2 else 1
    img = po.gen_noise(w, h, ch, seed) if kind == "noise" else \
        np.roll(po.gen_gradient_rgb(w, h).reshape(h, -1), seed, axis=1).reshape(-1)[: w * h * ch].copy()
    hist = po.jpeg_histograms(*po.jpeg_coefficients(img, w, h, ct, ss, 75), w, h, ct, ss, ri)
    t, ok = oracle_tables(po, hist, ct != 0)
    assert ok
    got = jpeg.write_headers_dht(options(w, h, ct, 75, ss, ri), dht_from_oracle(t))
    assert got == headers_hist(w, h, ct, 75, ss, ri, hist)


def test_headers_and_scan_make_the_oracle_file(po):
    """jpeg_file = headers for the tables + scan + EOI: the oracle's file when the scan is the oracle's."""
    w, h = 40, 24
    img = po.gen_noise(w, h, 3, 9)
    want = po.jpeg_encode(img, w, h, 2, 90, 1, 2, True)
    hist = po.jpeg_histograms(*po.jpeg_coefficients(img, w, h, 2, 1, 90), w, h, 2, 1, 2)
    t, _ = oracle_tables(po, hist, True)
    o = options(w, h, 2, 90, 1, 2)
    hdr = jpeg.write_headers_dht(o, dht_from_oracle(t))
    assert jpeg.jpeg_file(o, dht_from_oracle(t), want[len(hdr):-2]) == want


def _call(dht, cap=2048):
    buf = np.zeros(max(cap, 1), np.uint8)
    n = C.c_size_t()
    d = np.ascontiguousarray(dht, np.uint8)
    return _lib.load().pixo_b200_jpeg_write_headers_dht(64, 64, 2, 80, 1, 0, d.ctypes.data, buf.ctypes.data, cap,
                                                         C.byref(n)), n.value


def test_malformed_blocks_are_rejected(po):
    t = po.HuffTables()
    po.lib().po_huff_standard(C.byref(t))
    good = dht_from_oracle(t)
    assert _call(good)[0] == _lib.OK
    too_many = good.copy()
    too_many[2, 15] = 255   # 162 - 125 + 255 = 292 values
    assert _call(too_many)[0] == _lib.ERR_INVALID_ARGUMENT
    no_room = good.copy()
    no_room[0, :16] = 0
    no_room[0, 0] = 3       # three codes of length 1
    assert _call(no_room)[0] == _lib.ERR_INVALID_ARGUMENT
    assert _call(good, cap=1023)[0] == _lib.ERR_OUTPUT_TOO_SMALL
    with pytest.raises(_lib.PixoError) as e:
        jpeg.write_headers_dht(options(8, 8, 2, 80, 1, 0), good[:3])
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT


def test_a_block_of_256_values_per_table_fits_its_headers():
    """Four full tables (1024 values): 1299 header bytes for a colour frame without DRI, more than the
    1024 pixo_b200_jpeg_write_headers asks for."""
    d = np.zeros((4, 272), np.uint8)
    d[:, 8] = 255       # 255 codes of length 9 and one of length 10: they fit
    d[:, 9] = 1
    d[:, 16:] = np.arange(256, dtype=np.uint8)
    rc, n = _call(d)
    assert rc == _lib.OK and n == 275 + 1024
    assert _call(d, cap=n - 1)[0] == _lib.ERR_OUTPUT_TOO_SMALL
