"""The host entropy coder and the host band twins on constructed coefficients (tests/coef_corpus.py)
against the oracle, every output checked again by an independent T.81 decoder
(tests/jpeg_scan_decode.py).  CPU only."""
import json
import os

import numpy as np
import pytest

import coef_corpus as cc
import jpeg_scan_decode as jd
from golden_inputs import make_input
from pixo_b200 import ColorType, parallel
from pixo_b200.jpeg import JpegOptions, Subsampling, entropy_encode

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def restart_intervals(case):
    """none, 1, 3, and an interval of at least one 32-block chunk that does not divide the MCU count"""
    y, cb, cr, w, h, ct, ss = case
    bpm = (4 if ss == 1 and ct == 2 else 1) + (2 if ct == 2 else 0)
    mcus = len(cb) if ct == 2 else len(y)
    ri = (32 + bpm - 1) // bpm
    while mcus % ri == 0:
        ri += 1
    assert ri < mcus
    return (0, 1, 3, ri)


def encode_both(po, case, ri, opt):
    y, cb, cr, w, h, ct, ss = case
    ref = po.jpeg_encode_from_coefficients(y, cb, cr, w, h, ct, 80, ss, ri, opt)
    got = entropy_encode(y, cb, cr, JpegOptions(w, h, ColorType(ct), 80, Subsampling(ss), ri or None, opt))
    return got, ref


def assert_decodes_to(jpg, case, **kw):
    y, cb, cr = case[:3]
    d = jd.decode(jpg, **kw)
    assert np.array_equal(d.y, y) and np.array_equal(d.cb, cb) and np.array_equal(d.cr, cr)
    return d


def test_decoder_reproduces_the_golden_coefficients(po):
    """Ties the decoder to pixo itself: every golden JPEG (real pixo output) decodes to the
    coefficients of its input."""
    manifest = json.load(open(os.path.join(GOLD, "manifest.json")))
    for c in manifest["jpeg"]:
        img = make_input(c["kind"], c["w"], c["h"], 3 if c["ct"] == 2 else 1, c["seed"])
        want = po.jpeg_coefficients(img, c["w"], c["h"], c["ct"], c["s420"], c["q"])
        assert_decodes_to(open(os.path.join(GOLD, c["file"]), "rb").read(), want)


def test_decoder_rejects_what_a_baseline_encoder_must_not_write(po):
    case = cc.zero_runs(cc.GRAY, cc.S444)
    y, cb, cr, w, h, ct, ss = case
    jpg = po.jpeg_encode_from_coefficients(y, cb, cr, w, h, ct, 80, ss, 2)
    d = assert_decodes_to(jpg, case)
    assert d.tables[(1, 0)] == (cc.AC_LUM_BITS, list(cc.AC_LUM_VALS))      # the Annex K tables
    assert d.tables[(0, 0)] == (cc.DC_LUM_BITS, list(range(12)))
    scan = jd.scan_bytes(jpg)
    at = len(jpg) - 2 - len(scan)
    rst = jpg.index(b"\xff\xd0", at)
    bad = [jpg[:rst + 1] + b"\xd1" + jpg[rst + 2:],                        # RST1 where RST0 belongs
           jpg[:-2] + b"\xff\xd0\xff\xd9",                                 # RSTn right before EOI
           jpg[:rst - 1] + bytes([jpg[rst - 1] & 0xFE]) + jpg[rst:]]       # a 0-bit in the padding
    dht = jpg.index(b"\xff\xc4")           # the first DHT (luma DC) -> two 1-bit codes: a full code space
    full = b"\xff\xc4" + (2 + 1 + 16 + 2).to_bytes(2, "big") + bytes([0x00, 2] + [0] * 15 + [0, 1])
    bad.append(jpg[:dht] + full + jpg[dht + 2 + int.from_bytes(jpg[dht + 2:dht + 4], "big"):])
    for b in bad:
        with pytest.raises(jd.ScanError):
            jd.decode(b)


def test_corpus_reaches_its_edges(po):
    # every symbol of the standard tables, in both table classes, and every DC category
    y, cb, cr, w, h, ct, ss = cc.symbol_sweep()
    hist = po.jpeg_histograms(y, cb, cr, w, h, ct, ss)
    for base, syms in ((0, range(12)), (12, range(12)), (24, cc.AC_LUM_VALS), (280, cc.AC_CHR_VALS)):
        assert all(hist[base + s] for s in syms), base
    for arr in (y, cb, cr):     # both signs of every DC category
        d = np.diff(np.concatenate([[0], arr[:, 0].astype(np.int64)]))
        assert {int(np.sign(v)) * cc.category(v) for v in d} >= set(range(-11, 12))
    # runs of 15..62 zeros, ZRL counts of 1..3
    case = cc.zero_runs(cc.GRAY, cc.S444)
    hist = po.jpeg_histograms(*case)
    assert hist[24 + 0xF0] >= 12 and hist[24 + 0xEA]       # ZRLs; only zig-zag 63 set: 3 x ZRL + (14, 10)
    # Fibonacci statistics: an unconstrained tree deeper than 16 levels, and one with 16-bit codes
    deep = cc.fibonacci(22)
    assert cc.huffman_depth(po.jpeg_histograms(*deep[:3], *deep[3:6])[24:280]) > 16
    bits = jd.decode(po.jpeg_encode_from_coefficients(*cc.fibonacci(19)[:6], 80, 0, 0, True)).tables[(1, 0)][0]
    assert bits != cc.AC_LUM_BITS and bits[15] > 0                         # optimised AC table, 16-bit codes
    # DC values wrap through the int16 range
    y = cc.dc_climb()[0]
    assert y[:, 0].min() < -30000 and y[:, 0].max() > 30000


def test_block_lengths_and_stuffing_extremes(po):
    """Blocks of exactly 511..545 and 1658 bits at chunk lanes 0/15/31; a scan of mostly 0xFF."""
    case, want = cc.block_lengths()
    got, ref = encode_both(po, case, 0, False)
    assert got == ref
    d = assert_decodes_to(ref, case, block_starts=True)
    ends = np.append(d.block_start[1:], d.interval_end[-1])
    lens = ends - d.block_start
    assert {i: int(lens[i]) for i in want} == want
    case = cc.stuffing_gray()
    got, ref = encode_both(po, case, 0, False)
    assert got == ref
    scan = jd.scan_bytes(ref)
    share = scan.count(b"\xff\x00") / len(scan)
    assert share > 0.30, share
    assert_decodes_to(ref, case)


def straddling(po, nblocks, border, mcus_x=8):
    """The first phase whose border byte (holding the last bits of block border-1 and the first of
    block `border`) is 0xFF: (case, its JPEG)."""
    for phase in range(1, 8):
        case = cc.straddle(nblocks, border, phase, mcus_x)
        jpg = po.jpeg_encode_from_coefficients(*case[:6], 80, case[6], 0)
        d = assert_decodes_to(jpg, case, block_starts=True)
        s = int(d.block_start[border])
        if s % 8 and d.unstuffed[s // 8] == 0xFF:
            return case, jpg
    raise AssertionError("no phase puts a 0xFF byte on the border")


def test_ff_bytes_across_chunk_and_segment_borders(po):
    for nblocks, border in ((64, 32), (96, 48)):      # chunk border; the border of 2 segments of 48 MCUs
        case, ref = straddling(po, nblocks, border)
        assert encode_both(po, case, 0, False)[0] == ref


def band_border_straddle(po):
    """A 64x96 gray frame in two bands whose border byte is 0xFF: (case, its JPEG, the two band slices)."""
    case, ref = straddling(po, 96, 48)
    bands = band_slices(case, 2)
    assert len(bands[0][1]) == 48, "band 0 must end where the 0xFF byte straddles"
    return case, ref, bands


def test_ff_byte_across_a_band_border_host_twins(po):
    """The byte holding the last bits of band 0 and the first of band 1 is 0xFF: the host band twins
    (histogram, raw string, splice with the inherited bits) must stuff it exactly as one coder would."""
    case, ref, bands = band_border_straddle(po)
    y, cb, cr, w, h, ct, ss = case
    coders = [parallel.HostBandCoder(by, bcb, bcr, w, b.px_row1 - b.px_row0, ct, ss) for b, by, bcb, bcr in bands]
    for opt in (False, True):
        parts, hist = parallel.tiled_scan_parts_local(coders, opt)
        got = parallel.assemble_tiled(parts, hist, w, h, ct, 80, ss)
        assert got == po.jpeg_encode_from_coefficients(y, cb, cr, w, h, ct, 80, ss, 0, opt), opt
    assert parallel.assemble_tiled(parallel.tiled_scan_parts_local(coders)[0], None, w, h, ct, 80, ss) == ref


def test_restart_padding_completes_ff_bytes(po):
    case, ri = cc.restart_padding()
    got, ref = encode_both(po, case, ri, False)
    assert got == ref
    d = assert_decodes_to(ref, case)
    seen = set()
    for e in d.interval_end:
        pad = -e % 8
        if pad and d.unstuffed[e // 8] | ((1 << pad) - 1) == 0xFF:
            seen.add(pad)
    assert seen == set(range(1, 8))
    assert b"\xff\x00\xff\xd0" in jd.scan_bytes(ref)       # a padded 0xFF is stuffed before the marker


@pytest.mark.parametrize("name", sorted(cc.MATRIX))
@pytest.mark.parametrize("ct,ss", cc.geometries())
def test_host_coder_on_the_corpus(po, name, ct, ss):
    case = cc.MATRIX[name](ct, ss)
    for ri in restart_intervals(case):
        if ri and name in cc.NO_RESTART:
            continue
        for opt in (False, True):
            got, ref = encode_both(po, case, ri, opt)
            assert got == ref, (ri, opt)
            assert_decodes_to(ref, case)


def band_slices(case, world):
    y, cb, cr, w, h, ct, ss = case
    ypm = 4 if (ct == 2 and ss == 1) else 1
    mx = (w + (15 if ypm == 4 else 7)) // (16 if ypm == 4 else 8)
    out = []
    for b in parallel.plan_bands(w, h, world, gray=ct == 0, s420=ss == 1):
        m0, m1 = b.mcu_row0 * mx, b.mcu_row1 * mx
        out.append((b, y[m0 * ypm:m1 * ypm], cb[m0:m1], cr[m0:m1]))
    return out


@pytest.mark.parametrize("name,ct,ss,world", [("dc_chains", 2, 1, 3), ("symbol_sweep", 2, 0, 2),
                                              ("dc_climb", 0, 0, 4)])
def test_host_band_twins_on_the_corpus(po, name, ct, ss, world):
    """pixo_b200_jpeg_band_{histogram,entropy,splice} over bands of a constructed frame: the summed
    histograms and the assembled file equal the oracle's whole-frame ones."""
    case = cc.MATRIX[name](ct, ss)
    y, cb, cr, w, h = case[:5]
    coders = [parallel.HostBandCoder(by, bcb, bcr, w, max(b.px_row1 - b.px_row0, 1), ct, ss)
              for b, by, bcb, bcr in band_slices(case, world)]
    for opt in (False, True):
        parts, hist = parallel.tiled_scan_parts_local(coders, opt)
        if opt:
            assert np.array_equal(hist, po.jpeg_histograms(y, cb, cr, w, h, ct, ss))
        got = parallel.assemble_tiled(parts, hist, w, h, ct, 80, ss)
        assert got == po.jpeg_encode_from_coefficients(y, cb, cr, w, h, ct, 80, ss, 0, opt), opt
