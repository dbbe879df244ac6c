"""k_huff codes 96-block units (16 MCUs of 4:2:0, 32 of 4:4:4, 96 gray blocks) in three passes of one
component each.  Byte-identical to the oracle at the places the unit layout can get wrong: long blocks
at every pass and at lanes 0, 15, 16 and 31; 0xFF bytes across unit borders; MCU counts and restart
intervals around the unit size; dense units that do not fit one assembly window; segments and bands
that are not a whole number of units."""
import numpy as np
import pytest

import coef_corpus as cc
from pixo_b200 import ColorType, jpeg, parallel
from pixo_b200.jpeg import JpegOptions, Subsampling
from test_entropy_corpus import straddling
from test_entropy_corpus_gpu import device_coders, opts, oracle, upload

pytestmark = pytest.mark.gpu

GEOMETRIES = [(2, 1), (2, 0), (0, 0)]   # 4:2:0, 4:4:4, gray


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was silently finished by the host entropy coder"


def layout(ct, ss):
    """(Y blocks per MCU, MCUs per unit, MCU side in pixels)"""
    ypm = 4 if (ct == 2 and ss == 1) else 1
    bpm = ypm + (2 if ct == 2 else 0)
    return ypm, 96 // bpm, 16 if ypm == 4 else 8


def unit_slot(ct, ss, unit, p, lane):
    """(component, index in its array) of the block lane `lane` codes in pass p of unit `unit`"""
    ypm, umcus, _ = layout(ct, ss)
    m0 = unit * umcus
    if ypm == 4:
        if p < 2:
            return 0, m0 * 4 + 32 * p + lane
        return 1 + lane // 16, m0 + lane % 16
    if ct == 2:
        return p, m0 + lane
    return 0, m0 + 32 * p + lane


def random_frame(ct, ss, nmcus, seed, mcus_x=None, big=False):
    """nmcus MCUs of random sparse blocks (big: most coefficients set, up to +-1023), DC differences
    within +-2047, one MCU row unless mcus_x is given."""
    ypm, _, side = layout(ct, ss)
    rng = np.random.default_rng(seed)

    def arr(n):
        b = np.zeros((n, 64), np.int16)
        for i in range(n):
            k = rng.integers(40, 64) if big else rng.integers(0, 12)
            pos = rng.choice(np.arange(1, 64), size=k, replace=False)
            hi = 1024 if big else 200
            b[i, cc.ZIGZAG[pos]] = rng.integers(1, hi, size=k) * rng.choice([-1, 1], size=k)
            b[i, 0] = rng.integers(-1000, 1000)
        return b

    mx = mcus_x or nmcus
    assert nmcus % mx == 0
    y = arr(nmcus * ypm)
    z = np.zeros((0, 64), np.int16)
    cb, cr = (arr(nmcus), arr(nmcus)) if ct == 2 else (z, z)
    return y, cb, cr, mx * side, (nmcus // mx) * side, ct, ss


def check(po, gpu_ctx, case, ri=0):
    d = upload(case)
    for opt in (False, True):
        assert jpeg.entropy_encode_dev(*d, opts(case, ri, opt), ctx=gpu_ctx) == oracle(po, case, ri, opt), (ri, opt)


@pytest.mark.parametrize("ct,ss", GEOMETRIES)
def test_long_blocks_in_every_pass_and_at_lane_borders(po, gpu_ctx, ct, ss):
    """Blocks of 511-513 and 543-545 bits (around the 512-bit slot and its first spill word) and the
    1658-bit maximum (lengths on the luma tables; the chroma passes code the same blocks) in each of
    the three passes at lanes 0, 15, 16 and 31, between short blocks."""
    ypm, umcus, side = layout(ct, ss)
    nunits = len(cc.BLOCK_BITS) + 1
    nm = nunits * umcus
    fill = cc.block({1: 3, 5: -1})
    arrays = [[fill.copy() for _ in range(nm * ypm)]] + ([[fill.copy() for _ in range(nm)] for _ in range(2)]
                                                          if ct == 2 else [[], []])
    heavy = [[False] * len(a) for a in arrays]
    for u in range(nunits):
        for p in range(3):
            for j, lane in enumerate((0, 15, 16, 31)):
                comp, idx = unit_slot(ct, ss, u, p, lane)
                if u < len(cc.BLOCK_BITS):
                    arrays[comp][idx] = cc.exact_block(cc.BLOCK_BITS[(u + p + j) % len(cc.BLOCK_BITS)])
                else:
                    arrays[comp][idx] = cc.heavy_block(1 if lane % 2 else -1)
                    heavy[comp][idx] = True
    out = []
    for a, hv in zip(arrays, heavy):
        dc = 0
        for b, h in zip(a, hv):   # heavy blocks alternate their DC between 0 and 2047: category 11
            dc = (2047 if dc == 0 else 0) if h else dc
            b[0] = dc
        out.append(np.stack(a) if a else np.zeros((0, 64), np.int16))
    check(po, gpu_ctx, (out[0], out[1], out[2], umcus * side, nunits * side, ct, ss))


def test_ff_bytes_across_unit_borders(po, gpu_ctx):
    """Gray: the byte holding the last bits of block 95 (191) and the first of block 96 (192) is 0xFF."""
    for nblocks, border in ((192, 96), (288, 192)):
        case, ref = straddling(po, nblocks, border)
        d = upload(case)
        assert jpeg.entropy_encode_dev(*d, opts(case), ctx=gpu_ctx) == ref, border


@pytest.mark.parametrize("ct,ss", GEOMETRIES)
def test_mcu_counts_around_the_unit(po, gpu_ctx, ct, ss):
    """1, 15, 16, 17 MCUs, a multiple of 16 plus or minus one, and one unit plus or minus one MCU"""
    _, umcus, _ = layout(ct, ss)
    counts = sorted({1, 15, 16, 17, 47, 49, umcus - 1, umcus + 1, 2 * umcus + 1})
    for i, nm in enumerate(counts):
        check(po, gpu_ctx, random_frame(ct, ss, nm, seed=100 + i))


@pytest.mark.parametrize("ct,ss", GEOMETRIES)
def test_restart_intervals_around_the_unit(po, gpu_ctx, ct, ss):
    _, umcus, _ = layout(ct, ss)
    case = random_frame(ct, ss, 5 * 40, seed=7, mcus_x=40)
    for ri in sorted({1, 15, 16, 17, 33, umcus, umcus + 1}):
        check(po, gpu_ctx, case, ri)


@pytest.mark.parametrize("ct,ss", GEOMETRIES)
def test_dense_units_span_several_windows(po, gpu_ctx, ct, ss):
    """Units of up to ~19 KB (most coefficients set, up to +-1023): assembled and emitted over several
    windows, with and without restart intervals."""
    case = random_frame(ct, ss, 60, seed=11, mcus_x=20, big=True)
    for ri in (0, 17):
        check(po, gpu_ctx, case, ri)


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)])
def test_q100_noise(po, gpu_ctx, ct, ss):
    """The encode path (the transform's coefficient records) at q100 on noise: about 100 bytes per block."""
    w, h = 200, 136
    img = po.gen_noise(w, h, 3 if ct == 2 else 1, 5)
    o = JpegOptions(w, h, ColorType(ct), 100, Subsampling(ss))
    ref = po.jpeg_encode(img, w, h, po.RGB if ct == 2 else po.GRAY, 100, ss)
    assert jpeg.encode(img, o, ctx=gpu_ctx) == ref


@pytest.mark.parametrize("segments", ["3", "7"])
@pytest.mark.parametrize("ct,ss", GEOMETRIES)
def test_segments_of_partial_units(po, gpu_ctx, monkeypatch, ct, ss, segments):
    """Forced segments of 34 (15) MCUs: neither is a whole number of units."""
    monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
    check(po, gpu_ctx, random_frame(ct, ss, 100, seed=3, mcus_x=20))


@pytest.mark.parametrize("ct,ss,world", [(2, 1, 3), (2, 0, 2), (0, 0, 3)])
def test_bands_of_partial_units(po, gpu_ctx, ct, ss, world):
    """Bands of whole MCU rows of 20 MCUs: no band is a whole number of units."""
    case = random_frame(ct, ss, 9 * 20, seed=5, mcus_x=20)
    coders, _keep = device_coders(gpu_ctx, case, world)
    for opt in (False, True):
        assert parallel.encode_tiled_local(coders, *case[3:5], ct, 80, ss, opt) == oracle(po, case, 0, opt), opt
