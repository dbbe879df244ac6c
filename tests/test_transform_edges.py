"""The transform's constructed inputs sit where they are built to: tests/transform_ref.py equals the C oracle on every
quantiser case and on the colour conversion, every quantiser case is certified exactly and changes under the faults
it targets, and the walk shapes reach every branch of the persistent kernels' advance().  CPU only."""
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

import transform_inputs as I
import transform_ref as R

Q49 = float(np.nextafter(np.float32(0.5), np.float32(0)))   # 0.49999997, 0x3EFFFFFF
MODES = {"gray": (0, 0), "444": (2, 0), "420": (2, 1)}   # (colour type, subsampling) in the oracle's numbering


def test_restatement_equals_the_oracle_on_every_case_frame(po):
    for route in I.ROUTES:
        for fr in I.quantiser_frames(route):
            ct, ss = MODES[fr.mode]
            want = po.jpeg_coefficients(fr.pixels, fr.w, fr.h, ct, ss, lum_q=fr.lum_q, chr_q=fr.chr_q)
            for c in fr.cases:
                nb = 4 if fr.mode == "420" and c.comp == 0 else 1
                blk = want[c.comp][c.block * nb + c.sub]
                assert blk[c.pos] == c.want, (route, c)
                if c.comp == 0:   # the whole block through the restatement
                    assert R.quantize(np.float32([c.x]), [c.d])[0] == c.want
            # the whole frame through the restatement, block by block
            for comp, arr in enumerate(want[:1 if fr.mode == "gray" else 3]):
                blocks = _blocks(fr, comp)
                q = fr.lum_q if comp == 0 else fr.chr_q
                assert np.array_equal(R.quantize(R.dct_2d(blocks), q), arr), (route, comp)


def _blocks(fr, comp):
    """the frame's f32 blocks of one component, in the oracle's order (no edge replication: frames are whole MCUs)"""
    if fr.mode == "gray":
        return R.gray_block(fr.pixels.reshape(8, -1, 8).transpose(1, 0, 2).reshape(-1, 64))
    ycc = R.rgb_to_ycbcr(fr.pixels.reshape(fr.h, fr.w, 3)).astype(np.int32)[..., comp]
    if fr.mode == "444":
        return R.gray_block(ycc.reshape(8, -1, 8).transpose(1, 0, 2).reshape(-1, 64))
    if comp == 0:
        return R.gray_block(ycc.reshape(2, 8, -1, 2, 8).transpose(2, 0, 3, 1, 4).reshape(-1, 64))
    sums = ycc.reshape(8, 2, -1, 8, 2).sum(axis=(1, 4))           # [8, mcus, 8]
    return R.chroma_420_block(sums.transpose(1, 0, 2).reshape(-1, 64))


def test_every_case_is_certified_and_flips_its_mutants():
    for route in I.ROUTES:
        sc = 4 if route == "k1_c" else 1
        for fr in I.quantiser_frames(route):
            assert fr.lum_q.dtype == np.float32 and ((fr.lum_q >= 1) & (fr.lum_q <= 255)).all()
            for c in fr.cases:
                q = R.rn(Fraction(c.x) / c.d)
                assert float(q) == c.q == float(np.float32(c.x) / np.float32(c.d))
                t = np.float32(c.k + 0.5)   # |q| is k + 1/2, or the float32 just below or above it
                want_abs = {"tie": t, "below": np.nextafter(t, np.float32(0)), "above": np.nextafter(t, np.float32(9e9))}
                assert abs(q) == Fraction(float(want_abs[c.kind])) and (q < 0) == (c.x < 0), (route, c)
                assert c.want == R.pixo_quant(c.x, c.d) == R.kernel_quant(c.x, c.d, sc)
                for m in R.MUTANTS:
                    got = R.kernel_quant(c.x, c.d, sc, (m,))
                    assert (got != c.want) == (m in c.flips), (route, c, m)


def test_cases_cover_every_class_position_divisor_and_mutant():
    positions = set()
    for route in I.ROUTES:
        cases = [c for fr in I.quantiser_frames(route) for c in fr.cases]
        classes = {(c.x < 0, c.kind, min(c.k, I.LARGE_K)) for c in cases}
        for neg in (False, True):
            for kind in ("tie", "below", "above"):
                for k in (0, 1, 2, I.LARGE_K):
                    assert (neg, kind, k) in classes, (route, neg, kind, k)
        assert {1, 255} <= {c.d for c in cases}, route
        flips = Counter(m for c in cases for m in c.flips)
        for m in R.MUTANTS:
            if m != "no_fold" or route == "k1_c":
                assert flips[m] >= 2, (route, m, flips)
        assert any(c.q == Q49 for c in cases) and any(c.q == -Q49 for c in cases), route
        positions |= {c.pos for c in cases}
    assert positions == set(range(64))


def test_colour_conversion_equals_the_oracle(po):
    rng = np.random.default_rng(7)
    sample = rng.integers(0, 1 << 24, 20000)
    # every colour within 2 of a clamp boundary: Cb and Cr clamp only from above (256 -> 255; their least values
    # are 1), Y never
    c = np.arange(1 << 24)
    r, g, b = c >> 16, (c >> 8) & 255, c & 255
    cb = ((-43 * r - 85 * g + 128 * b + 128) >> 8) + 128
    cr = ((128 * r - 107 * g - 21 * b + 128) >> 8) + 128
    edge = np.flatnonzero((np.abs(cb - 255.5) <= 2) | (np.abs(cr - 255.5) <= 2))
    assert edge.size > 200
    ycc = R.all_colours_ycbcr()
    for v in np.concatenate([sample, edge]):
        assert tuple(ycc[v]) == po.rgb_to_ycbcr(int(v >> 16), int((v >> 8) & 255), int(v & 255)), hex(v)
    assert ycc[:, 1].min() == 1 and ycc[:, 2].min() == 1 and ycc[:, 1:].max() == 255


def test_flat_dc_tables_are_injective_and_equal_the_oracle(po):
    """All-ones tables: a flat block's DC is injective in its value and its AC is 0, for the 256 pixel values and
    for the 1021 quad sums of 4:2:0 chroma"""
    v = np.arange(256)
    dc = R.flat_dc(v)
    assert len(set(dc.tolist())) == 256
    sums = np.arange(1021)
    qdc = R.flat_dc(sums.astype(np.float32) / 4)
    assert len(set(qdc.tolist())) == 1021
    assert np.array_equal(qdc[::4], dc)
    ones = np.ones(64, np.float32)
    for s in list(range(0, 1021, 7)) + [4, 1020]:
        blk = np.full(64, s / 4 - 128, np.float32)
        want = po.quantize_block(po.dct_2d(blk), ones)
        assert want[0] == qdc[s] and not want[1:].any(), s
    for x in range(256):
        want = po.quantize_block(po.dct_2d(np.full(64, x - 128, np.float32)), ones)
        assert want[0] == dc[x] and not want[1:].any(), x


@pytest.mark.parametrize("mode", ["420", "444"])
def test_walk_shapes_reach_every_branch(mode):
    """For grids of 4 warps x {1, 2, 3} CTAs per SM x {114, 132} SMs, the walk shapes take the ux carry, the my
    wrap, both at once, and land exactly on units_x and on mcus_y; every unit is reached exactly once."""
    for sm in (114, 132):
        for bps in (1, 2, 3):
            stride = 4 * bps * sm
            seen = set()
            for w, h, n, ux, my in I.walk_shapes(mode):
                assert ux * my * n >= 3 * stride
                units, br = R.walk(ux, my, n, stride)
                u = np.arange(ux * my * n)
                assert np.array_equal(units, np.stack([u // (ux * my), u % (ux * my) // ux, u % ux], -1))
                seen |= br
            assert any(b[0] for b in seen) and any(b[1] for b in seen), (sm, bps)
            assert any(b[0] and b[1] for b in seen), (sm, bps)
            assert any(b[2] for b in seen) and any(b[3] for b in seen), (sm, bps)
            assert any(b[0] and not b[1] for b in seen) and any(b[1] and not b[0] for b in seen), (sm, bps)


def test_1080p_strides_never_carry_ux():
    """Why the walk shapes exist: 1080p 4:2:0 has 8 units per MCU row, and the H100's strides are multiples of 8"""
    for sm in (114, 132):
        _, br = R.walk(8, 68, 4, 4 * 2 * sm)
        assert not any(b[0] for b in br)
