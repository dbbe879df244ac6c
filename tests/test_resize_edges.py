"""The resizer edge tests' references and inputs, on the CPU: tests/resize_ref.py's numpy Nearest and Bilinear
equal oracle/resize.c on every small geometry and on the exact-half inputs (where round-half-even would
not), the integer expectations of the exact halves equal the oracle, and the band model gives each scratch
cap case of tests/test_resize_edges_gpu.py the paths it claims.  CPU only."""
import numpy as np
import pytest

import resize_edge_inputs as ei
import resize_ref as rr
from oracle import resize as rz

SIDES = range(1, 49)


@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("alg", [0, 1])
@pytest.mark.parametrize("axis", ["x", "y"])
def test_restatement_equals_oracle_on_every_small_geometry(axis, alg, bpp):
    """Every (src, dst) pair in 1..48 on one axis, the other 7 -> 5 (the GPU sweep's geometries)."""
    for s in SIDES:
        img = ei.noise(*((s, 7) if axis == "x" else (7, s)), bpp, 100 * s + bpp)
        for d in SIDES:
            g = (s, 7, d, 5) if axis == "x" else (7, s, 5, d)
            assert np.array_equal(rr.resize(img, *g, bpp, alg), rz.resize(img, *g, bpp - 1, alg)), g


@pytest.mark.parametrize("alg", [0, 1])
def test_restatement_equals_oracle_on_random_geometries(alg):
    rng = np.random.default_rng(alg)
    for _ in range(200):
        sw, sh, dw, dh = (int(x) for x in rng.integers(1, 400, 4))
        bpp = int(rng.integers(1, 5))
        img = ei.noise(sw, sh, bpp, sw * sh + dw)
        assert np.array_equal(rr.resize(img, sw, sh, dw, dh, bpp, alg), rz.resize(img, sw, sh, dw, dh, bpp - 1, alg))


def test_round_half_away_from_zero():
    v = np.array([0.5, 1.5, 2.5, -0.5, -2.5, 0.49999997, 254.5, 255.49998, 8388607.5, -0.0], np.float32)
    assert rr.round_f32(v).tolist() == [1, 2, 3, -1, -3, 0, 255, 255, 8388608, 0]
    assert rr.round_f32(v, "even").tolist() == [0, 2, 2, -0.0, -2, 0, 254, 255, 8388608, 0]


@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("dst", [3, 5])
def test_bilinear_exact_halves(dst, bpp):
    """Both axes: the integer expectation equals the oracle and the restatement.  Round-half-even moves
    16 384 of the blends at 1/2 (a + b odd, half of them) and, for 2 -> 5, 8 192 each at 1/4 and 3/4."""
    ab = ei.pairs(bpp)
    rows = ab.shape[0]
    e = ei.bilinear_halves(ab[:, 0].reshape(-1), ab[:, 1].reshape(-1), dst).reshape(rows, bpp, dst)
    for img, geom, want in ((ab, (2, rows, dst, rows), e.transpose(0, 2, 1)),
                            (ab.transpose(1, 0, 2), (rows, 2, rows, dst), e.transpose(2, 0, 1))):
        img, want = np.ascontiguousarray(img).reshape(-1), np.ascontiguousarray(want).reshape(-1)
        assert np.array_equal(rz.resize(img, *geom, bpp - 1, 1), want), geom
        assert np.array_equal(rr.resize(img, *geom, bpp, 1), want), geom
        even = rr.resize(img, *geom, bpp, 1, half="even")
        assert int((even != want).sum()) == 16384 * (dst - 1) // 2, geom


@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("r", [2, 4, 6])
def test_nearest_exact_halves(r, bpp):
    """src = r dst: the integer index equals the oracle's; half-even picks another source pixel at every
    position for r = 2 and 6, and at none for r = 4 (r d + 1.5 is already the even neighbour's half)."""
    for d in (1, 7, 48, 1000):
        idx = ei.nearest_halves(r * d, d)
        assert np.array_equal(rr.nearest_index(np.arange(d), np.float32(r * d) / np.float32(d), r * d), idx)
        even = rr.nearest_index(np.arange(d), np.float32(r * d) / np.float32(d), r * d, half="even")
        assert int((even != idx).sum()) == (0 if r == 4 else d)
        for geom in ((r * d, 3, d, 3), (3, r * d, 3, d)):
            img = ei.noise(*geom[:2], bpp, r * d)
            a = img.reshape(geom[1], geom[0], bpp)
            want = (a[:, idx] if geom[2] == d else a[idx]).reshape(-1)
            assert np.array_equal(rz.resize(img, *geom, bpp - 1, 0), want), geom


# ---- the band model -----------------------------------------------------------------------------------
CAP_CASES = ei.cap_cases()


def covered(bands, dw, dh, start, count, bpp, cap):
    """Every destination pixel in exactly one band, every band's window holds its rows' taps and fits the
    cap (a one-column chunk excepted: the planner cannot go narrower)"""
    seen = np.zeros((dh, dw), np.int32)
    for y0, y1, rs, re, x0, cw in bands:
        seen[y0:y1, x0:x0 + cw] += 1
        assert (re - rs) * cw * bpp <= cap or cw == 1
        for y in range(y0, y1):
            if count[y]:
                assert rs <= start[y] and start[y] + count[y] <= re
    assert (seen == 1).all()


@pytest.mark.parametrize("case", CAP_CASES, ids=[c[0] for c in CAP_CASES])
def test_cap_case_takes_the_paths_it_claims(case):
    name, (sw, sh, dw, dh), bpp, n, cap, claims = case
    bands, per, launches = ei.plan(sw, sh, dw, dh, bpp, n, cap)
    got = ei.paths(bands, n, per, bpp, dw, cap)
    assert claims <= got, (name, sorted(claims - got))
    start, count = rz.contrib(sh, dh)[:2]
    covered(bands, dw, dh, start, count, bpp, cap)
    assert launches == -(-n // per) * sum(1 + (b[3] > b[2]) for b in bands)
    assert launches <= 2 * n * dw * dh


def test_cap_cases_cover_every_path():
    """Across the cases, every path for every byte count per pixel, and column chunks only on calls of
    several frames (each frame reruns every chunk through one intermediate)."""
    for bpp in range(1, 5):
        got = set()
        for name, (sw, sh, dw, dh), b, n, cap, _ in CAP_CASES:
            if b == bpp:
                bands, per, _ = ei.plan(sw, sh, dw, dh, bpp, n, cap)
                got |= ei.paths(bands, n, per, bpp, dw, cap)
        assert got == {"one-band", "bands", "exact", "overlap", "chunks", "ragged", "single-col", "passes"}, bpp
    assert all(n >= 2 for _, _, _, n, _, claims in CAP_CASES if "chunks" in claims)


def test_real_cap_plans():
    """No hook: 2 x 65 536 gray to 4 096 x 1 is one band of exactly 2^28 bytes; to 4 097 x 1 the one
    destination row is split into chunks of 4 096 and 1 columns."""
    assert ei.plan(2, 65536, 4096, 1, 1, 1, rr.SCRATCH) == ([(0, 1, 0, 65536, 0, 4096)], 1, 2)
    assert 65536 * 4096 == rr.SCRATCH
    assert ei.plan(2, 65536, 4097, 1, 1, 1, rr.SCRATCH) == \
        ([(0, 1, 0, 65536, 0, 4096), (0, 1, 0, 65536, 4096, 1)], 1, 4)
