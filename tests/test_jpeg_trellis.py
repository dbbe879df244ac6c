"""The C trellis oracle (oracle/jpeg_trellis.c) on the CPU: pinned to real pixo output (max-preset files
from pixo's wasm build, tests/golden/trellis/, re-encoded scan by scan from the oracle's coefficients by
tests/jpeg_progressive_scans.py), the exact-value facts of pixo's own trellis tests
(src/jpeg/trellis.rs:323-617), and agreement with an independent pure-Python restatement
(tests/trellis_ref.py) on constructed blocks at several lambdas."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import jpeg_trellis as jt
import jpeg_progressive_scans as ps
import trellis_ref as tr
from trellis_inputs import make_trellis_input

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trellis")
FIXTURES = json.load(open(os.path.join(GOLDEN, "manifest.json")))["jpeg"]
FIXTURE_IDS = [c["file"] for c in FIXTURES]


def fixture_case(c):
    """(input pixels, subsampling, the file's 7 scans' entropy-coded bytes, its Huffman tables)"""
    img = make_trellis_input(c["kind"], c["w"], c["h"], 1 if c["ct"] == 0 else 3, c["seed"])
    assert hashlib.sha256(img.tobytes()).hexdigest() == c["input_sha256"], "input generator drifted"
    data = open(os.path.join(GOLDEN, c["file"]), "rb").read()
    sc = ps.scans(data)
    assert [(s[0], s[1], s[2], s[3], s[4]) for s in sc] == [([k], a, b, 0, 0) for k, a, b in ps.SCRIPT]
    return img, (1 if c["ct"] == 2 and c["s420"] else 0), [s[5] for s in sc], ps.dht(data)


@pytest.mark.parametrize("c", FIXTURES, ids=FIXTURE_IDS)
def test_fixture_reencoded_from_oracle(c):
    """Every scan of a real max-preset file, byte for byte, from the oracle's trellis coefficients."""
    img, ss, want, tables = fixture_case(c)
    y, cb, cr = jt.jpeg_coefficients(img, c["w"], c["h"], c["ct"], ss, c["q"])
    got = ps.encode_scans(y, cb, cr, tables)
    assert [g == w_ for g, w_ in zip(got, want)] == [True] * 7


def test_plain_rounding_fails_most_fixtures(po):
    """quantize_block's coefficients do not reproduce most fixtures: the fixtures exercise the trellis."""
    fails = 0
    for c in FIXTURES:
        img, ss, want, tables = fixture_case(c)
        y, cb, cr = po.jpeg_coefficients(img, c["w"], c["h"], c["ct"], ss, c["q"])
        fails += ps.encode_scans(y, cb, cr, tables) != want
    assert fails > len(FIXTURES) // 2


def test_fixtures_cover_zrl_and_all_modes():
    """The fixtures hold runs of 16+ zeros before a non-zero inside an AC scan (ZRL states), and span
    4:2:0 / 4:4:4 / Gray, qualities 1..100 and the sizes up to ~512x384."""
    zrl = 0
    for c in FIXTURES:
        if c["kind"] != "hifreq" and c["q"] < 95:
            continue
        img, ss, _, _ = fixture_case(c)
        for comp, arr in enumerate(jt.jpeg_coefficients(img, c["w"], c["h"], c["ct"], ss, c["q"])):
            for b in arr:
                zz = b[ps.ZIGZAG]
                for lo, hi in ([(1, 10), (11, 63)] if comp == 0 else [(1, 63)]):
                    nz = np.nonzero(zz[lo:hi + 1])[0]
                    zrl += bool(nz.size) and (nz[0] >= 16 or (np.diff(nz) > 16).any())
    assert zrl > 50
    assert {(c["ct"], c["s420"]) for c in FIXTURES} == {(2, 1), (2, 0), (0, 0)}
    assert {c["q"] for c in FIXTURES} >= {1, 25, 50, 75, 80, 90, 95, 100}
    assert {(1, 1), (512, 384)} <= {(c["w"], c["h"]) for c in FIXTURES}


@pytest.fixture(scope="module", autouse=True)
def oracle_built():
    jt.build()


def _block(**kv):
    d = np.zeros(64, np.float32)
    for k, v in kv.items():
        d[int(k[1:])] = v
    return d


Q16 = np.full(64, 16.0, np.float32)
Q10 = np.full(64, 10.0, np.float32)


def test_kat_zeros():
    assert not jt.trellis_quantize(np.zeros(64), Q16).any()


@pytest.mark.parametrize("dc,q,lam,want", [(800.0, Q16, None, 50), (400.0, Q16, None, 25), (160.0, Q16, 10.0, 10),
                                           (200.0, Q16, None, 13), (-100.0, Q10, None, -10), (500.0, Q16, None, 31)])
def test_kat_dc(dc, q, lam, want):
    assert jt.trellis_quantize(_block(k0=dc), q, lam)[0] == want


def test_kat_sparsity_high_lambda():
    d = np.full(64, 8.0, np.float32)
    d[0] = 0.0
    r = jt.trellis_quantize(d, Q16, 2.0)
    assert (r[1:] == 0).sum() > 30


def test_kat_adaptive():
    d = _block(k0=800.0, k1=50.0)
    hi = jt.trellis_quantize(d, Q16, jt.trellis_lambda(95))
    lo = jt.trellis_quantize(d, Q16, jt.trellis_lambda(30))
    assert hi[0] == lo[0] and abs(hi[1]) <= 5 and abs(lo[1]) <= 5
    for q in (1, 50, 80, 100):
        assert jt.trellis_quantize(_block(k0=500.0), Q16, jt.trellis_lambda(q))[0] == 31


def test_kat_lambda_order():
    d = np.full(64, 10.0, np.float32)
    d[0] = 800.0
    lo = (jt.trellis_quantize(d, Q16, 0.1)[1:] != 0).sum()
    hi = (jt.trellis_quantize(d, Q16, 10.0)[1:] != 0).sum()
    assert hi <= lo


def test_kat_near_threshold_and_zigzag():
    r = jt.trellis_quantize(_block(k0=160.0, k1=8.1, k2=7.9), Q16)
    assert abs(r[1]) <= 1 and abs(r[2]) <= 1
    assert jt.trellis_quantize(_block(k0=200.0, k1=50.0, k8=40.0), Q10, 0.5)[0] == 20


def test_candidates_and_category():
    assert set(tr.candidates(5.3)) >= {0, 5, 6} and set(tr.candidates(-5.3)) >= {0, -5, -6}
    assert tr.candidates(0.1) == [0, 1] and tr.candidates(-0.1) == [0, -1] and tr.candidates(0.0) == [0]
    assert tr.candidates(5.0) == [0, 5, 6] and tr.candidates(-3.7) == [0, -4, -3, -5]
    assert tr.candidates(1.5) == [0, 1, 2] and tr.candidates(1.5001) == [0, 1, 2, 3]
    assert [tr.category(v) for v in (0, 1, -1, 2, 3, 127, -128, 32767, -32767, 16383, -16384)] == \
        [0, 1, 1, 2, 2, 7, 8, 15, 15, 14, 15]


def test_lambda_formula():
    assert [jt.trellis_lambda(q) for q in (100, 80, 79, 50, 49, 1)] == \
        [float(tr.adaptive_lambda(q)) for q in (100, 80, 79, 50, 49, 1)]
    assert jt.trellis_lambda(100) == 0.5 and jt.trellis_lambda(80) == 1.0 and jt.trellis_lambda(50) == float(np.float32(1.99))


@pytest.mark.parametrize("lam", [None] + list(tr.LAMBDAS[:2]) + list(tr.LAMBDAS[3:]) + [tr.adaptive_lambda(30)])
def test_oracle_matches_python_restatement(lam):
    d, q = tr.constructed_blocks(seed=2, n_random=120)
    for i in range(len(d)):
        assert np.array_equal(jt.trellis_quantize(d[i], q[i], lam), tr.trellis_quantize(d[i], q[i], lam)), i


def test_trellis_differs_from_rounding(po):
    """On real image blocks the trellis is not plain rounding (so the checks above can tell them apart)."""
    from golden_inputs import make_input
    img = make_input("noise", 64, 64, 3, 1)
    y, _, _ = jt.jpeg_coefficients(img, 64, 64, 2, 1, 80)
    py, _, _ = po.jpeg_coefficients(img, 64, 64, po.RGB, po.S420, 80)
    assert (y[:, 0] == py[:, 0]).all()          # DC is plain rounding in both
    assert (y != py).any(1).mean() > 0.1
