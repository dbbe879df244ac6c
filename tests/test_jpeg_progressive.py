"""CPU checks of the progressive references the GPU tests compare against: the C restatement
oracle/jpeg_progressive.c, the composed reference tests/progressive_ref.py and the scan restatement
tests/jpeg_progressive_scans.py - whole real-pixo max-preset files (tests/golden/trellis/ and
tests/golden/progressive/), agreement on constructed coefficient arrays and on an option matrix, and the
EOB-run lengths the progressive fixtures must hold."""
import json
import os

import numpy as np
import pytest

import jpeg_progressive_scans as ps
import progressive_ref as pr
from oracle import jpeg_progressive as jp
from oracle import jpeg_trellis as jt
from progressive_inputs import make_progressive_input
from trellis_inputs import make_trellis_input

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trellis")
GOLDEN_P = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "progressive")


@pytest.fixture(scope="module", autouse=True)
def oracles_built(po):
    jt.build()
    jp.build()


def _manifest(d=GOLDEN):
    with open(os.path.join(d, "manifest.json")) as f:
        return json.load(f)["jpeg"]


def _read(d, name):
    with open(os.path.join(d, name), "rb") as f:
        return f.read()


@pytest.mark.parametrize("e", _manifest(), ids=lambda e: e["file"])
def test_c_oracle_reproduces_pixo_max_files_whole(e):
    img = make_trellis_input(e["kind"], e["w"], e["h"], 1 if e["ct"] == 0 else 3, e["seed"])
    assert jp.encode(img, e["w"], e["h"], e["ct"], e["s420"], e["q"]) == _read(GOLDEN, e["file"])


@pytest.mark.parametrize("e", _manifest(GOLDEN_P), ids=lambda e: e["file"])
def test_c_oracle_reproduces_progressive_fixtures_whole(e):
    img = make_progressive_input(e)
    assert jp.encode(img, e["w"], e["h"], e["ct"], e["s420"], e["q"]) == _read(GOLDEN_P, e["file"])


def _y_ac_empty_runs(e):
    """Empty blocks before each non-empty block, and after the last, of the fixture's two Y AC scans."""
    y, _, _ = jt.jpeg_coefficients(make_progressive_input(e), e["w"], e["h"], e["ct"], e["s420"], e["q"])
    z = y[:, np.array(ps.ZIGZAG)]
    runs = set()
    for ss, se in ((1, 10), (11, 63)):
        ne = np.nonzero((z[:, ss:se + 1] != 0).any(1))[0]
        runs |= set((np.diff(ne) - 1).tolist()) | {int(ne[0]), int(len(y) - 1 - ne[-1])}
    return runs


def test_progressive_fixtures_cover_0x7fff_runs_and_all_modes():
    man = _manifest(GOLDEN_P)
    runs = set().union(*(_y_ac_empty_runs(e) for e in man))
    assert {32766, 32767, 32768} <= runs
    assert max(runs) + 1 >= 2 * 0x7FFF          # one run reaches 0x7FFF twice (init + empties)
    assert {(e["ct"], e["s420"]) for e in man} == {(0, 0), (2, 0), (2, 1)}
    # the files hold EOBRUN symbols their tables lack: pixo's (0, 4) fallback is exercised
    for e in man:
        t = ps.dht(_read(GOLDEN_P, e["file"]))
        assert 0xE0 not in t[(1, 0)][1]


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
def test_c_oracle_matches_composed_reference_on_options(ct, ss):
    for i, (w, h) in enumerate([(1, 1), (7, 9), (17, 15), (64, 33)]):
        for trellis in (True, False):
            for optimize in (True, False):
                for restart in (0, 5):
                    img = make_trellis_input(["noise", "smooth", "hifreq"][i % 3], w, h, 1 if ct == 0 else 3, i)
                    q = [1, 50, 80, 100][i]
                    assert jp.encode(img, w, h, ct, ss, q, restart, optimize, trellis) == \
                        pr.encode(img, w, h, ct, ss, q, restart, optimize, trellis), (w, h, trellis, optimize, restart)


def test_c_oracle_scans_match_restatement_on_constructed_arrays():
    from pixo_b200.jpeg import dht_array
    rng = np.random.default_rng(11)
    tables = [ps.dht(_read(GOLDEN, "t008.jpg")), ps.dht(_read(GOLDEN, "t000.jpg"))]
    n = 3000
    y = np.zeros((n, 64), np.int16)
    for i in range(n):
        k = i % 6
        if k == 0:
            y[i, ps.ZIGZAG[1 + int(rng.integers(16, 50))]] = int(rng.integers(1, 30))     # ZRL
        elif k == 1:
            y[i, 0] = int(rng.choice([-1, 1])) * int(rng.integers(1024, 16384))            # categories 11..15
            y[i, ps.ZIGZAG[int(rng.integers(1, 64))]] = int(rng.choice([-1, 1])) * int(rng.integers(1024, 16384))
        elif k == 2:
            y[i, ps.ZIGZAG[1:20]] = -1                                                      # 0xFF bytes
        elif k == 3:
            y[i] = rng.integers(-300, 300, 64)
    y[1500:1500 + 1400] = 0                                                                # a long EOB run
    cb = np.where(rng.random((700, 64)) < 0.05, rng.integers(-40, 40, (700, 64)), 0).astype(np.int16)
    cr = np.where(rng.random((700, 64)) < 0.02, rng.integers(-40, 40, (700, 64)), 0).astype(np.int16)
    for t in tables:
        assert jp.scans(y, cb, cr, dht_array(t)) == ps.encode_scans(y, cb, cr, t)
        assert jp.scans(y, cb[:0], cr[:0], dht_array(t)) == ps.encode_scans(y, cb[:0], cr[:0], t)


@pytest.mark.parametrize("e", _manifest(), ids=lambda e: e["file"])
def test_reference_reproduces_pixo_max_files_whole(e):
    img = make_trellis_input(e["kind"], e["w"], e["h"], 1 if e["ct"] == 0 else 3, e["seed"])
    with open(os.path.join(GOLDEN, e["file"]), "rb") as f:
        want = f.read()
    assert pr.encode(img, e["w"], e["h"], e["ct"], e["s420"], e["q"]) == want


def test_eob_run_quirks_on_constructed_blocks():
    """A non-empty block whose last non-zero lies below Se sets the EOB run to 1, later empty blocks add
    to it, and the scan's end flushes it with its extra bits."""
    tables = ps.dht(open(os.path.join(GOLDEN, "t000.jpg"), "rb").read())
    y = np.zeros((3, 64), np.int16)
    y[0, 1] = 5                      # ends below Se=10 -> run 1, then two empties -> run 3
    segs = ps.encode_scans(y, np.zeros((0, 64)), np.zeros((0, 64)), tables)
    w = ps.BitWriterMsb()
    code = ps.code_from_table(*tables[(1, 0)], 0x03)
    w.write(code[0], code[1]); w.write(5, 3)
    eob = ps.code_from_table(*tables[(1, 0)], 0x10)   # run 3: symbol 1 << 4, one extra bit
    w.write(*eob); w.write(1, 1)
    assert segs[3] == w.finish()
    assert segs[1] == segs[2] == b""
