"""pixo's resizers (src/resize.rs) restated in oracle/resize.c, pinned to real pixo output: tests/golden/resize/
(pixo's wasm build, resizeImage, via oracle/wasm_ref/gen_golden_resize.py), and the sinf that build runs
(tests/golden/resize/sinf.npy).  The library's Lanczos3 tables (pixo_b200_resize_weights, host only) are
compared with the oracle's bit for bit.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import resize as rz
from resize_inputs import make_resize_input

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resize")
MANIFEST = json.load(open(os.path.join(GOLD, "manifest.json")))
CASES = MANIFEST["resize"]

# (args, status): the wasm binding's enum checks first, then resize_impl's order
ERRORS = [
    ((4, 4, 2, 2, 4, 0), 7),          # unknown colour type
    ((4, 4, 2, 2, 3, 3), 7),          # unknown algorithm
    ((0, 0, 0, 0, 9, 9), 7),          # enums before dimensions
    ((0, 4, 2, 2, 3, 0), 2),          # zero source
    ((4, 0, 0, 2, 3, 1), 2),          # zero source before zero destination
    ((4, 4, 2, 0, 3, 2), 2),          # zero destination
    ((0, 4, (1 << 24) + 1, 2, 3, 0), 2),  # zero before too large
    ((4, 4, (1 << 24) + 1, 2, 3, 0), 3),  # too large (destination)
    (((1 << 24) + 1, 1, 2, 2, 0, 0), 3),  # too large (source) before the length check
    ((4, 4, 2, 2, 3, 1), 5),          # wrong data length
]


def case_input(c):
    img = make_resize_input(c)
    assert hashlib.sha256(img.tobytes()).hexdigest() == c["input_sha256"], "input generator drifted"
    return img


def fixture(c):
    return np.fromfile(os.path.join(GOLD, c["file"]), np.uint8)


def test_fixture_coverage():
    assert {(c["ct"], c["alg"]) for c in CASES} == {(ct, a) for ct in range(4) for a in range(3)}
    geo = {(c["sw"], c["sh"], c["dw"], c["dh"]) for c in CASES}
    assert any(s == d for s, d in [((g[0], g[1]), (g[2], g[3])) for g in geo])            # identity
    assert (1, 1) in {(g[0], g[1]) for g in geo} and (1, 1) in {(g[2], g[3]) for g in geo}
    assert any(g[0] == 1024 and g[2] == 3 for g in geo)
    lz = [fixture(c) for c in CASES if c["alg"] == 2 and c["kind"] == "edges"]
    assert any(f.min() == 0 and f.max() == 255 for f in lz)


@pytest.mark.parametrize("k", range(len(CASES)))
def test_oracle_reproduces_pixo(k):
    c = CASES[k]
    got = rz.resize(case_input(c), c["sw"], c["sh"], c["dw"], c["dh"], c["ct"], c["alg"])
    assert np.array_equal(got, fixture(c))


def test_oracle_sinf_equals_wasm_sinf():
    pairs = np.load(os.path.join(GOLD, "sinf.npy"))
    assert pairs.dtype == np.uint32 and len(pairs) == MANIFEST["sinf"]["pairs"]
    x = pairs[:, 0].view(np.float32)
    got = rz.sinf(x).view(np.uint32)
    bad = np.nonzero(got != pairs[:, 1])[0]
    assert bad.size == 0, [(hex(pairs[i, 0]), hex(pairs[i, 1]), hex(got[i])) for i in bad[:10]]
    # the fixture holds arguments where the wasm's sinf is not the correctly rounded sine
    assert MANIFEST["sinf"]["differ_from_double_sin"] > 0
    assert np.abs(x).max() <= np.float32(3 * np.pi)


@pytest.mark.parametrize("args,status", ERRORS)
def test_oracle_validation_order(args, status):
    sw, sh, dw, dh, ct, alg = args
    n = sw * sh * (ct + 1) if status != 5 and ct <= 3 and sw <= 1 << 24 else 3
    with pytest.raises(rz.OracleError) as e:
        rz.resize(np.zeros(max(n, 1) if status == 5 else n, np.uint8), sw, sh, dw, dh, ct, alg)
    assert e.value.code == status


def _same_tables(src, dst):
    from pixo_b200 import resize as pr
    got, want = pr.weights(src, dst), rz.contrib(src, dst)
    for g, w, name in zip(got, want, ("start", "count", "offset", "weights")):
        assert g.dtype == w.dtype and np.array_equal(g.view(np.uint8), w.view(np.uint8)), (src, dst, name)


def test_library_weights_small(lib):
    for src in range(1, 65):
        for dst in range(1, 65):
            _same_tables(src, dst)


@pytest.mark.parametrize("src,dst", [(1024, 3), (3, 1024), (16384, 3), (3, 16384), (16384, 12000),
                                     (12000, 16384), (3840, 1920), (2160, 1080), (3840, 7680), (1080, 360),
                                     (1000003, 999983), (1 << 24, 1), (1 << 24, 4099), (1, 1 << 20), (7, 1 << 22)])
def test_library_weights_large(lib, src, dst):
    _same_tables(src, dst)


def test_library_weights_errors(lib):
    import ctypes as C
    from pixo_b200 import _lib
    n = C.c_size_t()
    assert lib.pixo_b200_resize_weights(0, 4, None, None, None, None, 0, C.byref(n)) == _lib.ERR_INVALID_DIMENSIONS
    assert lib.pixo_b200_resize_weights(4, 0, None, None, None, None, 0, C.byref(n)) == _lib.ERR_INVALID_DIMENSIONS
    assert lib.pixo_b200_resize_weights((1 << 24) + 1, 4, None, None, None, None, 0, C.byref(n)) == \
        _lib.ERR_IMAGE_TOO_LARGE
    w = np.empty(4, np.float32)
    assert lib.pixo_b200_resize_weights(64, 64, None, None, None, w.ctypes.data, w.size, C.byref(n)) == \
        _lib.ERR_OUTPUT_TOO_SMALL
    assert n.value == rz.contrib(64, 64)[3].size


def test_options_builder_defaults():
    from pixo_b200 import ColorType
    from pixo_b200.resize import ResizeAlgorithm, ResizeOptions
    o = ResizeOptions.builder(100, 50).build()
    assert (o.dst_width, o.dst_height, o.color_type, o.algorithm) == (100, 50, ColorType.Rgba, ResizeAlgorithm.Bilinear)
    o = ResizeOptions.builder(100, 50).dst(7, 9).color_type(ColorType.Gray).algorithm(ResizeAlgorithm.Lanczos3).build()
    assert (o.dst_width, o.dst_height, o.color_type, o.algorithm) == (7, 9, ColorType.Gray, ResizeAlgorithm.Lanczos3)
