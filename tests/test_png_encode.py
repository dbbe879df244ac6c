"""Whole PNG files (pixo_b200_png_encode*), without a device: the oracle composition in png_encode_ref.py against
every preset-0/1 golden, the options, encode_capacity, the plain-C client, the refusals in pixo's order and the
staging of the host call."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import png_encode_ref as R
from conftest import ROOT

# The preset-0 goldens taller than 32 rows whose filter choice pixo's wasm build makes with sequential AdaptiveFast;
# the library follows pixo's default (parallel) build, so these files differ in their filtered stream alone.
SEQUENTIAL_ADAPTIVE_FAST = ["p000.png", "p006.png", "p009.png", "p012.png", "p021.png", "p036.png", "p039.png",
                            "p041.png", "p043.png", "p058.png", "p060.png", "p062.png"]


def test_oracle_rebuilds_every_golden_whole():
    """199 goldens (46 top-level, 119 reduce/, 34 quantize/ with the trunc palettes): pixels to file, byte for byte,
    with the sequential filter; the parallel filter changes exactly the 12 files listed."""
    jobs = R.golden_jobs()
    subs = [os.path.dirname(name) for name, *_ in jobs]
    assert (len(jobs), subs.count(""), subs.count("reduce"), subs.count("quantize")) == (199, 46, 119, 34)
    parallel_differs = []
    for name, preset, img, o, pal in jobs:
        want = R.golden_bytes(name)
        assert R.encode(img, o, pal, parallel_feature=False) == want, name
        if R.encode(img, o, pal, parallel_feature=True) != want:
            assert preset == 0 and o.height > 32, name
            parallel_differs.append(name)
    assert parallel_differs == SEQUENTIAL_ADAPTIVE_FAST


def test_options_from_preset():
    from pixo_b200.png import PngOptions
    for preset, level in ((0, 2), (1, 6), (2, 9)):
        o = PngOptions.from_preset(4, 4, preset)
        assert (o.compression_level, o.optimal_compression) == (level, preset == 2)
    assert (PngOptions().compression_level, PngOptions().optimal_compression) == (2, False)
    # the strategy words of the filter-stage calls are the parent's
    words = {(0, True): 0x7, (0, False): 0x2807, (1, True): 0x706, (1, False): 0x2F06, (2, True): 0x708,
             (2, False): 0x2F08}
    for (preset, lossless), w in words.items():
        assert PngOptions.from_preset_with_lossless(8, 8, preset, lossless).strategy_word() == w


def _capacity_images():
    """(name, img, color_type) over noise, gradients, 1x1, 1xN, Nx1 and palette images of every colour type."""
    rng = np.random.default_rng(5)
    out = []
    for ct in range(4):
        ch = ct + 1
        for w, h in ((1, 1), (1, 300), (300, 1), (37, 29), (64, 64)):
            out.append((f"noise{ct}_{w}x{h}", rng.integers(0, 256, (h, w, ch), dtype=np.uint8), ct))
            g = ((np.arange(w)[None, :, None] * 7 + np.arange(h)[:, None, None] * 3 + np.arange(ch)) % 256)
            out.append((f"grad{ct}_{w}x{h}", np.broadcast_to(g, (h, w, ch)).astype(np.uint8), ct))
            pal = rng.integers(0, 256, (256, ch), dtype=np.uint8)
            out.append((f"pal{ct}_{w}x{h}", pal[rng.integers(0, 256, (h, w))], ct))
    return out


def test_encode_capacity_bounds_every_file():
    from pixo_b200.png import PngOptions, encode_capacity
    from pixo_b200.color import ColorType
    for name, img, ct in _capacity_images():
        h, w = img.shape[:2]
        for preset in (0, 1):
            for lossless in (True, False):
                o = PngOptions.from_preset_with_lossless(w, h, preset, lossless)
                o.color_type = ColorType(ct)
                assert len(R.encode(img, o, parallel_feature=True)) <= encode_capacity(w, h, ct), (name, preset)
    # reached exactly: RGBA noise, stored, its filtered stream no multiple of 65 535 bytes
    img = np.random.default_rng(9).integers(0, 256, (64, 64, 4), dtype=np.uint8)
    o = PngOptions.from_preset(64, 64, 0)
    assert len(R.encode(img, o, parallel_feature=True)) == encode_capacity(64, 64, ColorType.Rgba)


def test_c_client_compiles_links_and_runs(lib, tmp_path):
    if not shutil.which("gcc"):
        pytest.skip("no C compiler")
    exe = str(tmp_path / "png_encode_client")
    pkg = os.path.join(ROOT, "pixo_b200")
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "c", "png_encode_client.c"), "-o", exe, "-L", pkg, "-lpixo_b200",
                    f"-Wl,-rpath,{pkg}"], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "png_encode_client ok" in out.stdout, (out.returncode, out.stdout, out.stderr)


def test_new_symbols_are_bound(lib):
    from pixo_b200 import _lib
    for name in ("pixo_b200_png_encode", "pixo_b200_png_encode_on_device"):
        assert name in _lib.SYMBOLS and hasattr(lib, name)


# ---- refusals in pixo's order, no device -----------------------------------------------------------------------
AUTO, FORCE, OPTIMAL = 0x800, 0x1000, 0x4000


def _host(lib, w=4, h=4, ct=3, word=7, level=6, data_len=None, max_colors=256):
    data = np.zeros(max(w * h * (ct + 1), 1), np.uint8)
    out, n = np.zeros(16, np.uint8), C.c_size_t()
    rc = lib.pixo_b200_png_encode(None, data.ctypes.data, w * h * (ct + 1) if data_len is None else data_len, w, h,
                                  ct, word, level, max_colors, None, 0, out.ctypes.data, out.size, C.byref(n))
    return rc, lib.pixo_b200_last_error(None).decode()


def _device(lib, word=7, level=6, d_data=0x10000, d_out=0x20000, n=2, stride=64, cap=4096):
    lens, st = (C.c_size_t * 2)(), (C.c_int32 * 2)()
    rc = lib.pixo_b200_png_encode_on_device(None, d_data, stride, n, 4, 4, 3, word, level, 256, None, None, d_out,
                                            cap, lens, st, None)
    return rc, lib.pixo_b200_last_error(None).decode()


def test_refusals_in_pixos_order(lib):
    from pixo_b200 import _lib as L
    cases = [
        (dict(level=0), L.ERR_INVALID_COMPRESSION_LEVEL, "Invalid compression level 0"),
        (dict(level=10), L.ERR_INVALID_COMPRESSION_LEVEL, "Invalid compression level 10"),
        (dict(level=0, w=0), L.ERR_INVALID_COMPRESSION_LEVEL, None),
        (dict(w=0), L.ERR_INVALID_DIMENSIONS, "Invalid image dimensions: 0x4"),
        (dict(h=0), L.ERR_INVALID_DIMENSIONS, "Invalid image dimensions: 4x0"),
        (dict(w=(1 << 24) + 1, h=1, data_len=5), L.ERR_IMAGE_TOO_LARGE, "exceed maximum"),
        (dict(ct=4), L.ERR_UNSUPPORTED_COLOR, "Unsupported color type: 4"),
        (dict(word=7 | AUTO | FORCE), L.ERR_INVALID_ARGUMENT, "exclusive"),
        (dict(data_len=63), L.ERR_INVALID_DATA_LENGTH, "expected 64 bytes, got 63"),
        # OPTIMAL_COMPRESSION after every one of pixo's checks
        (dict(word=7 | OPTIMAL, level=0), L.ERR_INVALID_COMPRESSION_LEVEL, None),
        (dict(word=7 | OPTIMAL, w=0), L.ERR_INVALID_DIMENSIONS, None),
        (dict(word=7 | OPTIMAL, w=(1 << 24) + 1, h=1, data_len=5), L.ERR_IMAGE_TOO_LARGE, None),
        (dict(word=7 | OPTIMAL | AUTO | FORCE), L.ERR_INVALID_ARGUMENT, "exclusive"),
        (dict(word=7 | OPTIMAL, max_colors=70000), L.ERR_INVALID_ARGUMENT, "u16"),
        (dict(word=7 | OPTIMAL, data_len=63), L.ERR_INVALID_DATA_LENGTH, None),
        (dict(word=0x708 | OPTIMAL), L.ERR_UNSUPPORTED, "optimal_compression (pixo's max preset) is not built"),
        # a valid call reaches the context last
        (dict(), L.ERR_INVALID_ARGUMENT, "ctx is null"),
    ]
    for kw, code, msg in cases:
        rc, err = _host(lib, **kw)
        assert rc == code, (kw, rc, err)
        assert msg is None or msg in err, (kw, err)


def test_device_call_refusals(lib):
    from pixo_b200 import _lib as L
    assert _device(lib, level=10)[0] == L.ERR_INVALID_COMPRESSION_LEVEL
    assert _device(lib, stride=63)[0] == L.ERR_INVALID_DATA_LENGTH
    assert _device(lib, word=7 | OPTIMAL, stride=63)[0] == L.ERR_INVALID_DATA_LENGTH
    rc, err = _device(lib, word=7 | OPTIMAL, d_out=0x10000 + 64)
    assert rc == L.ERR_UNSUPPORTED and "optimal_compression" in err
    for d_out in (0x10000 + 127, 0x10000 - 2 * 4096 + 1):   # the output slots overlap the frames from either side
        rc, err = _device(lib, d_out=d_out)
        assert rc == L.ERR_INVALID_ARGUMENT and "overlap" in err, d_out
    for d_out in (0x10000 + 128, 0x10000 - 2 * 4096):
        assert _device(lib, d_out=d_out) == (L.ERR_INVALID_ARGUMENT, "ctx is null"), d_out


def test_host_call_is_staged_through_the_helper():
    from test_host_staging import callers
    from test_launch_sites import sources
    helper = re.compile(r"\bstage_host_call\s*\(")
    calling = {fn for name, code in sources() for _, fn in callers(code, helper) if fn}
    assert "pixo_b200_png_encode" in calling
