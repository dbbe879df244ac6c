"""pixo's lossy PNG path (QuantizationMode Auto / Force, src/png/mod.rs:469-511,1505-1902) restated in
oracle/png_quantize.py and oracle/png_quantize.c, pinned to real pixo output: tests/golden/quantize/
(pixo's wasm build with lossy = 1, oracle/wasm_ref/gen_golden_quantize.py).  CPU only."""
import hashlib
import os

import numpy as np
import pytest

from oracle import png_quantize as pq
from oracle import png_reduce as pr
from quantize_inputs import GOLD, load_manifest, make_quantize_input, png_parts
from reduce_inputs import PNG_STRATEGY

MANIFEST = load_manifest()


def quantize_case_input(c):
    img = make_quantize_input(c["kind"], c["w"], c["h"], (1, 2, 3, 4)[c["ct"]], c["seed"], c["n"])
    assert hashlib.sha256(img.tobytes()).hexdigest() == c["input_sha256"], "input generator drifted"
    return img


def fixture_parts(c):
    return png_parts(open(os.path.join(GOLD, c["file"]), "rb").read())


def fixture_palette(parts):
    """The RGBA palette a quantised fixture carries: PLTE, alphas from tRNS, 255 past its end."""
    rgb = np.frombuffer(parts["PLTE"], np.uint8).reshape(-1, 3)
    a = np.full(len(rgb), 255, np.uint8)
    if parts["tRNS"]:
        t = np.frombuffer(parts["tRNS"], np.uint8)
        a[:len(t)] = t
    return np.concatenate([rgb, a[:, None]], 1)


def oracle_case(po, img, c, palette=None):
    """What encode_into(lossy = 1) hands DEFLATE: ('indexed', palette, filtered) or ('lossless', ...)."""
    w, h, ct = c["w"], c["h"], c["ct"]
    if not pq.should_quantize(img, ct, "auto", 256):
        red = pr.reduce(img, w, h, ct, c["preset"] in (1, 2), c["preset"] in (1, 2))
        f = po.apply_filters(pr.filter_input(red, c["preset"] in (1, 2)), w, h, red.bytes_per_pixel,
                             PNG_STRATEGY[c["preset"]], row_bytes=red.row_bytes, parallel_feature=False)
        return "lossless", red, f
    pal, idx = pq.quantize(img, w, h, ct, 256, True, palette)
    f = po.apply_filters(idx, w, h, 1, pq.indexed_strategy(PNG_STRATEGY[c["preset"]]), parallel_feature=False)
    return "indexed", pal, f


def test_generators_match_manifest():
    for c in MANIFEST["png"]:
        quantize_case_input(c)


def test_manifest_covers_the_paths():
    """Quantised fixtures with and without tRNS, truncation cases, and inputs that stay lossless."""
    kinds = set()
    for c in MANIFEST["png"]:
        p = fixture_parts(c)
        img = quantize_case_input(c)
        quantised = pq.should_quantize(img, c["ct"], "auto", 256)
        assert (p["ihdr"][3] == 3 and p["ihdr"][2] == 8) or not quantised
        if quantised:
            keys, _ = pq.histogram(img, c["ct"])
            kinds.add("trunc" if len(keys) > 8192 else "early" if len(keys) <= 256 else
                      "trns" if p["tRNS"] else "opaque")
        else:
            kinds.add("lossless")
    assert kinds == {"trunc", "early", "trns", "opaque", "lossless"}


@pytest.mark.parametrize("c", MANIFEST["png"], ids=lambda c: c["file"])
def test_oracle_reproduces_pixo(po, c):
    img = quantize_case_input(c)
    parts = fixture_parts(c)
    given = None
    if c["kind"] == "trunc":
        with pytest.raises(pq.TruncationCase):
            pq.quantize(img, c["w"], c["h"], c["ct"], 256, True)
        given = fixture_palette(parts)
    path, pal, f = oracle_case(po, img, c, given)
    assert parts["ihdr"][:2] == (c["w"], c["h"])
    if path == "indexed":
        assert (parts["ihdr"][2], parts["ihdr"][3]) == (8, 3)
        assert parts["PLTE"] == pal[:, :3].tobytes()
        assert parts["tRNS"] == pq.trimmed_trns(pal)
    else:
        red = pal
        assert (parts["ihdr"][2], parts["ihdr"][3]) == (red.bit_depth, red.color_type_byte)
    assert bytes(f) == parts["raw"]
    assert po.adler32(f) == parts["adler"]


# ---- the reference's own unit tests of this path ------------------------------------------------------
def test_trim_transparency():
    """maybe_trim_transparency: absent when all opaque, cut after the last translucent entry."""
    p = np.array([[0, 0, 0, 255], [1, 1, 1, 0], [2, 2, 2, 255]], np.uint8)
    assert pq.trimmed_trns(p) == bytes([255, 0])
    assert pq.trimmed_trns(p[[0, 2]]) is None
    p[2, 3] = 7
    assert pq.trimmed_trns(p) == bytes([255, 0, 7])


def test_perceptual_distance():
    """perceptual_distance_sq: zero on equal colours, green weighs more than blue, alpha unweighted."""
    c = np.array([[100, 100, 100, 255]], np.uint8)
    d = pq.distances(c, np.array([[100, 100, 100, 255], [100, 110, 100, 255], [100, 100, 110, 255],
                                  [100, 100, 100, 245]], np.uint8))[0]
    assert d[0] == 0 and d[1] > d[2] and d[3] == 100


def test_few_colours_keep_their_palette():
    """Force on an image with <= max_colors colours: the key-ordered colours, exact indices, no dither
    (quantize_image's early out ignores dithering)."""
    cols = np.array([[200, 0, 0], [0, 200, 0], [0, 0, 200], [9, 9, 9]], np.uint8)
    idx = np.arange(64) % 4
    img = cols[idx].reshape(-1)
    pal, got = pq.quantize(img, 8, 8, 2, 256, True)
    order = np.argsort([(int(c[0]) << 16) | (int(c[1]) << 8) | int(c[2]) for c in cols])
    assert np.array_equal(pal[:, :3], cols[order]) and (pal[:, 3] == 255).all()
    assert np.array_equal(pal[got, :3], img.reshape(-1, 3))


def test_max_colors_bounds_the_palette():
    img = make_quantize_input("grad", 64, 48, 3, 1)
    for m in (0, 1, 2, 16, 255, 256, 300):
        pal, idx = pq.quantize(img, 64, 48, 2, m, True)
        assert 1 <= len(pal) <= max(min(m, 256), 1) and idx.max() < len(pal)


def test_auto_decision_thresholds():
    """should_quantize_auto: more than max_colors, at most 32 x max_colors distinct sampled colours."""
    for n, want in ((256, False), (257, True), (8192, True), (8193, False)):
        img = make_quantize_input("pal", 128, 128, 3, 3, n)
        assert pq.should_quantize(img, 2, "auto", 256) == want
    gray = make_quantize_input("gray", 20, 20, 1, 1)
    assert not pq.should_quantize(gray, 0, "force", 256)
    assert pq.should_quantize(make_quantize_input("pal", 8, 8, 3, 1, 3), 2, "force", 256)
    assert not pq.should_quantize(make_quantize_input("pal", 64, 64, 3, 1, 300), 2, "off", 256)


# ---- the kernels' integer dither step ------------------------------------------------------------------
def test_sixteenths_equal_pixo_f32_step():
    """clamp(16 v + E16, 0, 4080) >> 4 equals (v as f32 + E16 / 16).clamp(0, 255) as u8 for every v and
    every reachable E16, with E16 / 16 formed as pixo forms it: a sum of er * k / 16 terms."""
    v = np.arange(256, dtype=np.int64)[:, None]
    e16 = np.arange(-4080, 4081, dtype=np.int64)[None, :]
    want = np.clip(v.astype(np.float32) + (e16.astype(np.float32) / np.float32(16)), 0, 255).astype(np.uint8)
    got = (np.clip(16 * v + e16, 0, 4080) >> 4).astype(np.uint8)
    assert np.array_equal(got, want)
    # the f32 sums of the four terms are exact: any order gives the same value
    rng = np.random.default_rng(0)
    er = rng.integers(-255, 256, (100000, 4)).astype(np.float32)
    k = np.array([7, 3, 5, 1], np.float32)
    terms = er * k / np.float32(16)
    s1 = ((terms[:, 0] + terms[:, 1]) + terms[:, 2]) + terms[:, 3]
    s2 = ((terms[:, 3] + terms[:, 2]) + terms[:, 1]) + terms[:, 0]
    assert np.array_equal(s1, s2) and np.array_equal(s1 * 16, (er * k).sum(1))


# ---- options -------------------------------------------------------------------------------------------
def test_options_mapping():
    from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode
    for preset in (0, 1, 2):
        o = PngOptions.from_preset_with_lossless(10, 20, preset, False)
        base = PngOptions.from_preset(10, 20, preset)
        assert (o.quantization_mode, o.max_colors, o.dithering) == (QuantizationMode.Auto, 256, True)
        assert (o.filter_strategy, o.optimize_alpha, o.reduce_color_type, o.reduce_palette) == \
            (base.filter_strategy, base.optimize_alpha, base.reduce_color_type, base.reduce_palette)
        ll = PngOptions.from_preset_with_lossless(10, 20, preset, True)
        assert ll.quantization_mode == QuantizationMode.Off and ll.strategy_word() == base.strategy_word()
    o = PngOptions(4, 4, 3, FilterStrategy.Paeth, quantization_mode=QuantizationMode.Force, dithering=True)
    assert o.strategy_word() == 4 | 0x1000 | 0x2000
    assert PngOptions(4, 4).strategy_word() == int(FilterStrategy.Adaptive)
    assert [pq.indexed_strategy(s) for s in range(9)] == [0, 1, 2, 3, 4, 0, 0, 0, 0]
