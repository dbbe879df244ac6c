"""pixo's lossless colour-type / palette reduction (maybe_reduce_color_type, src/png/mod.rs:683-1147)
restated in oracle/png_reduce.py, pinned to real pixo output: tests/golden/reduce/ (presets 1 and 2 of
pixo's wasm build, oracle/wasm_ref/gen_golden_reduce.py) and the tiny fixtures of tests/golden/ that
pixo reduced.  CPU only."""
import hashlib
import os

import numpy as np
import pytest

from oracle import png_reduce as pr
from reduce_inputs import GOLD, PNG_STRATEGY, load_manifest, make_reduce_input, png_parts, skipped_golden_cases
from golden_inputs import make_input

MANIFEST = load_manifest()
SKIPPED = skipped_golden_cases()


def reduce_case_input(c):
    img = make_reduce_input(c["kind"], c["w"], c["h"], (1, 2, 3, 4)[c["ct"]], c["seed"], c["n"])
    assert hashlib.sha256(img.tobytes()).hexdigest() == c["input_sha256"], "input generator drifted"
    return img


def golden_case_input(c):
    img = make_input(c["kind"], c["w"], c["h"], (1, 2, 3, 4)[c["ct"]], c["seed"])
    assert hashlib.sha256(img.tobytes()).hexdigest() == c["input_sha256"]
    return img


def expect_matches(parts, red, filtered, adler, c):
    """`red` (a ReducedImage-like description), its filtered stream and Adler-32 against a pixo PNG."""
    ihdr = parts["ihdr"]
    assert ihdr[:2] == (c["w"], c["h"])
    assert (ihdr[2], ihdr[3]) == (red.bit_depth, red.color_type_byte)
    pal = red.palette
    if pal is None:
        assert parts["PLTE"] is None and parts["tRNS"] is None
    else:
        assert parts["PLTE"] == pal[:, :3].tobytes()
        want_trns = pal[:, 3].tobytes() if (pal[:, 3] != 255).any() else None
        assert parts["tRNS"] == want_trns
    assert bytes(filtered) == parts["raw"]
    assert adler == parts["adler"]


def oracle_stream(po, img, c):
    red = pr.reduce(img, c["w"], c["h"], c["ct"], c["preset"] in (1, 2), c["preset"] in (1, 2))
    src = pr.filter_input(red, c["preset"] in (1, 2))
    f = po.apply_filters(src, c["w"], c["h"], red.bytes_per_pixel, PNG_STRATEGY[c["preset"]],
                         row_bytes=red.row_bytes, parallel_feature=False)
    return red, f, po.adler32(f)


def test_manifest_covers_the_reduction_branches():
    """Every outcome of maybe_reduce_color_type appears among the fixtures."""
    seen = set()
    for c in MANIFEST["png"]:
        ihdr = png_parts(open(os.path.join(GOLD, "reduce", c["file"]), "rb").read())["ihdr"]
        seen.add((ihdr[2], ihdr[3]))
    assert {(1, 3), (2, 3), (4, 3), (8, 3), (8, 2), (8, 4), (8, 6), (8, 0)} <= seen
    assert len(SKIPPED) == 8 and {c["file"] for c in SKIPPED} == {
        "p046.png", "p047.png", "p049.png", "p050.png", "p052.png", "p053.png", "p055.png", "p056.png"}


def test_generators_match_manifest():
    for c in MANIFEST["png"]:
        reduce_case_input(c)


@pytest.mark.parametrize("c", MANIFEST["png"], ids=lambda c: c["file"])
def test_oracle_reproduces_pixo_reduction(po, c):
    img = reduce_case_input(c)
    parts = png_parts(open(os.path.join(GOLD, "reduce", c["file"]), "rb").read())
    red, f, ad = oracle_stream(po, img, c)
    expect_matches(parts, red, f, ad, c)


@pytest.mark.parametrize("c", SKIPPED, ids=lambda c: c["file"])
def test_oracle_reproduces_reduced_golden_fixtures(po, c):
    img = golden_case_input(c)
    parts = png_parts(open(os.path.join(GOLD, c["file"]), "rb").read())
    red, f, ad = oracle_stream(po, img, c)
    expect_matches(parts, red, f, ad, c)


def test_most_popular_rotation_takes_both_branches():
    """The fixtures reach apply_most_popular_first's rotate_left and reverse + rotate_right arms."""
    arms = set()
    for c in MANIFEST["png"]:
        if c["kind"] != "dom":
            continue
        img = reduce_case_input(c).reshape(-1, 3)
        keys = pr._keys(img, pr.RGB)
        uniq, inv = np.unique(keys, return_inverse=True)
        idx = inv.astype(np.uint8)
        m = pr.co_occurrence(idx, uniq.size, c["w"], c["h"])
        remap = pr.mzeng_reindex(uniq.size, pr.weighted_edges(m), m)
        counts = np.bincount(idx, minlength=256)
        top = max(range(len(remap)), key=lambda k: (counts[remap[k]], k))
        if counts[remap[top]] >= idx.size * 3 // 20:
            arms.add(top >= len(remap) // 2)
        else:
            arms.add("below")
    assert arms == {True, False, "below"}


# ---- the reference's own unit-test answers (src/png/mod.rs tests, src/png/bit_depth.rs) ----------------
def test_reduce_rgb_to_gray():
    r = pr.reduce(np.array([10, 10, 10, 50, 50, 50], np.uint8), 2, 1, pr.RGB, True, False)
    assert r.effective_color_type == pr.GRAY and r.data.tolist() == [10, 50]


def test_reduce_rgba_drop_alpha():
    r = pr.reduce(np.array([1, 2, 3, 255, 4, 5, 6, 255], np.uint8), 2, 1, pr.RGBA, True, False)
    assert r.effective_color_type == pr.RGB and r.data.tolist() == [1, 2, 3, 4, 5, 6]


def test_reduce_rgba_to_gray_alpha():
    r = pr.reduce(np.array([8, 8, 8, 10, 9, 9, 9, 0], np.uint8), 2, 1, pr.RGBA, True, False)
    assert r.effective_color_type == pr.GRAY_ALPHA and r.data.tolist() == [8, 10, 9, 0]


def test_palette_reduction_writes_plte():
    r = pr.reduce(np.array([255, 0, 0, 255, 0, 255, 0, 255], np.uint8), 2, 1, pr.RGBA, False, True)
    assert (r.color_type_byte, r.bit_depth) == (3, 1) and r.palette.shape == (2, 4) and r.trns is None


def test_gray_input_is_not_bit_reduced():
    r = pr.reduce(np.array([0, 1, 1, 0], np.uint8), 4, 1, pr.GRAY, True, True)
    assert (r.color_type_byte, r.bit_depth, r.row_bytes) == (0, 8, 4)


def test_bit_depth_boundaries():
    assert [pr.palette_bit_depth(n) for n in (0, 1, 2, 3, 4, 5, 16, 17, 256)] == [8, 1, 1, 2, 2, 4, 4, 8, 8]
    assert [pr.gray_bit_depth(v) for v in (0, 1, 2, 3, 4, 15, 16, 255)] == [1, 1, 2, 2, 4, 4, 8, 8]


def test_pack_rows_pads_each_row():
    v = np.array([1, 0, 1, 1, 0, 1, 1, 1, 1, 0, 1, 0, 1, 0, 1, 1, 1, 1], np.uint8)   # 9 x 2, 1 bit
    assert pr.pack_rows(v, 9, 1).tolist() == [0b10110111, 0b10000000, 0b01010111, 0b10000000]
    assert pr.pack_rows(np.array([3, 2, 1], np.uint8), 3, 2).tolist() == [0b11100100]
    assert pr.pack_rows(np.array([15, 1, 7], np.uint8), 3, 4).tolist() == [0xF1, 0x70]
