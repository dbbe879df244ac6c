"""The PNG decoder's oracle (oracle/png_decode.c) on the CPU: it agrees with the independent Python restatement
(png_decode_ref.py) on a constructed corpus, with zlib and PIL on every valid stream, and decodes the 225 real-pixo
PNG goldens to their generator inputs; pixo's refusals come with its messages, in its order."""
import glob
import hashlib
import io
import json
import os
import zlib

import numpy as np
import pytest

import png_decode_ref as ref
from oracle import png_decode as pd
from png_decode_corpus import bit_flips, chunk, corpus, ihdr, png, SIG, truncations

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CORPUS = corpus()


def same(data):
    got = pd.decode(data)
    k, msg, w, h, ct, px = ref.decode(data)
    assert (got.kind, got.message) == (k, msg)
    if k == pd.OK:
        assert (got.width, got.height, got.color_type) == (w, h, ct)
        assert got.pixels.tobytes() == px
    return got


@pytest.mark.parametrize("name", [n for n, _ in CORPUS])
def test_oracle_equals_restatement(name):
    same(dict(CORPUS)[name])


def _idat(data):
    pos, out = 8, b""
    while pos + 12 <= len(data):
        n = int.from_bytes(data[pos:pos + 4], "big")
        if data[pos + 4:pos + 8] == b"IDAT":
            out += data[pos + 8:pos + 8 + n]
        if data[pos + 4:pos + 8] == b"IEND":
            break
        pos += 12 + n
    return out


def test_valid_streams_equal_zlib_and_pil():
    from PIL import Image
    valid = compared = 0
    for name, f in CORPUS:
        got = pd.decode(f)
        if got.kind != pd.OK:
            continue
        valid += 1
        z = _idat(f)
        try:
            raw = zlib.decompress(z)
        except zlib.error:
            continue   # pixo accepts tables zlib refuses (incomplete codes); the restatement covers those
        kind, msg, out = pd.inflate_zlib(z, len(raw))
        assert kind == pd.OK and out == raw, name
        try:
            im = Image.open(io.BytesIO(f))
            im.load()
        except (OSError, SyntaxError):
            continue   # PIL refuses some of what pixo accepts (data past the final block, IDAT before IHDR)
        mode = ("L", "LA", "RGB", "RGBA")[got.color_type]
        if im.mode in ("I", "I;16", "I;16B") or (im.mode == "RGB" and f[24] == 16):
            continue   # PIL scales 16-bit samples; pixo keeps the high byte (checked by the restatement)
        if im.mode == "P" and got.color_type == 3 and not any(b != 255 for b in im.info.get("transparency", b"")):
            continue
        if im.mode == "P" and name.endswith(("short_plte", "empty_plte", "long_trns")):
            continue   # indices past PLTE: pixo gives black, PIL its own padding
        want = np.asarray(im.convert(mode)).reshape(-1)
        assert np.array_equal(want, got.pixels), name
        compared += 1
    assert valid > 100 and compared > 80


def _widen(px, ct):
    n = {0: 1, 1: 2, 2: 3, 3: 4}[ct]
    a = np.asarray(px, np.uint8).reshape(-1, n)
    if n == 1:
        return np.concatenate([a, a, a, np.full_like(a, 255)], 1)
    if n == 2:
        return np.concatenate([a[:, :1]] * 3 + [a[:, 1:]], 1)
    if n == 3:
        return np.concatenate([a, np.full_like(a[:, :1], 255)], 1)
    return a


def _goldens():
    """(file, generator input, input colour type, lossless) of the 225 real-pixo PNGs."""
    import golden_inputs
    import quantize_inputs
    import reduce_inputs
    out = []
    m = json.load(open(os.path.join(GOLD, "manifest.json")))
    for e in m["png"]:
        out.append((os.path.join(GOLD, e["file"]), golden_inputs.make_input(e["kind"], e["w"], e["h"],
                    (1, 2, 3, 4)[e["ct"]], e["seed"]), e, True))
    m = json.load(open(os.path.join(GOLD, "reduce", "manifest.json")))
    for e in m["png"]:
        out.append((os.path.join(GOLD, "reduce", e["file"]), reduce_inputs.make_reduce_input(
            e["kind"], e["w"], e["h"], (1, 2, 3, 4)[e["ct"]], e["seed"], e.get("n", 0)), e, True))
    m = json.load(open(os.path.join(GOLD, "quantize", "manifest.json")))
    for e in m["png"]:
        out.append((os.path.join(GOLD, "quantize", e["file"]), quantize_inputs.make_quantize_input(
            e["kind"], e["w"], e["h"], (1, 2, 3, 4)[e["ct"]], e["seed"], e.get("n", 0)), e, False))
    return out


def test_goldens_decode_to_their_inputs():
    gs = _goldens()
    assert len(gs) == 225
    lossless = 0
    for path, inp, e, is_lossless in gs:
        assert hashlib.sha256(np.ascontiguousarray(inp).tobytes()).hexdigest() == e["input_sha256"], path
        got = pd.decode(open(path, "rb").read())
        assert got.kind == pd.OK and (got.width, got.height) == (e["w"], e["h"]), path
        if is_lossless:
            lossless += 1
            a, b = _widen(got.pixels, got.color_type), _widen(inp, e["ct"])
            a[a[:, 3] == 0, :3] = b[b[:, 3] == 0, :3] = 0   # presets may clear the colour of transparent pixels
            assert np.array_equal(a, b), path
    assert lossless == 189


@pytest.mark.parametrize("k", range(0, 225, 9))
def test_truncations_and_flips_of_goldens(k):
    path = _goldens()[k][0]
    data = open(path, "rb").read()
    for f in truncations(data, max(1, len(data) // 9)) + bit_flips(data, 12, k):
        same(f)


# pixo's refusals, one case per precedence rule: (corpus name, kind, message)
REFUSALS = [
    ("not_png", pd.INVALID, "Decode error: not a PNG file"),
    ("truncated_chunk", pd.INVALID, "Decode error: truncated PNG chunk"),
    ("crc_unknown_chunk", pd.INVALID, "Decode error: CRC mismatch in abCd chunk"),
    ("crc_non_utf8_type", pd.INVALID, "Decode error: CRC mismatch in ��(A chunk"),
    ("crc_ihdr", pd.INVALID, "Decode error: CRC mismatch in IHDR chunk"),
    ("ihdr_length", pd.INVALID, "Decode error: invalid IHDR length"),
    ("ihdr_color_type", pd.INVALID, "Decode error: invalid PNG color type: 5"),
    ("plte_length", pd.INVALID, "Decode error: invalid PLTE length"),
    ("no_iend", pd.INVALID, "Decode error: missing IEND chunk"),
    ("no_iend_and_no_ihdr", pd.INVALID, "Decode error: missing IEND chunk"),
    ("no_ihdr", pd.INVALID, "Decode error: missing IHDR chunk"),
    ("zero_dims_and_adam7", pd.DIMENSIONS, "Invalid image dimensions: 0x0"),
    ("too_wide", pd.TOO_LARGE, "Image 16777217x2 exceeds maximum dimension 16777216"),
    ("compression_method", pd.INVALID, "Decode error: unsupported compression method"),
    ("filter_method", pd.INVALID, "Decode error: unsupported filter method"),
    ("adam7_and_bad_depth", pd.UNSUPPORTED, "Unsupported: Adam7 interlaced images not supported"),
    ("bad_depth_and_no_idat", pd.INVALID, "Decode error: invalid bit depth 3 for color type Grayscale"),
    ("no_idat", pd.INVALID, "Decode error: no IDAT data"),
    ("zlib_too_short", pd.INVALID, "Decode error: zlib stream too short"),
    ("zlib_bad_cm", pd.INVALID, "Decode error: invalid zlib compression method"),
    ("zlib_bad_fcheck", pd.INVALID, "Decode error: invalid zlib header checksum"),
    ("fdict", pd.UNSUPPORTED, "Unsupported: preset dictionary not supported"),
    ("idat_crc_before_truncation", pd.INVALID, "Decode error: CRC mismatch in IDAT chunk"),
    ("idat_crc_before_bad_plte", pd.INVALID, "Decode error: CRC mismatch in IDAT chunk"),
    ("idat_crc_before_missing_iend", pd.INVALID, "Decode error: CRC mismatch in IDAT chunk"),
    ("idat_crc_beats_zlib_header", pd.INVALID, "Decode error: CRC mismatch in IDAT chunk"),
    ("bad_plte_before_idat_crc", pd.INVALID, "Decode error: invalid PLTE length"),
    ("block_type_3", pd.INVALID, "Decode error: reserved block type"),
    ("len_nlen_mismatch", pd.INVALID, "Decode error: stored block LEN/NLEN mismatch"),
    ("stored_past_end", pd.INVALID, "Decode error: unexpected end of stream"),
    ("empty_distance_table", pd.INVALID, "Decode error: empty Huffman table"),
    ("incomplete_table", pd.INVALID, "Decode error: invalid Huffman code"),
    ("repeat_at_start", pd.INVALID, "Decode error: repeat code at start"),
    ("too_many_lengths_18", pd.INVALID, "Decode error: too many code lengths"),
    ("fixed_litlen_286", pd.INVALID, "Decode error: invalid literal/length code: 286"),
    ("dynamic_litlen_287", pd.INVALID, "Decode error: invalid literal/length code: 287"),
    ("fixed_dist_30", pd.INVALID, "Decode error: invalid distance code"),
    ("distance_too_far", pd.INVALID, "Decode error: distance too far back"),
    ("bad_adler", pd.INVALID, "Decode error: Adler32 mismatch: expected 236C0444, got 236C0445"),
    ("adler_beats_size", pd.INVALID, "Decode error: Adler32 mismatch: expected 005C0000, got 005C0016"),
    ("output_short", pd.INVALID, "Decode error: decompressed size mismatch: expected 24, got 23"),
    ("expansion_1000x", pd.INVALID, "Decode error: decompressed size mismatch: expected 24, got 24024"),
    ("size_beats_bad_filter", pd.INVALID, "Decode error: decompressed size mismatch: expected 8, got 9"),
    ("bad_filter_row1", pd.INVALID, "Decode error: invalid filter type: 7"),
    ("bad_filter_beats_missing_plte", pd.INVALID, "Decode error: invalid filter type: 7"),
    ("missing_plte", pd.INVALID, "Decode error: missing PLTE chunk"),
]


@pytest.mark.parametrize("name,kind,msg", REFUSALS)
def test_refusals(name, kind, msg):
    got = same(dict(CORPUS)[name])
    assert (got.kind, got.message) == (kind, msg)


@pytest.mark.parametrize("name", ["trailing_bytes_ignored", "bytes_after_iend_chunk", "two_ihdr",
                                  "idat_after_iend_ignored", "split_idat", "zero_length_idats", "unknown_chunks",
                                  "idat_before_ihdr", "trailing_after_final", "cinfo_unchecked", "stored_then_fixed",
                                  "final_symbol_near_end", "slow_path_codes", "fifteen_bit_codes", "gray_trns",
                                  "rgb_trns", "pal4_opaque_trns", "pal8_long_trns"])
def test_accepted_quirks(name):
    got = same(dict(CORPUS)[name])
    assert got.kind == pd.OK
    if name in ("gray_trns", "pal4_opaque_trns"):
        assert got.color_type in (0, 2)
    if name == "pal8_long_trns":   # one value != 255 anywhere in tRNS makes the frame RGBA
        assert got.color_type == 3


def test_info_reports_idat_crc_only_with_another_refusal():
    from pixo_b200 import _lib, decode
    try:
        _lib.load()
    except Exception:
        pytest.skip("library not built")
    assert decode.png_info(dict(CORPUS)["plain"]) == (3, 2, 0)
    assert decode.png_info(dict(CORPUS)["idat_crc"]) == (3, 2, 0)   # decided on the device
    for name in ("idat_crc_before_truncation", "idat_crc_beats_zlib_header", "missing_plte", "adam7"):
        want = pd.decode(dict(CORPUS)[name])
        if name == "missing_plte":
            assert decode.png_info(dict(CORPUS)[name])[2] == 2
            continue
        with pytest.raises(_lib.PixoError) as e:
            decode.png_info(dict(CORPUS)[name])
        assert want.message in str(e.value)


def sparse_files():
    """Mostly blank bilevel and palette images: their frames are many times their inflated rows, which a small
    stream can produce"""
    out = []
    for (w, h, depth, ct) in ((4096, 4096, 1, 0), (2000, 2000, 1, 3), (3000, 3000, 8, 3)):
        sb = (w * depth + 7) // 8
        pre = [chunk(b"PLTE", bytes(range(12)))] if ct == 3 else []
        out.append(png(w, h, depth, ct, zlib.compress(bytes(h * (1 + sb)), 9), pre=pre))
    return out


def test_producible_is_decided_on_the_inflated_rows():
    """A file is producible when its rows, not its frame, fit what its IDAT can produce: the sparse files decode and
    are producible although their frames are far larger than the bound; a header that claims more rows than the
    stream can produce is not producible and fails with the size error."""
    from pixo_b200 import _lib, decode
    try:
        _lib.load()
    except Exception:
        pytest.skip("library not built")
    for f in sparse_files():
        w, h, ct, ok = decode._png_info(f)
        got = pd.decode(f, pixels=False)
        assert ok and got.kind == pd.OK
        assert w * h * ct.bytes_per_pixel() > 1032 * (len(_idat(f)) - 6) + 65535
    w, h, ct, ok = decode._png_info(dict(CORPUS)["huge_claim_small_idat"])
    assert not ok and "decompressed size mismatch" in pd.decode(dict(CORPUS)["huge_claim_small_idat"]).message
