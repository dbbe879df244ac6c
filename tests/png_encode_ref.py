"""pixo's png::encode_into at presets 0 and 1 (src/png/mod.rs:437-630, encode_indexed_into :1814-1886), pixels to
whole file, composed from the oracle's stages: oracle/png_quantize.py's decision and quantiser, oracle/png_reduce.py's
reduction, pyoracle.apply_filters, png_deflate.deflate_zlib and png_deflate.png_file.  Test infrastructure only.

encode(img, options, palette=None, parallel_feature=False) -> bytes
    options: anything with PngOptions' fields (width, height, color_type, filter_strategy, optimize_alpha,
    reduce_color_type, reduce_palette, quantization_mode, max_colors, dithering, compression_level).
    parallel_feature=False is pixo's wasm build (the goldens), True its default build (what the library follows).
"""
from __future__ import annotations

import numpy as np

from oracle import png_deflate as pd
from oracle import png_quantize as pq
from oracle import png_reduce as pr
from oracle import pyoracle as po

MODES = {0: "off", 1: "auto", 2: "force"}


def stages(img, o, palette=None, parallel_feature=False):
    """(bit_depth, color_type_byte, palette or None, tRNS or None, filtered stream) as encode_into hands them to
    DEFLATE and the container writers."""
    w, h, ct, strategy = int(o.width), int(o.height), int(o.color_type), int(o.filter_strategy)
    if pq.should_quantize(img, ct, MODES[int(o.quantization_mode)], min(int(o.max_colors), 256)):
        pal, idx = pq.quantize(img, w, h, ct, int(o.max_colors), bool(o.dithering), palette)
        f = po.apply_filters(idx, w, h, 1, pq.indexed_strategy(strategy), parallel_feature=parallel_feature)
        return 8, 3, pal, pq.trimmed_trns(pal), f
    red = pr.reduce(img, w, h, ct, bool(o.reduce_color_type), bool(o.reduce_palette))
    f = po.apply_filters(pr.filter_input(red, bool(o.optimize_alpha)), w, h, red.bytes_per_pixel, strategy,
                         row_bytes=red.row_bytes, parallel_feature=parallel_feature)
    return red.bit_depth, red.color_type_byte, red.palette, red.trns, f


def encode(img, o, palette=None, parallel_feature=False) -> bytes:
    depth, ctb, pal, trns, f = stages(img, o, palette, parallel_feature)
    z = pd.deflate_zlib(f, int(o.compression_level))
    return pd.png_file(int(o.width), int(o.height), depth, ctb, z, pal, trns)


def golden_jobs():
    """[(name, preset, img, options, palette or None)] for every preset-0/1 golden, its input regenerated as the
    per-stage golden tests do and its options PngOptions::from_preset (with_lossless(false) under quantize/); name is
    the file's path under tests/golden."""
    import json
    import os

    from golden_inputs import make_input
    from pixo_b200.color import ColorType
    from pixo_b200.png import PngOptions
    from test_png_quantize import fixture_palette, fixture_parts, quantize_case_input
    from test_png_reduce import reduce_case_input
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    jobs = []
    for sub in ("", "reduce", "quantize"):
        for c in json.load(open(os.path.join(gold, sub, "manifest.json")))["png"]:
            if c["preset"] not in (0, 1):
                continue
            w, h, ct, pal = c["w"], c["h"], c["ct"], None
            if sub == "quantize":
                img = quantize_case_input(c)
                o = PngOptions.from_preset_with_lossless(w, h, c["preset"], False)
                if c["kind"] == "trunc":
                    pal = fixture_palette(fixture_parts(c))
            else:
                img = reduce_case_input(c) if sub == "reduce" else make_input(c["kind"], w, h, (1, 2, 3, 4)[ct], c["seed"])
                o = PngOptions.from_preset(w, h, c["preset"])
            o.color_type = ColorType(ct)
            jobs.append((os.path.join(sub, c["file"]) if sub else c["file"], c["preset"], img, o, pal))
    return jobs


def golden_bytes(name: str) -> bytes:
    import os
    return open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name), "rb").read()
