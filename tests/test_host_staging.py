"""Source checks on pixo_b200/csrc: every host-buffer entry point stages its input and copies its results back
through api.cu's stage_host_call, so the staging copies (h2d_copy, d2h_copy_sync) and the drain-on-error guard
(DrainOnError) are used in that one function and by the host JPEG encode loops, which pipeline several groups of
frames on three streams.  Needs no GPU."""
import re

import pytest

from test_launch_sites import scopes, sources, strip

STAGING = re.compile(r"\b(?:h2d_copy|d2h_copy_sync)\s*\(|\bDrainOnError\b")
# the functions that may use them, by file: their own definitions and the helper; the host JPEG encode loops
# (encode_host, EncodeGroups::upload and the baseline and progressive group loops)
ALLOWED = {
    "api.cu": {"h2d_copy", "d2h_copy_sync", "stage_host_call"},
    "api_jpeg.cu": {"encode_host", "upload", "encode_baseline_groups", "encode_progressive_groups"},
}
DECLARED_IN = {"api.hpp", "api.cu"}   # where they may appear outside a function: declarations and the guard's type
ENTRY_POINTS = {"pixo_b200_jpeg_coefficients", "pixo_b200_png_filter", "pixo_b200_png_reduce_filter",
                "pixo_b200_png_quantize_filter", "pixo_b200_adler32", "pixo_b200_deflate_zlib", "pixo_b200_resize",
                "decode_one"}


def function_name(header: str) -> str:
    """The name of the function whose body a code block header opens ('' at namespace or class scope)."""
    m = re.search(r"(~?\w+)\s*\(", header)
    return m.group(1) if m else header


def callers(code: str, pattern):
    """(use, enclosing function name) for every match of pattern in code."""
    code = re.sub(r"(?m)^[ \t]*#[^\n]*", lambda m: " " * len(m.group(0)), code)   # preprocessor lines
    sc = scopes(code)
    return [(m.group(0), function_name(sc[m.start()][0]) if sc[m.start()] else "") for m in pattern.finditer(code)]


def findings(name: str, code: str):
    return [(name, use, fn) for use, fn in callers(code, STAGING)
            if not (fn in ALLOWED.get(name, ()) or (fn == "" and name in DECLARED_IN))]


def test_staging_goes_through_the_helper():
    bad = [f for name, code in sources() for f in findings(name, code)]
    assert not bad, "staging copies or DrainOnError outside stage_host_call and the encode loops:\n" + \
        "\n".join(map(str, bad))


def test_host_buffer_entry_points_call_the_helper():
    helper = re.compile(r"\bstage_host_call\s*\(")
    calling = {fn for name, code in sources() for _, fn in callers(code, helper) if fn}
    assert ENTRY_POINTS <= calling, sorted(ENTRY_POINTS - calling)


@pytest.mark.parametrize("name,src,want", [
    ("api_png.cu", "int f(X *ctx) { DrainOnError drain(ctx); return h2d_copy(ctx, a, b, n, s); }", 2),
    ("api_png.cu", "int g(X *ctx) { auto k = [&] { return d2h_copy_sync(ctx, a, b, n, s); }; return k(); }", 1),
    ("api_jpeg.cu", "struct EncodeGroups { int upload(uint32_t gi) const { return h2d_copy(c, a, b, n, s); } };", 0),
    ("api_png.cu", "struct EncodeGroups { int upload(uint32_t gi) const { return h2d_copy(c, a, b, n, s); } };", 1),
    ("api.hpp", "namespace pixo { int h2d_copy(X *ctx); struct DrainOnError { ~DrainOnError() { f(); } }; }", 0),
    ("api.hpp", "#define HIDDEN __attribute__((visibility(1)))\nnamespace pixo {\nHIDDEN int h2d_copy(X *ctx);\n}", 0),
    ("api_png.cu", "int d2h_copy_sync(X *ctx);", 1),
    ("api.cu", "int stage_host_call(X *ctx) { DrainOnError drain(ctx); return d2h_copy_sync(ctx, a, b, n, s); }", 0),
    ("api_png.cu", 'int f() { /* h2d_copy(x) */ return g("DrainOnError"); }', 0),
])
def test_scanner(name, src, want):
    assert len(findings(name, strip(src))) == want
