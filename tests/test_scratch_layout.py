"""Source checks on pixo_b200/csrc: every scratch layout is described through pixo::Layout (common.cuh),
the one place that knows the 256-byte region rule, so that no buffer is sized by one copy of a layout and
bound by another.  Needs no GPU."""
import os
import re

from test_launch_sites import CSRC, strip

# a 256-byte round-up or round-down written out by hand
ROUND_UP = re.compile(r"\balign_up\s*\(|/\s*256\s*\*\s*256|&\s*~\s*\(\s*size_t\s*\)\s*255")
# a region derived by an offset or an index from a Buffer's pointer (Buffer::slot is the one allowance: slot i
# of a buffer used as an array of equal slots)
PTR_ARITH = re.compile(r"\.ptr\s*\)?\s*(?:[-+](?![-+=])|\[)")


def layout_class(code: str):
    """The span of `class Layout { ... };` in code, or None."""
    m = re.search(r"\bclass\s+Layout\s*\{", code)
    if not m:
        return None
    depth, i = 0, m.end() - 1
    while True:
        depth += {"{": 1, "}": -1}.get(code[i], 0)
        if depth == 0:
            return m.start(), i
        i += 1


def findings(name: str, code: str):
    span = layout_class(code) if name == "common.cuh" else None
    out = []
    for pat, what in ((ROUND_UP, "256-byte round-up"), (PTR_ARITH, "pointer arithmetic on .ptr")):
        for m in pat.finditer(code):
            if span and span[0] <= m.start() <= span[1]:
                continue
            out.append(f"{name}:{code.count(chr(10), 0, m.start()) + 1}: {what}")
    return out


def test_layouts_go_through_the_helper():
    names = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".cpp", ".hpp")))
    assert "common.cuh" in names
    code = {n: strip(open(os.path.join(CSRC, n)).read()) for n in names}
    assert layout_class(code["common.cuh"]), "common.cuh has no class Layout"
    bad = [f for n in names for f in findings(n, code[n])]
    assert not bad, "scratch laid out by hand (use pixo::Layout):\n" + "\n".join(bad)


def test_patterns():
    for s in ("align_up(n * 8, 256)", "(x + 255) / 256 * 256", "(v + 255) & ~(size_t)255", "(2 * c + 256) / 256 * 256",
              "(cap - t) / 256 * 256", "static_cast<uint8_t *>(ctx->d_misc.ptr) + hist_bytes", "(uint8_t *)buf.ptr + 4",
              "&static_cast<uint8_t *>(ctx->h_in.ptr)[i * SLOT]", "b.ptr[4]"):
        assert findings("x.cu", s), s
    for s in ("(total + 255) / 256", "L.take<uint32_t>(n)", "ctx->h_in.slot(i, SLOT)", "ctx->d_out.ptr, bytes",
              "if (ptr) cudaFree(ptr);"):
        assert not findings("x.cu", s), s
    helper = "class Layout {\n  size_t round(size_t b) { return (b + 255) / 256 * 256; }\n};\nalign_up(1, 2)"
    assert len(findings("common.cuh", helper)) == 1
