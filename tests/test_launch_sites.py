"""Source checks on pixo_b200/csrc: every kernel is launched through pixo::launch (common.cuh), which
enqueues it on the context's stream, counts it and checks it, and no function keeps mutable static
state (kernel attributes are kept per context).  Needs no GPU."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pixo_b200", "csrc")


def strip(src: str) -> str:
    """Comments, string and character literals blanked out (newlines kept)."""
    tok = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
    return tok.sub(lambda m: re.sub(r"[^\n]", " ", m.group(0)) if m.group(0)[0] == "/" else
                   m.group(0)[0] + " " * (len(m.group(0)) - 2) + m.group(0)[-1], src)


def scopes(code: str):
    """For every offset, the headers of the code blocks (function bodies, statements, lambdas,
    initialisers) that enclose it: a list per '{', innermost last.  Namespace, class, struct, union, enum
    and extern "C" braces are not code blocks."""
    stack, out, start = [], [], 0   # stack: (is a code block, header)
    for i, ch in enumerate(code):
        if ch == "{":
            header = code[start:i].strip()
            code_block = (")" in header or "=" in header or header.endswith("]") or
                          header in ("", "else", "do", "try") or bool(stack and stack[-1][0]))
            stack.append((code_block, header))
            start = i + 1
        elif ch == "}":
            stack.pop()
            start = i + 1
        elif ch == ";":
            start = i + 1
        out.append([h for c, h in stack if c])
    return out


def enclosing_function(code: str, pos: int, sc) -> str:
    """The header of the outermost code block around pos ('' at namespace scope)."""
    return sc[pos][0] if sc[pos] else ""


def mutable_statics(code: str):
    """Function-local static variables that are neither const nor constexpr: (line, declaration)."""
    sc = scopes(code)
    found = []
    for m in re.finditer(r"\bstatic\b([^;={(\[]*)", code):
        if sc[m.start()] and not re.search(r"\b(const|constexpr)\b", m.group(1)):
            found.append((code.count("\n", 0, m.start()) + 1, m.group(0).strip()))
    return found


LAUNCH_WRITE = re.compile(r"(->|\.)\s*launches\s*(\+\+|--|[-+*/%&|^]?=(?!=))|(\+\+|--)\s*[\w.>-]*(->|\.)\s*launches\b")


def sources():
    names = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".cpp", ".hpp")))
    assert "common.cuh" in names
    return [(n, strip(open(os.path.join(CSRC, n)).read())) for n in names]


def test_every_launch_goes_through_the_helper():
    sites = []
    for name, code in sources():
        sc = scopes(code)
        for m in re.finditer(r"<<<", code):
            sites.append((name, enclosing_function(code, m.start(), sc)))
    assert len(sites) == 1, sites
    name, fn = sites[0]
    assert name == "common.cuh" and re.search(r"\bint launch\(", fn), sites


def test_launch_count_is_written_by_the_helper_only():
    writes = []
    for name, code in sources():
        sc = scopes(code)
        writes += [(name, enclosing_function(code, m.start(), sc)) for m in LAUNCH_WRITE.finditer(code)]
    assert len(writes) == 1, writes
    name, fn = writes[0]
    assert name == "common.cuh" and re.search(r"\bint launch\(", fn), writes


def test_no_mutable_function_local_statics():
    found = [(name,) + f for name, code in sources() if name.endswith((".cu", ".cpp")) for f in mutable_statics(code)]
    assert not found, found


@pytest.mark.parametrize("src,want", [
    ("static int counter;\nnamespace a { static bool flag; struct S { static int n; }; }", []),
    ("static int f(int x) { static const int t[2] = {1, 2}; static constexpr int k = 3; return t[x] + k; }", []),
    ("int f() { static int calls; return ++calls; }", [(1, "static int calls")]),
    ("namespace {\nvoid g(bool b)\n{\n    if (b) {\n        static bool done[64];\n    }\n}\n}", [(5, "static bool done")]),
    ("auto h = [] { static thread_local int n; return n; };", [(1, "static thread_local int n")]),
    ('void k() { const char *s = "static int x;"; /* static int y; */ auto p = static_cast<int>(1.0); }', []),
])
def test_static_scanner(src, want):
    assert mutable_statics(strip(src)) == want


@pytest.mark.parametrize("src,want", [
    ("void f(pixo_b200_ctx *ctx) { ctx->launches++; }", 1),
    ("void f(pixo_b200_ctx *ctx) { ctx->launches += 4; ++ctx->launches; }", 2),
    ("uint64_t n(const pixo_b200_ctx *c) { return c->launches; } bool e(X *c) { return c->launches == 0; }", 0),
    ("struct pixo_b200_ctx { uint64_t launches = 0; };", 0),
])
def test_launch_write_pattern(src, want):
    assert len(LAUNCH_WRITE.findall(strip(src))) == want
