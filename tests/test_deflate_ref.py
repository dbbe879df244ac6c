"""Two restatements of pixo's DEFLATE check each other: oracle/png_deflate.c (C) and tests/deflate_ref.py (Python,
written separately from pixo's source).  Every constructed stream is asserted to take the branch it was built for.
CPU only."""
import zlib

import numpy as np
import pytest

import deflate_ref as R
from deflate_inputs import constructed, small_cases, stored_rule_stream
from oracle import png_deflate as pd

# the branch each small case is built to reach, and the levels where it must
EXPECT = {
    "zeros_2000": ({"run_dist1", "run_nice"}, range(2, 10)),
    "incompressible_exit": ({"incompressible_enter", "probe_exit"}, range(1, 10)),
    "gate_8192": ({"gate_8192"}, range(2, 10)),
    "tail_match": ({"tail_match"}, range(1, 10)),
    "sawtooth": ({"nice_exit"}, range(1, 10)),
    "lazy": ({"lazy_defer"}, range(5, 8)),
    "window_edge": ({"window_break"}, range(2, 10)),
    "text": ({"lazy2_defer"}, range(8, 10)),
    "short_noise": ({"incompressible_enter"}, range(1, 10)),
}


@pytest.fixture(scope="module", autouse=True)
def _build():
    pd.build()


@pytest.mark.parametrize("level", range(1, 10))
def test_token_streams_agree(level):
    seen = set()
    for name, data in small_cases().items():
        tok, ev = R.lz77(data, level)
        assert tok == pd.lz77(data, level).tolist(), (name, level)
        want, levels = EXPECT.get(name, (set(), ()))
        if level in levels:
            assert want <= ev, (name, level, ev)
        seen |= ev
    assert "hash4_zero" in seen or level == 1
    assert ("ht" in seen) == (level == 1)
    assert ("lazy2_defer" in seen) == (level >= 8) and ("lazy_defer" in seen) == (5 <= level <= 7)


@pytest.mark.parametrize("level", [1, 2, 6, 9])
def test_code_lengths_agree_on_every_histogram(level):
    for name, data in small_cases().items():
        lit, dist = pd.histogram(pd.lz77(data, level))
        lit = lit.copy()
        lit[256] += 1
        if not dist.any():
            dist = dist.copy()
            dist[0] = 1
        for f in (lit, dist):
            assert R.build_lengths(f.tolist(), 15)[0] == pd.code_lengths(f, 15).tolist(), (name, level)


def test_limits_at_15_and_7_bits():
    fib = [1, 1]
    while len(fib) < 22:
        fib.append(fib[-1] + fib[-2])
    f15 = fib + [0] * (286 - 22)
    got, ev = R.build_lengths(f15, 15)
    assert "limit_15" in ev and got == pd.code_lengths(np.array(f15, np.uint32), 15).tolist()
    f7 = fib[:12] + [0] * 7
    got, ev = R.build_lengths(f7, 7)
    assert "limit_7" in ev and got == pd.code_lengths(np.array(f7, np.uint32), 7).tolist()


def test_equal_frequency_internal_nodes_follow_rusts_heap_order():
    """Frequencies where popping tied internal nodes in another order gives other code lengths: both restatements
    follow Rust's BinaryHeap, and its order is not the insertion order."""
    rng = np.random.default_rng(5)
    differing = 0
    for _ in range(400):
        f = rng.integers(0, 4, int(rng.integers(5, 30))).tolist()
        rust, ev = R.build_lengths(f, 15)
        assert rust == pd.code_lengths(np.array(f, np.uint32), 15).tolist(), f
        if rust != R.build_lengths(f, 15, "fifo")[0]:
            assert "internal_tie" in ev
            differing += 1
    assert differing >= 10


def _header(z: bytes):
    """(BTYPE, HCLEN, the 19 3-bit code-length-code lengths in transmission order) of a one-block zlib stream."""
    bits = int.from_bytes(z[2:16], "little")
    take = lambda at, n: (bits >> at) & ((1 << n) - 1)
    btype, hclen = take(1, 2), take(13, 4)
    return btype, hclen, [take(17 + 3 * i, 3) for i in range(hclen + 4)]


def test_hclen_is_clamped_to_15():
    """One distance code gets a 1-bit length, so the code-length code of length 1 (18th in transmission order) is
    used: pixo's HCLEN index 17 is clamped to 15, which still sends all 19 entries."""
    rng = np.random.default_rng(2)
    data = rng.integers(0, 256, 300, dtype=np.uint8).tobytes() + bytes(3000)
    z = pd.deflate_zlib(data, 6)
    btype, hclen, cl = _header(z)
    assert btype == 2 and hclen == 15 and cl[17] > 0
    assert zlib.decompress(z) == data


def test_stored_rule_at_a_multiple_of_65535():
    """should_use_stored counts n / 65535 + 1 block headers: this stream's dynamic block is 6 bytes longer than the
    input, under the 10 it allows, so pixo keeps it although stored blocks would be a byte shorter."""
    d = stored_rule_stream()
    z = pd.deflate_zlib(d, 6)
    assert pd.deflate_kind(d, 6) == 2 and len(z) - 6 - len(d) == 6
    assert zlib.decompress(z) == d


def test_constructed_kinds():
    c = constructed()
    kinds = {name: pd.deflate_kind(d, 6) for name, d in c.items()}
    assert kinds["tiny_fixed"] == 1 and kinds["empty"] == 1
    assert kinds["noise_12k"] == 0 and kinds["noise_70k"] == 0
    assert len(R.lz77(c["short_noise"], 6)[0]) == 600 and kinds["short_noise"] == 0   # stored by should_use_stored
    assert kinds["text"] == 2
