"""The DEFLATE oracle (oracle/png_deflate.c, pixo's deflate_zlib_packed at levels 1-9) against real pixo output and
zlib.  CPU only."""
import zlib

import numpy as np
import pytest

from deflate_inputs import constructed, golden_pngs, idat
from oracle import png_deflate as pd


@pytest.fixture(scope="module", autouse=True)
def _build():
    pd.build()


def test_oracle_reproduces_every_golden_png_whole():
    """Each preset-0/1 golden is rebuilt from its own filtered stream and pre-IDAT chunks: the oracle's zlib stream at
    the preset's level, cut into 256 KiB IDAT chunks with their CRCs, then IEND, equals pixo's file byte for byte."""
    files = golden_pngs()
    assert len(files) == 199
    for path, level in files:
        png = open(path, "rb").read()
        ch = pd.chunks(png)
        head = pd.SIGNATURE + b"".join(pd.chunk(k, p) for k, p in ch if k not in (b"IDAT", b"IEND"))
        z = pd.deflate_zlib(zlib.decompress(idat(png)), level)
        rebuilt = head + b"".join(pd.chunk(b"IDAT", z[i:i + pd.IDAT_CHUNK]) for i in range(0, len(z), pd.IDAT_CHUNK))
        assert rebuilt + pd.chunk(b"IEND", b"") == png, path


def test_png_file_writer_matches_a_golden():
    path, level = golden_pngs()[0]
    png = open(path, "rb").read()
    ch = dict(pd.chunks(png))
    w, h, depth, ct = np.frombuffer(ch[b"IHDR"][:8], ">u4").tolist() + list(ch[b"IHDR"][8:10])
    pal = np.frombuffer(ch[b"PLTE"], np.uint8).reshape(-1, 3) if b"PLTE" in ch else None
    got = pd.png_file(w, h, depth, ct, pd.deflate_zlib(zlib.decompress(idat(png)), level), pal, ch.get(b"tRNS"))
    assert got == png


@pytest.mark.parametrize("level", range(1, 10))
def test_constructed_streams_inflate_to_their_input(level):
    for name, data in constructed().items():
        z = pd.deflate_zlib(data, level)
        assert zlib.decompress(z) == data, (name, level)
        assert z[:2] == bytes([0x78, 0x5E if level <= 2 else 0x9C if level <= 6 else 0xDA]), name


def test_constructed_streams_reach_each_block_kind():
    kinds = {name: pd.deflate_kind(d, 6) for name, d in constructed().items()}
    assert kinds["tiny_fixed"] == 1 and kinds["empty"] == 1
    assert kinds["noise_12k"] == 0 and kinds["noise_70k"] == 0 and kinds["short_noise"] == 0
    assert kinds["text"] == 2 and kinds["zeros_9000"] in (1, 2)
    assert len(pd.deflate_zlib(constructed()["noise_70k"], 6)) == 2 + 70000 + 2 * 5 + 4


def test_distance_one_run_and_window_edge_tokens():
    t = pd.lz77(bytes(9000), 6)
    assert (t[0] >> 31) == 1 and (t[1] & 0xFFFF) == 258 and (t[1] >> 16) == 0   # a literal, then runs at distance 1
    inside, edge = constructed()["window_inside"], constructed()["window_edge"]
    dist = lambda tok: [(x >> 16) + 1 for x in tok if not x >> 31]
    assert max(dist(pd.lz77(inside, 6))) == 32000
    assert max(dist(pd.lz77(edge, 6)), default=0) < 32768 - 0 and 33000 not in dist(pd.lz77(edge, 6))


def test_histogram_counts_every_token():
    t = pd.lz77(constructed()["text"], 6)
    lit, dist = pd.histogram(t)
    assert lit.sum() == t.size and dist.sum() == int((t >> 31 == 0).sum())


def test_code_lengths_are_limited_and_tie_sensitive():
    # Fibonacci counts make a 21-deep tree: limit_code_lengths truncates it to 15 bits, then lengthens the shortest
    # codes until the Kraft sum fits and shortens the longest while it stays within it
    f = np.zeros(286, np.uint32)
    a, b = 1, 1
    for i in range(22):
        f[i] = a
        a, b = b, a + b
    ln = pd.code_lengths(f, 15)
    assert ln.tolist()[:22] == [5] + [6] * 16 + [5, 4, 3, 2, 2] and not ln[22:].any()
    assert sum(2.0 ** -int(x) for x in ln[:22]) <= 1.0
    assert pd.code_lengths(f[:14], 15).max() == 13   # within the limit: the plain Huffman depths
    # equal counts: internal nodes tie; the lengths still form a complete code
    eq = pd.code_lengths(np.full(19, 5, np.uint32), 7)
    assert sum(2.0 ** -int(x) for x in eq) == 1.0


def test_high_entropy_bail_never_fires_on_the_samples():
    """is_high_entropy_data needs fewer than 5 % repeated 4-gram hashes; n - 3 4-grams in 4 096 slots repeat at
    least n - 4 099 times, so from 4 315 bytes on it cannot fire.  Random data near 4 096 bytes does not reach it
    either (test_deflate_edges.py builds streams that do)."""
    rng = np.random.default_rng(3)
    for n in (4096, 4200, 4311, 8192, 100000):
        assert not pd.high_entropy(rng.integers(0, 256, n, dtype=np.uint8).tobytes()), n
