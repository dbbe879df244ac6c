"""The inputs of test_deflate_edges_gpu.py land where they are built to: the is_high_entropy_data streams on their
side of 5 % in both oracle/png_deflate.c and tests/deflate_ref.py, with the block kind that side gives at every
level; the tails flip what a read past the stream would see; the stored-block streams are stored.  CPU only."""
import numpy as np
import pytest

import deflate_ref as R
from deflate_inputs import (LONGEST_BAIL, constructed, entropy_cases, entropy_stream, families, read_past_tail,
                            stored_block_noise)
from oracle import png_deflate as pd


@pytest.fixture(scope="module", autouse=True)
def _build():
    pd.build()


def test_the_f32_division_decides_at_exactly_five_percent():
    f = np.float32
    assert f(205) / f(4100) == f(0.05) and not f(205) / f(4100) < f(0.05)   # 4 103 bytes, 205 collisions: no bail
    assert f(204) / f(4100) < f(0.05)
    assert f(204) / f(4093) < f(0.05) < f(205) / f(4093)                    # 4 096 bytes


def test_longest_stream_that_can_fire():
    """Counting bound: min(n, 8192) - 3 4-grams in 4 096 slots repeat at least that many minus 4 096 times.  At
    4 314 bytes that is 215 of 4 311 (4.99 %), so the bail is not excluded; from 4 315 bytes on it is."""
    f = np.float32
    lows = {n: f(n - 3 - 4096) / f(n - 3) < f(0.05) for n in range(4096, 4400)}
    assert max(n for n, ok in lows.items() if ok) == 4314 and not any(lows[n] for n in range(4315, 4400))


@pytest.mark.parametrize("name", list(entropy_cases()))
def test_bail_streams_fall_on_their_side(name):
    s, coll, fires, _ = entropy_cases()[name]
    assert set(s) <= set(range(32))
    assert R.is_high_entropy_data(s) == (fires, coll if len(s) >= 4096 else 0)
    assert pd.high_entropy(s) == fires
    for level in range(1, 10):
        assert pd.deflate_kind(s, level) == (0 if fires else 2), level


def test_bail_tails_flip_the_decision():
    """A sample that read 8 bytes past the stream into its tail would decide the other way (the 4 095-byte stream: a
    length check that counted the tail would take the sample and fire)."""
    for name, (s, _, fires, tail) in entropy_cases().items():
        assert pd.high_entropy(s + tail[:8]) != fires, name
        assert R.is_high_entropy_data(s + tail[:8])[0] != fires, name


def test_longest_bail_is_the_best_prefix_of_its_seed():
    n, seed = LONGEST_BAIL
    s, _, _ = entropy_stream(n + 1, seed=seed)
    assert pd.high_entropy(s[:n]) and not pd.high_entropy(s)


def test_read_past_tails():
    """The default tail starts with the stream's last 300 bytes; below 4 096 bytes the values a stream lacks sit in
    the census' reach, so counting the tail moves the distinct count past 96 (minimum match 6 at levels 7-9)."""
    for name, s in constructed().items():
        t = read_past_tail(s, 4096 + 258 + 301)
        if s:
            assert t.startswith(s[-300:]) or len(s) > 3700, name
        if s and len(s) < 4096:
            assert len(set((s + t)[:4096])) == 256, name
            if len(set(s)) <= 96:
                assert pd.lz77(s + t[:4096 - len(s)], 9).size != pd.lz77(s, 9).size or len(s) < 64, name


def test_families_share_content_and_come_shuffled():
    fam = families(400, seed=1)
    lens = np.array([len(s) for s in fam])
    assert lens.min() >= 1024 and lens.max() <= 4096
    assert (np.argsort(-lens, kind="stable") != np.arange(lens.size)).any()
    prefixes = {s[:1024] for s in fam}
    assert len(prefixes) == 10


@pytest.mark.parametrize("level", [1, 6, 9])
def test_stored_block_streams_are_stored(level):
    for n, s in stored_block_noise().items():
        z = pd.deflate_zlib(s, level)
        assert pd.deflate_kind(s, level) == 0
        assert len(z) == 2 + n + 5 * -(-n // 65535) + 4
