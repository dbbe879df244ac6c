"""What crosses a band boundary in the progressive scans of a tiled frame (pixo_b200.parallel): the EOB-run carries
of the AC scans, the DC predictors and every scan's bit offsets.  CPU only: the carries are checked against a
brute-force walk of pixo's EOB-run rule (encode_ac_first / flush_eob_run) over constructed flag sequences."""
import numpy as np
import pytest

from pixo_b200 import parallel

EOBRUN_MAX = 0x7FFF


def walk(flags):
    """pixo's rule over a whole scan: flags[i] = (non-empty, init).  -> [(block, run)] of every EOB-run flush, in
    order: a non-empty block flushes the pending run before its symbols; an empty one counts, and flushes at 0x7FFF;
    the scan's end flushes what is pending."""
    out, run = [], 0
    for i, (ne, init) in enumerate(flags):
        if ne:
            if run:
                out.append((i, run))
            run = int(init)
        else:
            run += 1
            if run == EOBRUN_MAX:
                out.append((i, run))
                run = 0
    if run:
        out.append((len(flags) - 1, run))
    return out


def enc_of(i, ne, init):
    return ((i + 1) << 1 | int(init)) if ne else 0


def band_flushes(flags, base, n_frame, carry):
    """One band's flushes from its carry alone, as the band kernels place them (frame indices)."""
    out, excl = [], int(carry)
    for k, (ne, init) in enumerate(flags):
        b = base + k
        p1, ini = excl >> 1, excl & 1
        empties = b - p1
        if ne:
            r = (ini + empties) % EOBRUN_MAX
            if r:
                out.append((b, r))
            pending = int(init)
            excl = enc_of(b, ne, init)
        else:
            pending = (ini + empties + 1) % EOBRUN_MAX
            if pending == 0:
                out.append((b, EOBRUN_MAX))
        if b + 1 == n_frame and pending:
            out.append((b, pending))
    return out


def tiled(flags, cuts):
    """The flushes of the bands flags[cuts[r]:cuts[r+1]], each from ac_carries over the earlier bands' summaries."""
    bounds = list(zip(cuts, cuts[1:]))
    last = [[max([enc_of(lo + k, *f) for k, f in enumerate(flags[lo:hi])], default=0)] * 4 for lo, hi in bounds]
    out = []
    for r, (lo, hi) in enumerate(bounds):
        carry = parallel.ac_carries(last, r)
        assert len(set(carry.tolist())) == 1
        out += band_flushes(flags[lo:hi], lo, len(flags), carry[0])
    return out


def seq(*parts):
    """('e', n) n empty blocks; ('n', init) one non-empty block."""
    out = []
    for kind, v in parts:
        out += [(False, False)] * v if kind == "e" else [(True, bool(v))]
    return out


M = EOBRUN_MAX
CASES = {
    "short": (seq(("n", 1), ("e", 3), ("n", 0), ("e", 2), ("n", 1)), [0, 2, 2, 4, 8]),
    "empty bands": (seq(("e", 5), ("n", 1), ("e", 4)), [0, 0, 3, 3, 3, 8, 10, 10]),
    "run over bands": (seq(("n", 1), ("e", 3 * 1000), ("n", 0)), [0, 1, 500, 1500, 2999, 3002]),
    "0x7FFF on a boundary": (seq(("n", 0), ("e", M), ("e", 5), ("n", 1)), [0, 1, M + 1, M + 7]),
    "0x7FFF - 1 with init": (seq(("n", 1), ("e", M - 1), ("e", 3)), [0, M, M + 3]),
    "twice 0x7FFF on boundaries": (seq(("e", 2 * M), ("e", 1)), [0, M, 2 * M, 2 * M + 1]),
    "exact multiple at the end": (seq(("n", 1), ("e", 2 * M - 1)), [0, 1, M, 2 * M]),
    "last band empty of non-empty": (seq(("n", 0), ("e", 10), ("n", 1), ("e", 40)), [0, 6, 12, 30, 52]),
    "all empty": (seq(("e", M + 9)), [0, 4, M + 9]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_carries_against_pixo_walk(name):
    flags, cuts = CASES[name]
    assert cuts[0] == 0 and cuts[-1] == len(flags)
    assert tiled(flags, cuts) == walk(flags)
    assert tiled(flags, [0, len(flags)]) == walk(flags)


def test_carries_on_random_flags():
    rng = np.random.default_rng(7)
    for trial in range(60):
        n = int(rng.integers(1, 400))
        p = [0.5, 0.05, 0.0][trial % 3]
        flags = [(bool(rng.random() < p), bool(rng.random() < 0.5)) for _ in range(n)]
        cuts = sorted([0, n] + [int(c) for c in rng.integers(0, n + 1, int(rng.integers(0, 9)))])
        assert tiled(flags, cuts) == walk(flags), (trial, cuts)


def test_ac_carries_take_the_nearest_non_empty_band():
    last = [[6, 0, 4, 0], [0, 0, 0, 0], [20, 8, 0, 0], [0, 0, 0, 0]]
    assert parallel.ac_carries(last, 0).tolist() == [0, 0, 0, 0]
    assert parallel.ac_carries(last, 2).tolist() == [6, 0, 4, 0]
    assert parallel.ac_carries(last, 3).tolist() == [20, 8, 4, 0]
    assert parallel.ac_carries(last, 4).tolist() == [20, 8, 4, 0]


def test_dc_seeds_per_component():
    last = np.array([[5, 7, 9], [0, 0, 0], [-3, 0, 0], [11, 12, 13]])
    counts = np.array([[4, 1, 1], [0, 0, 0], [4, 0, 0], [4, 1, 1]])
    assert parallel.prog_dc_seeds(last, counts, 0).tolist() == [0, 0, 0]
    assert parallel.prog_dc_seeds(last, counts, 1).tolist() == [5, 7, 9]
    assert parallel.prog_dc_seeds(last, counts, 2).tolist() == [5, 7, 9]
    assert parallel.prog_dc_seeds(last, counts, 3).tolist() == [-3, 7, 9]   # band 2 has Y blocks only


def bits_of(parts):
    """[(bit count, value)] -> the stream as a '0'/'1' string."""
    return "".join(format(v, f"0{n}b") if n else "" for n, v in parts)


@pytest.mark.parametrize("lens", [[13, 0, 3, 2, 9, 0], [0, 0, 5], [1, 1, 1, 1, 1, 1, 1, 1, 1], [7, 8, 0, 0, 1],
                                  [0, 0, 0], [20, 0, 0, 0]])
def test_scan_bit_offsets(lens):
    rng = np.random.default_rng(sum(lens))
    parts = [(n, int(rng.integers(0, 1 << n)) if n else 0) for n in lens]
    stream = bits_of(parts)
    tails = [v & 0x7F if n >= 7 else v for n, v in parts]
    for r, (n, _) in enumerate(parts):
        start, tail_in, is_last = parallel.scan_bit_offsets(lens, tails, r)
        assert start == sum(lens[:r])
        ph = start & 7
        want = int(stream[start - ph:start], 2) if ph else 0
        assert tail_in == want, (r, lens)
        assert is_last == (n > 0 and not any(lens[r + 1:]))
