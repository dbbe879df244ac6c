"""The rows of filter_inputs.py sit where they are built to: tests/filter_ref.py equals the C oracle on every image for
all nine strategies, each constructed row lands on the route its faults live on, and each row's output changes
under every fault (filter_ref mutant) it targets.  CPU only."""
import numpy as np
import pytest

import filter_inputs as I
import filter_ref as R


def _images():
    return (I.band_images() + I.row_images() + I.alpha_images() + I.sticky_images() + I.bigram_images()
            + [I.longest_band_image()])


def _ref(po, im, st):
    d = po.optimize_alpha(im.data, 1 if im.oa == 2 else 3) if im.oa else im.data
    return po.apply_filters(d, im.width, im.height, im.bpp, st, row_bytes=im.rb)


def test_restatement_equals_the_oracle(po):
    for im in _images():
        for st in range(9):
            got, _ = R.apply_filters(im.data, im.width, im.height, im.bpp, st, im.rb, im.oa)
            assert np.array_equal(got, _ref(po, im, st)), (im.name, st)


def test_every_row_changes_under_the_faults_it_targets():
    for im in _images():
        for st in im.strategies:
            want, info = R.apply_filters(im.data, im.width, im.height, im.bpp, st, im.rb, im.oa)
            n = im.rb + 1
            for r, (flips, sts) in im.flips.items():
                if st not in sts:
                    continue
                for m in flips:
                    got, _ = R.apply_filters(im.data, im.width, im.height, im.bpp, st, im.rb, im.oa,
                                             mut=frozenset([m]))
                    assert not np.array_equal(got[r * n:(r + 1) * n], want[r * n:(r + 1) * n]), (im.name, st, r, m)


def test_rows_land_on_their_routes():
    """Coverage, from the route model: the faults' rows are scored on the route the fault lives on."""
    seen = set()
    for im in _images():
        for st in im.strategies:
            _, info = R.apply_filters(im.data, im.width, im.height, im.bpp, st, im.rb, im.oa)
            for r, (flips, sts) in im.flips.items():
                for m in flips if st in sts else ():
                    seen.add((str(m[0] if isinstance(m, tuple) else m), info[r].route, im.bpp))
    for bpp in (1, 2, 3, 4):
        for m, route in (("paeth_le:two", "two"), ("paeth_le:fused", "fused"), ("paeth_le:two", "first"), ("lane0_shfl", "two"),
                         ("no_ragged", "two"), ("no_trailing", "two"), ("fast_lt", "two"), ("adaptive_lt", "two"),
                         ("paeth_le:row", "row"), ("pass0_unmasked", "row"), ("drop", "row"), ("drop", "two")):
            assert (m, route, bpp) in seen, (m, route, bpp)
    for bpp in (1, 4):
        assert ("paeth_le:row", "sticky", bpp) in seen and ("fast_lt", "sticky", bpp) in seen
    for bpp in (2, 4):
        assert ("alpha_x0", "two", bpp) in seen
    for bpp in (1, 3, 4):
        assert ("bigram_seam", "bigrams", bpp) in seen


def test_routing_limits():
    assert R.use_band(68224) and not R.use_band(68225)
    assert R.effective_strategy(R.ADAPTIVE, 128, 32) == R.SUB and R.effective_strategy(R.ADAPTIVE, 241, 17) == R.ADAPTIVE
    assert R.effective_strategy(R.FAST, 64, 64) == R.SUB and R.effective_strategy(R.BIGRAMS, 17, 241) == R.BIGRAMS


@pytest.mark.parametrize("fast", [False, True])
def test_threshold_rows_score_exactly(fast):
    for rb in range(4128, 4136):
        for bpp in (1, 2, 3, 4):
            E = R.early_of(R.FAST if fast else R.ADAPTIVE, rb)
            (a0, r0), (a1, r1) = I.threshold_rows(rb, bpp, fast)
            s0, s1 = R.scores(r0.x, a0, bpp), R.scores(r1.x, a1, bpp)
            f = R.SUB if fast else R.NONE
            assert (s0[f], s1[f]) == (E, E + 1)
            p0 = R.ladder(s0, R.FAST if fast else R.ADAPTIVE, rb)
            assert p0.exit == "early" and p0.margin == 0 and min(s0) < E
            assert R.ladder(s1, R.FAST if fast else R.ADAPTIVE, rb).winner != f or not fast
