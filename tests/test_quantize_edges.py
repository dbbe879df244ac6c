"""The cases of quantize_edge_inputs.py sit where they are built to: tests/quantize_ref.py equals the oracle
(oracle/png_quantize.py / .c) on every case (palette, indices, decision and refusal), each case changes its output under
every mutant it targets, each mutant's cases reach the route its fault lives on with the tie it needs, and the ties,
near misses, sample counts and dither extremes are exact.  The 512 x 512 and 2^24-colour images are checked on the GPU
against the C oracle only.  CPU only."""
import numpy as np
import pytest

import quantize_edge_inputs as I
import quantize_ref as R
from oracle import png_quantize as pq


@pytest.fixture(scope="module")
def cases():
    return {"tie": I.tie_cases(), "sweep": I.sweep_cases(), "early": I.early_cases(), "kmeans": I.kmeans_cases(),
            "cut": I.cut_cases(), "decision": I.decision_cases(), "dither": I.dither_cases()}


@pytest.fixture(scope="module")
def results(cases):
    out = {}
    for fam, cs in cases.items():
        for c in cs:
            try:
                out[c.name] = c.run()
            except R.Refused:
                out[c.name] = "refused"
    return out


def oracle(c):
    """('lossless',) / 'refused' / (palette, indices) from the oracle."""
    if not pq.should_quantize(c.data, c.ct, c.mode, min(c.m, 256)):
        return ("lossless",)
    try:
        pal, idx = pq.quantize(c.data, c.w, c.h, c.ct, c.m, c.dither, c.palette)
    except pq.TruncationCase:
        return "refused"
    return pal, idx


@pytest.mark.parametrize("family", ["tie", "sweep", "early", "kmeans", "cut", "decision", "dither"])
def test_restatement_equals_the_oracle(cases, results, family):
    for c in cases[family]:
        got, want = results[c.name], oracle(c)
        if isinstance(want, str) or len(want) == 1:
            assert (got if isinstance(got, str) else got.key()) == (want if isinstance(want, str) else want), c.name
            continue
        assert got != "refused" and got.kind != "lossless", c.name
        assert np.array_equal(got.palette, want[0]), c.name
        assert np.array_equal(got.indices, want[1]), (c.name, np.flatnonzero(got.indices != want[1])[:5])
        assert R.trimmed_trns(got.palette) == pq.trimmed_trns(want[0]), c.name


def _key(c, m):
    if m in c.keys:
        return c.keys[m]
    try:
        return c.run(frozenset([m])).key()
    except R.Refused:
        return "refused"


@pytest.mark.parametrize("family", ["tie", "sweep", "early", "kmeans", "cut", "decision", "dither"])
def test_every_case_changes_under_the_mutants_it_targets(cases, results, family):
    for c in cases[family]:
        base = results[c.name]
        base = base if isinstance(base, str) else base.key()
        for m in c.targets:
            assert m in R.MUTANTS, m
            assert _key(c, m) != base, (c.name, m)


def test_every_mutant_is_targeted(cases):
    targeted = {m for cs in cases.values() for c in cs for m in c.targets}
    # rm_ceil: a tie between r + 1 and b + 1 keeps its weights when r_mean rounds up; no case is built for it
    assert set(R.MUTANTS) - targeted == {"rm_ceil"}, set(R.MUTANTS) - targeted
    assert not set(R.EQUIVALENT) & set(R.MUTANTS)


def test_cases_land_on_their_routes(cases, results):
    """Each tie sits in the tie set of a pixel on the route its mutants live on; every placement and palette size is
    reached on the table and the warp search."""
    seen = set()
    for fam in ("tie", "early", "dither", "sweep"):
        for c in cases[fam]:
            r = results[c.name]
            if "tie" not in c.expect:
                continue
            i, j = c.expect["tie"]
            routes = {rt for rt, tt in zip(r.routes, r.ties) if i in tt and j in tt}
            assert c.expect["route"] in routes, c.name
            for m in c.targets:
                seen.add((m, c.expect["route"]))
            if fam == "tie":
                seen.add(("n", c.expect["n"], c.expect["route"]))
                seen.add(("where", c.expect["where"], c.expect["route"]))
    for m, route in (("warp_lane", "warp"), ("warp_lane", "early-miss"), ("warp_lane", "dither-warp"),
                     ("warp_last", "warp"), ("warp_last", "early-miss"), ("warp_last", "dither-warp"),
                     ("seq_last", "table"), ("dist_exact", "table"), ("dist_exact", "warp"),
                     ("dist_exact", "early-miss"), ("table_alpha", "warp")):
        assert (m, route) in seen, (m, route)
    for route in ("table", "warp"):
        for n in I.SIZES:
            assert ("n", n, route) in seen, (n, route)
        for where in ("first-last", "cross-lane", "same-lane", "same-lane-64", "adjacent"):
            assert ("where", where, route) in seen, (where, route)
    # the sweeps: one tie per r <= 254 on the warp search, every cell r6 <= 62 on the table
    rs = [r for c in cases["sweep"] if c.name.startswith("sweep-warp") for r in c.expect["rs"]]
    assert sorted(rs) == list(range(255))
    sw = results["sweep-table"]
    assert all(rt == "table" and len(t) == 2 for rt, t in zip(sw.routes, sw.ties))
    # k-means ties in each pass, and an entry emptied
    km = {c.expect["kmeans"]: results[c.name].kmeans for c in cases["kmeans"]}
    assert km["km-tie-pass1"].tied[0] and km["km-tie-pass2"].tied[1] and km["km-empty-pass1"].empty[0]
    # median cut's tie rules
    cut = {c.expect["cut"]: results[c.name].cut for c in cases["cut"]}
    assert cut["cut-box-tie"].box_tie and cut["cut-channel-tie"].channel_tie and cut["cut-split-eq"].split_eq
    assert cut["cut-clamp"].clamped


def test_ties_and_near_misses_are_exact(cases):
    for c in cases["tie"]:
        if "tie" in c.expect:
            i, j = c.expect["tie"]
            t = R.pixels(c.data, c.ct)[0]
            d = R.distance(t[None], c.palette[[i, j]])[0]
            assert d[0] == d[1], c.name
            if c.expect["kind"] in ("trunc", "floor"):
                e = R.distance(t[None], c.palette[[i, j]], frozenset(["dist_exact"]))[0]
                assert e[0] != e[1], c.name
        elif "miss" in c.expect:
            i, j = c.expect["miss"]
            d = R.distance(R.pixels(c.data, c.ct)[:1], c.palette[[i, j]])[0]
            assert abs(int(d[0]) - int(d[1])) == 1, c.name
    # every r <= 254: red + 1 and blue + 1 both at distance 2
    for r in range(255):
        t = np.array([[r, 7, 9, 255]])
        assert list(R.distance(t, np.array(I._pair("trunc", tuple(t[0])))[None][0])[0]) == [2, 2]


def test_samplers_read_exactly_the_intended_counts(cases, results):
    for c in cases["decision"]:
        px = R.pixels(c.data, c.ct)
        if "unique" in c.expect:
            assert R.decision_unique(px) == c.expect["unique"], c.name
            if "stride" in c.expect:
                assert max(len(px) // R.DECISION_CAP, 1) == c.expect["stride"]
        if "hist" in c.expect:
            assert len(R.histogram(px)[0]) == c.expect["hist"], c.name
    assert results["trunc-8193"] == "refused" and results["trunc-8192"].kind == "lut"
    assert results["trunc-8193-palette"].kind == "given"


def test_dither_reaches_full_scale(results, cases):
    st = [results[c.name].dither for c in cases["dither"] if c.expect.get("full")]
    assert max(s.max_err for s in st) == 255
    assert any(s.low for s in st) and any(s.high for s in st)


@pytest.mark.parametrize("n", [63, 64, 65, 128, 129])
def test_batch_sampler_and_the_sort_bits(n):
    """The device sampler's per-image results equal each image's own samples, and sorting on bits 0-37 instead of
    0-38 changes nothing (EQUIVALENT['sort_bits_38']); the decisions alternate."""
    frames = I.batch_frames(n)
    want = []
    for f in frames:
        px = R.pixels(f, 2)
        k, cnt = R.histogram(px)
        want.append((R.decision_unique(px), k.tolist(), cnt.tolist()))
    for end_bit in (39, 38):
        assert R.batch_samples(frames, 2, end_bit) == want, end_bit
    assert [R.auto_quantises(u, 4) for u, _, _ in want] == [i % 2 == 1 for i in range(n)]
