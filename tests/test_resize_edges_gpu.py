"""The CUDA resizers (csrc/resize.cu) at their edges, every output compared byte for byte with oracle/resize.c
inside guard bytes:

- Lanczos3 under small scratch caps (PIXO_B200_RESIZE_SCRATCH): row bands closed exactly at the cap and one
  byte under it, column chunks with a one-column last chunk, one column per chunk, and one-band batches split
  into frame passes.  Each case's launch count is the one resize_ref's band model plans for it, so a case
  cannot take another path, or multiply its launches, unnoticed.
- The real 256 MiB cap, no hook: gray 2 x 65 536 to 4 096 x 1 needs exactly the cap (one band), to
  4 097 x 1 one column more (column chunks of 4 096 and 1).
- Every (src, dst) pair in 1..48 on each axis, all three algorithms, 1 and 4 bytes per pixel; Nearest and
  Bilinear also against the numpy restatement in resize_ref.
- Exact halves: Bilinear 2 -> 3 and 2 -> 5 over every (a, b) byte pair, and Nearest at even integer ratios,
  whose expected bytes come from integer arithmetic.
- Lanczos3 calls with growing tables queued behind a delay on the caller's stream, reusing both pinned
  upload buffers."""
import numpy as np
import pytest
import torch

import resize_edge_inputs as ei
import resize_ref as rr
from oracle import resize as rz
from pixo_b200 import Context, _lib
from test_dev_layouts_gpu import GUARD8, Buf, assert_guard, guarded
from test_resize_gpu import resize_dev
from test_stream_contract_gpu import DELAY, resize_case, sleep_on

pytestmark = pytest.mark.gpu
HOOK = "PIXO_B200_RESIZE_SCRATCH"


@pytest.fixture(autouse=True)
def no_hook_no_host_fallback(gpu_ctx, monkeypatch):
    monkeypatch.delenv(HOOK, raising=False)
    yield
    assert gpu_ctx.host_fallbacks == 0


def counted(ctx, frames, geom, bpp, alg, **layout):
    """resize_dev (guarded output, odd offsets and strides) and the number of kernels it launched"""
    before = ctx.launch_count
    got = resize_dev(ctx, frames, *geom, bpp - 1, alg, **layout)
    return got, ctx.launch_count - before


# ---- scratch caps -------------------------------------------------------------------------------------
CAP_CASES = ei.cap_cases()


@pytest.mark.parametrize("case", CAP_CASES, ids=[c[0] for c in CAP_CASES])
def test_lanczos_under_scratch_cap(gpu_ctx, monkeypatch, case):
    name, geom, bpp, n, cap, _ = case
    frames = ei.frames(*geom[:2], bpp, n, seed=len(name) + cap % 997)
    want = [rz.resize(f, *geom, bpp - 1, 2) for f in frames]
    layout = dict(off=1, pad=3, out_off=65, out_pad=5)
    whole, k = counted(gpu_ctx, frames, geom, bpp, 2, **layout)
    assert k == ei.plan(*geom, bpp, n, rr.SCRATCH)[2] == 2
    monkeypatch.setenv(HOOK, str(cap))
    got, k = counted(gpu_ctx, frames, geom, bpp, 2, **layout)
    assert k == ei.plan(*geom, bpp, n, cap)[2], (name, k)
    for i in range(n):
        assert np.array_equal(whole[i], want[i]), (name, "uncapped", i)
        assert np.array_equal(got[i], want[i]), (name, i, int((got[i] != want[i]).sum()))


@pytest.mark.parametrize("dw,launches", [(4096, 2), (4097, 4)])
def test_lanczos_at_the_real_cap(gpu_ctx, dw, launches):
    """2 x 65 536 gray -> dw x 1: one destination row whose window is all 65 536 source rows, so the
    intermediate is 65 536 dw bytes: exactly 2^28 for 4 096 columns, just over for 4 097."""
    assert ei.plan(2, 65536, dw, 1, 1, 1, rr.SCRATCH)[2] == launches
    f = ei.noise(2, 65536, 1, dw)
    got, k = counted(gpu_ctx, [f], (2, 65536, dw, 1), 1, 2)
    assert k == launches
    assert np.array_equal(got[0], rz.resize(f, 2, 65536, dw, 1, 0, 2))


# ---- every small geometry -----------------------------------------------------------------------------
SIDES = range(1, 49)
OTHER = (7, 5)   # the axis not swept: 7 -> 5


def geometry(axis, s, d):
    return (s, OTHER[0], d, OTHER[1]) if axis == "x" else (OTHER[0], s, OTHER[1], d)


@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("alg", range(3))
@pytest.mark.parametrize("axis", ["x", "y"])
def test_every_small_geometry(gpu_ctx, axis, alg, bpp):
    """All 48 x 48 calls queued on the context's stream, one synchronisation; each output in its own slot
    (4-byte aligned: RGBA Nearest takes the word copies) between guard bytes."""
    srcs = {s: ei.noise(*geometry(axis, s, 1)[:2], bpp, 7 * s + alg) for s in SIDES}
    base, at = [], 0
    for s in SIDES:
        base.append(at)
        at += (srcs[s].size + 255) // 256 * 256
    src = Buf(np.concatenate([np.pad(srcs[s], (0, (-srcs[s].size) % 256)) for s in SIDES]))
    slots, at = {}, 64
    for s in SIDES:
        for d in SIDES:
            g = geometry(axis, s, d)
            slots[s, d] = (at, g[2] * g[3] * bpp)
            at += (slots[s, d][1] + 16 + 3) // 4 * 4
    out = guarded(at - 64, np.uint8, GUARD8)
    lib = _lib.load()
    torch.cuda.synchronize()
    for i, s in enumerate(SIDES):
        for d in SIDES:
            g = geometry(axis, s, d)
            _lib.check(gpu_ctx.handle, lib.pixo_b200_resize_dev(gpu_ctx.handle, src.ptr(base[i]), 0, 1, *g, bpp - 1,
                                                                alg, out.ptr(slots[s, d][0]), 0))
    gpu_ctx.sync()
    o = out.get()
    assert_guard(o, list(slots.values()), GUARD8, "resize output")
    for s in SIDES:
        for d in SIDES:
            g, (at, n) = geometry(axis, s, d), slots[s, d]
            want = rz.resize(srcs[s], *g, bpp - 1, alg)
            assert np.array_equal(o[at:at + n], want), (g, int((o[at:at + n] != want).sum()))
            if alg < 2:
                assert np.array_equal(rr.resize(srcs[s], *g, bpp, alg), want), g


# ---- exact halves -------------------------------------------------------------------------------------
@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("dst", [3, 5])
@pytest.mark.parametrize("axis", ["x", "y"])
def test_bilinear_exact_halves(gpu_ctx, axis, dst, bpp):
    """Every (a, b) byte pair blended at 1/2 (and 1/4, 3/4) of the way: half the sums that end in .5 round
    the other way under round-half-even."""
    ab = ei.pairs(bpp)                                   # (rows, 2, bpp)
    rows = ab.shape[0]
    e = ei.bilinear_halves(ab[:, 0].reshape(-1), ab[:, 1].reshape(-1), dst).reshape(rows, bpp, dst)
    if axis == "x":
        img, geom, want = ab, (2, rows, dst, rows), e.transpose(0, 2, 1)
    else:
        img, geom, want = ab.transpose(1, 0, 2), (rows, 2, rows, dst), e.transpose(2, 0, 1)
    img, want = np.ascontiguousarray(img).reshape(-1), np.ascontiguousarray(want).reshape(-1)
    assert np.array_equal(rz.resize(img, *geom, bpp - 1, 1), want)
    got, _ = counted(gpu_ctx, [img], geom, bpp, 1, off=1, out_off=67)
    assert np.array_equal(got[0], want), int((got[0] != want).sum())


@pytest.mark.parametrize("bpp", [1, 2, 4])
@pytest.mark.parametrize("r", [2, 4, 6])
@pytest.mark.parametrize("axis", ["x", "y"])
def test_nearest_exact_halves(gpu_ctx, axis, r, bpp):
    """src = r dst: every position (d + 0.5) r - 0.5 lands on r d + r/2 - 1/2 exactly, which rounds up."""
    for d in (1, 7, 48, 1000):
        geom = (r * d, 3, d, 3) if axis == "x" else (3, r * d, 3, d)
        img = ei.noise(*geom[:2], bpp, r * d + bpp)
        idx = ei.nearest_halves(r * d, d)
        a = img.reshape(geom[1], geom[0], bpp)
        want = (a[:, idx] if axis == "x" else a[idx]).reshape(-1)
        assert np.array_equal(rz.resize(img, *geom, bpp - 1, 0), want)
        for off in (0, 1):   # aligned: pixel-wide copies for 2 and 4 bytes per pixel; offset: byte copies
            got, _ = counted(gpu_ctx, [img], geom, bpp, 0, off=off, out_off=64 + off)
            assert np.array_equal(got[0], want), (geom, off)


# ---- queued tables ------------------------------------------------------------------------------------
def test_queued_lanczos_tables_reuse_the_upload_buffers():
    """Four Lanczos3 calls, each with larger tables than the one before, queued behind a delay on the
    caller's stream with no host synchronisation.  Calls 3 and 4 rewrite the pinned buffers calls 1 and 2
    uploaded from, and every call's tables overwrite the device tables the one before reads: each output
    is the oracle's only if every upload and every kernel ran in order.  A context warmed with larger
    tables and intermediate on both buffers grows nothing, so nothing synchronises for scratch."""
    geoms = [(64, 48, 97, 61, 3), (256, 256, 300, 200, 2), (640, 480, 1000, 700, 0), (1297, 35, 2500, 900, 3)]
    cases = [resize_case(sw, sh, dw, dh, ct, 2, seed=20 + i) for i, (sw, sh, dw, dh, ct) in enumerate(geoms)]
    sizes = [sum(x.nbytes for x in rz.contrib(sw, dw) + rz.contrib(sh, dh)) for sw, sh, dw, dh, _ in geoms]
    assert sizes == sorted(sizes) and len(set(sizes)) == len(sizes)
    ctx, s = Context(0), torch.cuda.Stream()
    try:
        ctx.set_stream(s.cuda_stream)
        warm = resize_case(1400, 1000, 2600, 1000, 3, 2, seed=19)
        torch.cuda.synchronize()
        for _ in range(2):
            for _, fn in warm.calls:
                _lib.check(ctx.handle, fn(ctx))
        s.synchronize()
        torch.cuda.synchronize()
        sleep_on(s, DELAY)
        delayed = torch.cuda.Event()
        delayed.record(s)
        with torch.cuda.stream(s):
            for c in cases:
                for dst, src in c.stage:
                    dst.copy_(src)
        for i, c in enumerate(cases):
            for _, fn in c.calls:
                _lib.check(ctx.handle, fn(ctx))
            if i < 2:
                assert not delayed.query(), f"call {i + 1} waited for the stream"
        with torch.cuda.stream(s):
            res = [[o.clone() for o in c.outs] for c in cases]
        s.synchronize()
        for c, r in zip(cases, res):
            c.check([x.cpu().numpy() for x in r], c.host)
        assert ctx.host_fallbacks == 0
    finally:
        s.synchronize()
        ctx.close()
