"""pixo_b200_jpeg_encode_dev_progressive: device frames to pixo's progressive scans, queued on the context's
stream.  Every file here is pixo_b200_jpeg_progressive_file(the frame's DHT block, its slot, its 7 lengths),
compared byte for byte with real pixo output, with pixo_b200_jpeg_encode_progressive_batch and with the
oracle; no frame may be finished by the host coder."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import jpeg_progressive as jp
from pixo_b200 import ColorType, Context, _lib, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from progressive_inputs import make_progressive_input
from test_dev_layouts_gpu import GUARD8, GUARD32, GUARD64, assert_guard, guarded, jpeg_frames, placed, stripes
from test_jpeg_encode_dev_opts_gpu import big_frames, opts_case
from test_stream_contract_gpu import (DELAY, Case, P, jpeg_frame, lane, poisoned, resize_case, run_case,  # noqa: F401
                                      sleep_on)
from trellis_inputs import make_trellis_input

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DHT = jpeg.DHT_BYTES
NO_FIT = 1


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was finished by the host entropy coder"


@pytest.fixture(scope="module", autouse=True)
def _oracle():
    jp.build()


def opts(w, h, ct, q, ss, ri=0, opt=1, trellis=1):
    return JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), ri or None, bool(opt), True, bool(trellis))


def cap_for(w, h, ct):
    return (2 * w * h * (3 if ct == 2 else 1) + 8192 + 15) // 16 * 16


def run(ctx, frames, o, cap=None, with_dht=True):
    """frames (n equal-size uint8 arrays) -> (slots [n, cap], DHT blocks, lengths [n, 7], flags [n])."""
    n, flen = len(frames), frames[0].size
    cap = cap or cap_for(o.width, o.height, int(o.color_type))
    d_px = torch.from_numpy(np.stack(frames)).cuda()
    out = torch.empty(n * cap, dtype=torch.uint8, device="cuda")
    lens = torch.full((n, 7), -1, dtype=torch.int64, device="cuda")
    ovf = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    dht = torch.empty((n, DHT), dtype=torch.uint8, device="cuda") if with_dht else None
    torch.cuda.synchronize()
    jpeg.encode_progressive_dev(d_px, flen, n, o, out, cap, lens, ovf, dht, ctx=ctx)
    ctx.sync()
    return (out.cpu().numpy().reshape(n, cap), None if dht is None else dht.cpu().numpy(), lens.cpu().numpy(),
            ovf.cpu().numpy())


def files_of(o, slots, tabs, lens, ovf):
    assert not ovf.any(), ovf[ovf != 0][:8]
    return [jpeg.progressive_file(o, None if tabs is None else tabs[i], slots[i], lens[i]) for i in range(len(slots))]


def encode(ctx, frames, o, cap=None):
    return files_of(o, *run(ctx, frames, o, cap))


def oracle(f, o):
    return jp.encode(f, o.width, o.height, int(o.color_type), int(o.subsampling), o.quality, o.restart_interval or 0,
                     o.optimize_huffman, o.trellis_quant)


# ---- real pixo -------------------------------------------------------------------------------------------
def _manifest(sub):
    with open(os.path.join(GOLD, sub, "manifest.json")) as f:
        return json.load(f)["jpeg"]


@pytest.mark.parametrize("e", _manifest("trellis"), ids=lambda e: e["file"])
def test_pixo_max_preset_goldens(gpu_ctx, e):
    img = make_trellis_input(e["kind"], e["w"], e["h"], 1 if e["ct"] == 0 else 3, e["seed"])
    assert hashlib.sha256(img.tobytes()).hexdigest() == e["input_sha256"]
    o = opts(e["w"], e["h"], e["ct"], e["q"], e["s420"])
    assert encode(gpu_ctx, [img], o)[0] == open(os.path.join(GOLD, "trellis", e["file"]), "rb").read()


@pytest.mark.parametrize("e", _manifest("progressive"), ids=lambda e: e["file"])
def test_eob_run_fixtures(gpu_ctx, e):
    o = opts(e["w"], e["h"], e["ct"], e["q"], e["s420"])
    assert encode(gpu_ctx, [make_progressive_input(e)], o)[0] == \
        open(os.path.join(GOLD, "progressive", e["file"]), "rb").read()


# ---- the option matrix against the host batch call and the oracle --------------------------------------------
@pytest.mark.parametrize("ri", [0, 5, 60000])
@pytest.mark.parametrize("opt,trellis", [(1, 1), (1, 0), (0, 1), (0, 0)])
@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
def test_option_matrix(po, gpu_ctx, ct, ss, opt, trellis, ri):
    for w, h in ((1, 1), (17, 9), (333, 217), (1297, 35)):
        for q in (1, 50, 100):
            o = opts(w, h, ct, q, ss, ri, opt, trellis)
            frames = jpeg_frames(po, w, h, ct, 2, 5 * w + q)
            got = encode(gpu_ctx, frames, o)
            assert got == jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx), (w, h, q)
            assert got[0] == oracle(frames[0], o), (w, h, q)


# ---- batches ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 17, 300])
def test_batch_frames_get_their_own_tables(po, gpu_ctx, n):
    w, h = 72, 40
    for ct, ss, ri in ((2, 1, 0), (2, 0, 3), (0, 0, 0)):
        o = opts(w, h, ct, 85, ss, ri)
        frames = jpeg_frames(po, w, h, ct, n, 13 * n + ct)
        slots, tabs, lens, ovf = run(gpu_ctx, frames, o)
        got = files_of(o, slots, tabs, lens, ovf)
        assert got == jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx), (ct, ss)
        for i in sorted({0, n // 2, n - 1}):
            assert got[i] == oracle(frames[i], o), (ct, ss, i)
        assert len({t.tobytes() for t in tabs}) >= min(n, 4), "the frames were meant to differ in their tables"


def test_several_scratch_passes(po, gpu_ctx):
    """A 32 MiB slot per frame puts 15 frames in a pass: 40 frames take three, with three times the launches."""
    w, h = 64, 48
    o = opts(w, h, 2, 80, 1, 2)
    frames = jpeg_frames(po, w, h, 2, 40, 9)
    before = gpu_ctx.launch_count
    got = encode(gpu_ctx, frames, o, cap=32 << 20)
    assert gpu_ctx.launch_count - before == 3 * LAUNCHES[(2, 1, 1)]
    assert got == jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx)


def test_more_frames_than_one_splice_grid(po, gpu_ctx):
    """8 200 small frames: two passes, the second past the splice grid's 8 192 rows."""
    w, h, n = 8, 8, 8200
    rng = np.random.default_rng(5)
    frames = list(rng.integers(0, 256, (n, w * h * 3), dtype=np.uint8))
    o = opts(w, h, 2, 75, 1)
    got = encode(gpu_ctx, frames, o, cap=4096)
    assert got == jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx)


# ---- full size -------------------------------------------------------------------------------------------------
def test_32_4k_frames_max_preset(po, gpu_ctx):
    w, h = 3840, 2160
    o = opts(w, h, 2, 80, 1)
    frames = big_frames(po, w, h, range(32), 400)
    slots, tabs, lens, ovf = run(gpu_ctx, frames, o, cap=(w * h * 3 // 2 + 65536) // 16 * 16)
    got = files_of(o, slots, tabs, lens, ovf)
    sample = [0, 13, 31]
    want = jpeg.encode_progressive_batch(np.stack([frames[i] for i in sample]), o, ctx=gpu_ctx)
    for k, i in enumerate(sample):
        assert got[i] == want[k], i
    assert len({t.tobytes() for t in tabs}) > 1


def test_16k_frame(po, gpu_ctx):
    w = h = 16384
    f = big_frames(po, w, h, [3], 500)[0]
    o = opts(w, h, 2, 80, 1)
    got = encode(gpu_ctx, [f], o, cap=(w * h * 3 // 2 + 65536) // 16 * 16)[0]
    assert hashlib.sha256(got).hexdigest() == hashlib.sha256(jpeg.encode_progressive(f, o, ctx=gpu_ctx)).hexdigest()


# ---- capacity ----------------------------------------------------------------------------------------------
def run_placed(ctx, frames, o, px_off, px_pad, cap, out_off=64, fill=stripes):
    """frames at pixel offset px_off, px_pad bytes between them (the gap from `fill`), every output inside
    guards; returns (slots, DHT blocks, lengths, flags) after checking the guards."""
    n, flen = len(frames), frames[0].size
    src = placed(frames, px_off, flen + px_pad, fill)
    out = guarded(n * cap, np.uint8, GUARD8, base=out_off)
    dht = guarded(n * DHT, np.uint8, GUARD8, base=19, tail=16)
    lens = guarded(n * 7, np.int64, GUARD64, base=2, tail=2)
    ovf = guarded(n, np.int32, GUARD32, base=2, tail=2)
    torch.cuda.synchronize()
    jpeg.encode_progressive_dev(src.ptr(px_off), flen + px_pad, n, o, out.ptr(out_off), cap, lens.ptr(2), ovf.ptr(2),
                                dht.ptr(19), ctx=ctx)
    ctx.sync()
    s, d, ln, ov = out.get(), dht.get(), lens.get(), ovf.get()
    assert_guard(s, [(out_off, n * cap)], GUARD8, "d_out")
    assert_guard(d, [(19, n * DHT)], GUARD8, "d_dht")
    assert_guard(ln, [(2, n * 7)], GUARD64, "d_scan_len")
    assert_guard(ov, [(2, n)], GUARD32, "d_overflow")
    return (s[out_off:out_off + n * cap].reshape(n, cap), d[19:19 + n * DHT].reshape(n, DHT),
            ln[2:2 + 7 * n].reshape(n, 7), ov[2:2 + n])


def test_frames_that_do_not_fit(po, gpu_ctx):
    """Flat and noise frames in one batch: the noise ones do not fit, keep their guard-filled slots and report
    lengths whose sum is enough; the flat ones are right.  A second call with that sum fits every frame."""
    w, h = 256, 128
    rng = np.random.default_rng(3)
    flat = [np.full(w * h * 3, v, np.uint8) for v in (40, 200)]
    noise = [rng.integers(0, 256, w * h * 3, dtype=np.uint8) for _ in range(2)]
    frames = [flat[0], noise[0], flat[1], noise[1]]
    o = opts(w, h, 2, 95, 0, 0, 1, 0)
    want = jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx)
    cap = 4096
    slots, tabs, lens, ovf = run_placed(gpu_ctx, frames, o, 0, 0, cap)
    for i in (0, 2):
        assert ovf[i] == 0 and jpeg.progressive_file(o, tabs[i], slots[i], lens[i]) == want[i], i
    for i in (1, 3):
        assert ovf[i] == NO_FIT, ovf[i]
        assert (slots[i] == GUARD8).all(), "a frame that did not fit wrote into its slot"
    cap2 = (int(lens.sum(1).max()) + 15) // 16 * 16
    slots, tabs, lens, ovf = run_placed(gpu_ctx, frames, o, 0, 0, cap2)
    assert not ovf.any()
    assert [jpeg.progressive_file(o, tabs[i], slots[i], lens[i]) for i in range(4)] == want


def test_stuffed_bytes_decide_the_fit(po, gpu_ctx):
    """A slot between a frame's raw bytes and its stuffed bytes: bit 0, the exact lengths, nothing written."""
    w, h = 64, 64
    f = np.random.default_rng(8).integers(0, 256, w * h * 3, dtype=np.uint8)
    o = opts(w, h, 2, 100, 0, 0, 0, 0)
    slots, tabs, lens, ovf = run(gpu_ctx, [f], o)
    want = files_of(o, slots, tabs, lens, ovf)[0]
    body = int(lens[0].sum())
    stuffed = int((slots[0][:body] == 0xFF).sum())   # one 0x00 follows every 0xFF
    assert stuffed >= 8, "the frame was meant to hold stuffed bytes"
    cap = (body - stuffed // 2) // 4 * 4
    s2, _, l2, ov2 = run_placed(gpu_ctx, [f], o, 0, 0, cap)
    assert ov2[0] == NO_FIT and l2[0].tolist() == lens[0].tolist() and (s2[0] == GUARD8).all()
    s3, t3, l3, ov3 = run_placed(gpu_ctx, [f], o, 0, 0, (body + 3) // 4 * 4)
    assert ov3[0] == 0 and jpeg.progressive_file(o, t3[0], s3[0], l3[0]) == want


# ---- layouts -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
def test_layouts(po, gpu_ctx, ct, ss):
    """Differing frames at odd pixel offsets and strides (poisoned gaps), outputs at odd offsets in guards."""
    w, h = 530, 41
    frames = jpeg_frames(po, w, h, ct, 3, 3 * w)
    o = opts(w, h, ct, 80, ss, 4)
    refs = jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx)
    cap = max(len(r) for r in refs) + 3
    for px_off, px_pad, out_off in ((0, 0, 64), (3, 0, 7), (0, 5, 1), (5, 4099, 13)):
        slots, tabs, lens, ovf = run_placed(gpu_ctx, frames, o, px_off, px_pad, cap, out_off, fill=GUARD8)
        assert not ovf.any(), (px_off, px_pad)
        for i, r in enumerate(refs):
            assert jpeg.progressive_file(o, tabs[i], slots[i], lens[i]) == r, (px_off, px_pad, i)


def test_without_dht_the_standard_tables(po, gpu_ctx):
    w, h = 100, 75
    frames = jpeg_frames(po, w, h, 2, 2, 1)
    o = opts(w, h, 2, 80, 1, 0, 0, 1)
    slots, _, lens, ovf = run(gpu_ctx, frames, o, with_dht=False)
    assert files_of(o, slots, None, lens, ovf) == jpeg.encode_progressive_batch(np.stack(frames), o, ctx=gpu_ctx)


def test_refused_before_any_launch(gpu_ctx):
    lib = _lib.load()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    call = lambda px=p, n=1, w=8, q=80, ri=0, out=p, lens=p, ovf=p, ct=2: \
        lib.pixo_b200_jpeg_encode_dev_progressive(gpu_ctx.handle, px, 192, n, w, 8, ct, q, 1, ri, 1, 1, out, 1024,
                                                  lens, ovf, p + 8192)
    before = gpu_ctx.launch_count
    assert call(q=0) == _lib.ERR_INVALID_QUALITY
    assert call(ri=65536) == _lib.ERR_INVALID_RESTART
    assert call(w=0) == _lib.ERR_INVALID_DIMENSIONS
    assert call(ct=3) == _lib.ERR_UNSUPPORTED_COLOR
    assert call(px=None) == _lib.ERR_INVALID_ARGUMENT
    assert call(out=None) == _lib.ERR_INVALID_ARGUMENT
    assert call(lens=None) == _lib.ERR_INVALID_ARGUMENT
    assert call(ovf=None) == _lib.ERR_INVALID_ARGUMENT
    assert call(n=65536) == _lib.ERR_INVALID_ARGUMENT
    assert call(lens=p + 4) == _lib.ERR_INVALID_ARGUMENT
    assert call(ovf=p + 2) == _lib.ERR_INVALID_ARGUMENT
    assert call(n=0) == _lib.OK
    assert lib.pixo_b200_jpeg_encode_dev_progressive(None, p, 192, 1, 8, 8, 2, 80, 1, 0, 1, 1, p, 1024, p, p,
                                                     None) == _lib.ERR_INVALID_ARGUMENT
    assert gpu_ctx.launch_count == before


# ---- launches per pass ---------------------------------------------------------------------------------------
# (ct, optimize, trellis) -> launches of a one-pass call: the transform (for the statistics or the plain
# coefficients), K3, k_huff_tables, COEF_TRELLIS (its DCT transform and one k_trellis per component), then the
# progressive stage's twelve (k_prog_dht_tables, four measuring kernels, k_prog_place, k_prog_emit_at, five splice)
LAUNCHES = {(2, 1, 1): 19, (2, 1, 0): 15, (2, 0, 1): 17, (2, 0, 0): 14, (0, 1, 1): 17, (0, 0, 0): 14}


@pytest.mark.parametrize("ct,opt,trellis", list(LAUNCHES))
def test_launch_count(po, ct, opt, trellis):
    ctx = Context(0)
    try:
        frames = jpeg_frames(po, 96, 64, ct, 2, 1)
        o = opts(96, 64, ct, 80, 1 if ct else 0, 0, opt, trellis)
        run(ctx, frames, o)   # scratch allocated
        before = ctx.launch_count
        got = encode(ctx, frames, o)
        assert ctx.launch_count - before == LAUNCHES[(ct, opt, trellis)]
        assert got == [oracle(f, o) for f in frames]
    finally:
        ctx.close()


# ---- stream contract ----------------------------------------------------------------------------------------
def dev_progressive_case(po, w, h, ct, ss, ri, opt, trellis, seed=70):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    o = opts(w, h, ct, 80, ss, ri, opt, trellis)
    want = oracle(real, o)
    cap = (len(want) + 64 + 15) // 16 * 16
    px = c.input(real, stale)
    out = c.out(poisoned(cap))
    lens = c.out(poisoned(7, torch.int64, -1))
    ovf = c.out(poisoned(1, torch.int32, -1))
    dht = c.out(poisoned(DHT))
    c.call("jpeg_encode_dev_progressive", lambda ctx: _lib.load().pixo_b200_jpeg_encode_dev_progressive(
        ctx.handle, P(px), real.size, 1, w, h, ct, 80, ss, ri, opt, trellis, P(out), cap, P(lens), P(ovf), P(dht)))

    def check(res, _):
        assert int(res[2][0]) == 0, int(res[2][0])
        assert jpeg.progressive_file(o, res[3], res[0], res[1]) == want
    c.check = check
    return c


STREAM_CASES = [(640, 480, 2, 1, 0, 1, 1), (333, 222, 2, 0, 5, 1, 0), (257, 129, 0, 0, 3, 0, 1), (200, 75, 2, 1, 2, 0, 0)]


@pytest.mark.parametrize("w,h,ct,ss,ri,opt,trellis", STREAM_CASES)
def test_ordered_on_the_callers_stream(po, lane, w, h, ct, ss, ri, opt, trellis):
    ctx, s = lane
    run_case(ctx, s, dev_progressive_case(po, w, h, ct, ss, ri, opt, trellis))


@pytest.mark.parametrize("w,h,ct,ss,ri,opt,trellis", STREAM_CASES)
def test_returns_with_its_work_queued(po, lane, w, h, ct, ss, ri, opt, trellis):
    """On a context warmed with the same geometry, the call returns while the delay before it still runs."""
    ctx, s = lane
    c = dev_progressive_case(po, w, h, ct, ss, ri, opt, trellis)
    run_case(ctx, s, c, delay=False)
    busy = run_case(ctx, s, c, probe=True)
    assert busy["jpeg_encode_dev_progressive"], "jpeg_encode_dev_progressive waited for the device"


def mixed_cases(po, seed):
    return [dev_progressive_case(po, 640, 480, 2, 1, 0, 1, 1, seed=seed),
            opts_case(po, 640, 480, 2, 1, 0, 1, seed=seed + 1),
            resize_case(300, 200, 640, 71, 2, 1, seed=seed + 2),
            dev_progressive_case(po, 333, 222, 2, 1, 5, 1, 1, seed=seed + 3),
            opts_case(po, 333, 222, 2, 1, 3, 1, seed=seed + 4),
            dev_progressive_case(po, 640, 480, 0, 0, 0, 0, 1, seed=seed + 5)]


def test_mixed_with_encode_dev_opts_and_resize_on_one_stream(po):
    """Progressive, balanced and resize calls on one context behind one delay, one synchronisation at the end:
    every output is the oracle's, and no call waited for the stream (a first round of the same geometries has
    grown the context's scratch)."""
    ctx, s = Context(0), torch.cuda.Stream()
    try:
        ctx.set_stream(s.cuda_stream)
        for c in mixed_cases(po, 81):
            run_case(ctx, s, c, delay=False)
        cases = mixed_cases(po, 181)
        torch.cuda.synchronize()
        sleep_on(s, 2 * DELAY)
        delayed = torch.cuda.Event()
        delayed.record(s)
        with torch.cuda.stream(s):
            for c in cases:
                for dst, src in c.stage:
                    dst.copy_(src)
        for c in cases:
            for _, fn in c.calls:
                _lib.check(ctx.handle, fn(ctx))
        assert not delayed.query(), "a call waited for the stream"
        with torch.cuda.stream(s):
            res = [[o.clone() for o in c.outs] for c in cases]
        s.synchronize()
        for c, r in zip(cases, res):
            c.check([x.cpu().numpy() for x in r], c.host)
        assert ctx.host_fallbacks == 0
    finally:
        s.synchronize()
        ctx.close()


def test_two_contexts_on_one_gpu(po):
    """Two contexts on their own streams, calls interleaved from one thread: neither disturbs the other."""
    pairs = [(Context(0), torch.cuda.Stream()) for _ in range(2)]
    cases = [[dev_progressive_case(po, 640, 480, 2, 1, 0, 1, 1, seed=90 + 10 * k + j) for j in range(3)]
             for k in range(2)]
    try:
        for k, (ctx, s) in enumerate(pairs):
            ctx.set_stream(s.cuda_stream)
            for c in cases[k]:
                for dst, src in c.stage:
                    dst.copy_(src)
        torch.cuda.synchronize()
        for j in range(3):
            for k, (ctx, s) in enumerate(pairs):
                for _, fn in cases[k][j].calls:
                    _lib.check(ctx.handle, fn(ctx))
        for k, (ctx, s) in enumerate(pairs):
            s.synchronize()
            for c in cases[k]:
                c.check([o.cpu().numpy() for o in c.outs], c.host)
            assert ctx.host_fallbacks == 0
    finally:
        for ctx, s in pairs:
            s.synchronize()
            ctx.close()
