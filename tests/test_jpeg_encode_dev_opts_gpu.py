"""pixo_b200_jpeg_encode_dev_opts: device frames to scan bytes with a restart interval and optimised Huffman
tables built on the GPU (k_huff_tables), and each frame's tables back as a DHT block.  Every file here is
pixo_b200_jpeg_write_headers_dht(the frame's block) + its scan + EOI, compared byte for byte with the
oracle's pixo::jpeg::encode (or with real pixo output), and no frame may be finished by the host coder."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from golden_inputs import make_input
from oracle import jpeg_progressive as jp
from pixo_b200 import ColorType, Context, _lib, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from test_dev_layouts_gpu import GUARD8, GUARD32, GUARD64, assert_guard, guarded, jpeg_frames, placed, stripes
from test_jpeg_headers_dht import dht_from_oracle, oracle_tables
from test_stream_contract_gpu import Case, P, jpeg_frame, lane, poisoned, run_case  # noqa: F401  (lane: fixture)

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DHT = jpeg.DHT_BYTES


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was finished by the host entropy coder"


def opts(w, h, ct, q, ss, ri, opt):
    return JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), ri or None, bool(opt))


def encode(ctx, frames, o, cap=None):
    """frames (n equal-size uint8 arrays) -> (files, DHT blocks [n, 1088], lengths, flags); every frame
    must fit and finish."""
    n, flen = len(frames), frames[0].size
    if cap is None:
        cap = (2 * flen + 8192 + 15) // 16 * 16
    d_px = torch.from_numpy(np.stack(frames)).cuda()
    scan = torch.empty(n * cap, dtype=torch.uint8, device="cuda")
    lens = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    ovf = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    dht = torch.empty((n, DHT), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    jpeg.encode_dev(d_px, flen, n, o, scan, cap, lens, ovf, dht, ctx=ctx)
    ctx.sync()
    ln, ov, tabs = lens.cpu().numpy(), ovf.cpu().numpy(), dht.cpu().numpy()
    assert not ov.any(), ov[ov != 0][:8]
    s = scan.cpu().numpy()
    files = [jpeg.jpeg_file(o, tabs[i], s[i * cap:i * cap + ln[i]]) for i in range(n)]
    return files, tabs, ln, ov


def oracle_file(po, f, o):
    return po.jpeg_encode(f, o.width, o.height, int(o.color_type), o.quality, int(o.subsampling),
                          o.restart_interval or 0, o.optimize_huffman)


def oracle_dht(po, f, o):
    """The tables pixo codes frame f with, as a DHT block, and whether they are the optimised ones."""
    ct, ss = int(o.color_type), int(o.subsampling)
    co = po.jpeg_coefficients(f, o.width, o.height, ct, ss, o.quality)
    hist = po.jpeg_histograms(*co, o.width, o.height, ct, ss, o.restart_interval or 0)
    t, ok = oracle_tables(po, hist, ct != 0)
    return dht_from_oracle(t).reshape(-1), ok, t


# ---- files against the oracle ---------------------------------------------------------------------------
SIZES = [(1, 1), (7, 9), (17, 33), (96, 64), (1297, 35), (640, 480)]


@pytest.mark.parametrize("ct,ss", [(0, 0), (2, 1), (2, 0)])
@pytest.mark.parametrize("opt", [0, 1])
@pytest.mark.parametrize("ri", [0, 1, 5, 60000])
def test_files_match_the_oracle(po, gpu_ctx, ct, ss, opt, ri):
    """Sizes x qualities in one batch per (size, quality); restart 60 000 is longer than every frame."""
    for w, h in SIZES:
        for k, q in enumerate((1, 50, 80, 95, 100)):
            o = opts(w, h, ct, q, ss, ri, opt)
            frames = jpeg_frames(po, w, h, ct, 2, 7 * w + q)[k % 2:k % 2 + 1] + jpeg_frames(po, w, h, ct, 2, q)
            files, tabs, _, _ = encode(gpu_ctx, frames, o)
            for i, f in enumerate(frames):
                assert files[i] == oracle_file(po, f, o), (w, h, q, i)


# ---- batches whose frames have different tables ---------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 17, 300])
def test_batch_frames_get_their_own_tables(po, gpu_ctx, n):
    w, h = 72, 40
    for ct, ss, ri in ((2, 1, 0), (2, 0, 3), (0, 0, 0)):
        o = opts(w, h, ct, 85, ss, ri, 1)
        frames = jpeg_frames(po, w, h, ct, n, 11 * n + ct)
        files, tabs, _, _ = encode(gpu_ctx, frames, o)
        seen = set()
        for i, f in enumerate(frames):
            want, _, _ = oracle_dht(po, f, o)
            assert np.array_equal(tabs[i], want), (ct, ss, i)
            assert files[i] == oracle_file(po, f, o), (ct, ss, i)
            seen.add(tabs[i].tobytes())
        assert len(seen) >= min(n, 4), "the frames were meant to differ in their tables"


# ---- every branch of the table construction ------------------------------------------------------------
def ladder(w, h, ch, seed, chroma_only, ratio):
    """Bands of noise whose height shrinks by `ratio` as its amplitude doubles: symbol counts that fall
    off geometrically, which makes Huffman trees deep.  chroma_only: the noise moves R and B against each
    other and leaves the luma nearly flat."""
    rng = np.random.default_rng(seed)
    img = np.full((h, w, ch), 128, np.int32)
    row, amp, hh = 0, 1, h // 2
    while row < h:
        hh = max(hh, 8) if row + hh < h else h - row
        noise = rng.integers(-amp, amp + 1, (hh, w, ch))
        if chroma_only:
            img[row:row + hh, :, 0] += noise[..., 0]
            img[row:row + hh, :, 2] -= noise[..., 0]
        else:
            img[row:row + hh] += noise
        row, hh, amp = row + hh, max(int(hh * ratio), 8), min(amp * 2, 127)
    return np.clip(img, 0, 255).astype(np.uint8).reshape(-1)


STD = None


def is_standard(po, t, k):
    global STD
    if STD is None:
        STD = po.HuffTables()
        po.lib().po_huff_standard(C.byref(STD))
    return t.nvals[k] == STD.nvals[k] and list(t.bits[k]) == list(STD.bits[k]) and \
        list(t.vals[k])[:t.nvals[k]] == list(STD.vals[k])[:STD.nvals[k]]


def branch_case(po, name):
    if name == "all-optimised":
        return po.gen_noise(64, 64, 3, 5), opts(64, 64, 2, 75, 0, 0, 1)
    if name == "luma-fails-gray":
        return ladder(512, 1024, 1, 1, False, 0.5), opts(512, 1024, 0, 100, 0, 0, 1)
    if name == "luma-fails-rgb":
        return ladder(512, 1024, 3, 1, False, 0.5), opts(512, 1024, 2, 100, 0, 0, 1)
    if name == "one-chroma-fails":
        return ladder(512, 1024, 3, 1, True, 0.6), opts(512, 1024, 2, 100, 0, 0, 1)
    if name == "single-symbol":
        return np.full(64 * 48 * 3, 128, np.uint8), opts(64, 48, 2, 80, 1, 0, 1)
    return po.gen_noise(7, 9, 3, 2), opts(7, 9, 2, 90, 1, 2, 1)   # "ties": a few blocks, equal counts


@pytest.mark.parametrize("name", ["all-optimised", "luma-fails-gray", "luma-fails-rgb", "one-chroma-fails",
                                  "single-symbol", "ties"])
def test_every_table_branch(po, gpu_ctx, name):
    f, o = branch_case(po, name)
    want, ok, t = oracle_dht(po, f, o)
    std = [is_standard(po, t, k) for k in range(4)]
    # the input takes the branch it is named after
    if name == "all-optimised":
        assert ok and not any(std)
    elif name.startswith("luma-fails"):
        assert not ok and all(std)
    elif name == "one-chroma-fails":
        assert ok and std == [False, False, False, True]
    elif name == "single-symbol":
        assert ok and [t.nvals[k] for k in range(4)] == [1, 1, 1, 1] and [t.bits[k][0] for k in range(4)] == [1] * 4
    else:
        co = po.jpeg_coefficients(f, o.width, o.height, 2, 1, o.quality)
        hist = po.jpeg_histograms(*co, o.width, o.height, 2, 1, 2)
        nz = hist[24:280][hist[24:280] > 0]
        assert ok and len(nz) > len(set(nz.tolist()))
    files, tabs, _, _ = encode(gpu_ctx, [f, f], o)
    for i in range(2):
        assert np.array_equal(tabs[i], want), i
        assert files[i] == oracle_file(po, f, o), i
    # the host entry points build their tables with the same kernel
    assert jpeg.encode(f, o, ctx=gpu_ctx) == oracle_file(po, f, o)
    assert jpeg.encode_batch(np.stack([f, f]), o, ctx=gpu_ctx) == [oracle_file(po, f, o)] * 2
    ct, ss = int(o.color_type), int(o.subsampling)
    co = po.jpeg_coefficients(f, o.width, o.height, ct, ss, o.quality)
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() if ct or k == 0 else None for k, a in enumerate(co)]
    torch.cuda.synchronize()
    assert jpeg.entropy_encode_dev(*d, o, ctx=gpu_ctx) == po.jpeg_encode_from_coefficients(
        *co, o.width, o.height, ct, o.quality, ss, o.restart_interval or 0, True)
    jp.build()
    for trellis in (False, True):
        p = JpegOptions(o.width, o.height, o.color_type, o.quality, o.subsampling, o.restart_interval, True, True,
                        trellis)
        assert jpeg.encode_progressive(f, p, ctx=gpu_ctx) == jp.encode(f, o.width, o.height, ct, ss, o.quality,
                                                                        o.restart_interval or 0, True, trellis), trellis


# ---- real pixo: the balanced preset's fixtures ---------------------------------------------------------
BALANCED = [c for c in json.load(open(os.path.join(GOLD, "manifest.json")))["jpeg"] if c["preset"] == 1]


@pytest.mark.parametrize("c", BALANCED, ids=lambda c: c["file"])
def test_balanced_preset_goldens(gpu_ctx, c):
    img = make_input(c["kind"], c["w"], c["h"], 3 if c["ct"] == 2 else 1, c["seed"])
    assert hashlib.sha256(img.tobytes()).hexdigest() == c["input_sha256"]
    o = JpegOptions.from_preset(c["w"], c["h"], c["q"], c["preset"])
    o.color_type = ColorType(c["ct"])
    o.subsampling = Subsampling.S420 if c["s420"] else Subsampling.S444
    files, _, _, _ = encode(gpu_ctx, [img], o)
    assert files[0] == open(os.path.join(GOLD, c["file"]), "rb").read()


def test_balanced_goldens_cover_the_modes():
    assert len(BALANCED) >= 8 and {(c["ct"], c["s420"]) for c in BALANCED} >= {(2, 0), (2, 1), (0, 0)}


# ---- full size --------------------------------------------------------------------------------------------
def big_frames(po, w, h, idx, seed):
    """Differing frames: a gradient rolled by 37 i bytes per row, with a noise band of 16 (i % 7) rows."""
    grad = po.gen_gradient_rgb(w, h).reshape(h, w * 3)
    out = []
    for i in idx:
        f = np.roll(grad, 37 * i, axis=1)
        k = 16 * (i % 7)
        if k:
            f[:k] = po.gen_noise(w, k, 3, seed + i).reshape(k, w * 3)
        out.append(f.reshape(-1))
    return out


def test_32_4k_frames_balanced(po, gpu_ctx):
    w, h = 3840, 2160
    o = opts(w, h, 2, 75, 0, 0, 1)
    frames = big_frames(po, w, h, range(32), 100)
    files, tabs, _, _ = encode(gpu_ctx, frames, o, cap=(w * h * 3 + 65536) // 16 * 16)
    for i in (0, 5, 31):
        assert files[i] == oracle_file(po, frames[i], o), i
    assert len({t.tobytes() for t in tabs}) > 1


def test_16k_frame_segmented_with_its_own_tables(po, gpu_ctx):
    """One 16 384^2 frame is coded in segments (k_huff<RAW>) and spliced; with its optimised tables."""
    w = h = 16384
    f = big_frames(po, w, h, [1], 200)[0]
    o = opts(w, h, 2, 80, 1, 0, 1)
    files, _, _, _ = encode(gpu_ctx, [f], o, cap=(w * h * 3 // 2 + 65536) // 16 * 16)
    assert hashlib.sha256(files[0]).hexdigest() == hashlib.sha256(oracle_file(po, f, o)).hexdigest()


def test_256_1080p_frames_restart_8(po, gpu_ctx):
    w, h = 1920, 1080
    o = opts(w, h, 2, 80, 1, 8, 1)
    frames = big_frames(po, w, h, range(256), 300)
    files, _, _, _ = encode(gpu_ctx, frames, o, cap=(w * h * 3 // 2 + 65536) // 16 * 16)
    for i in (0, 129, 255):
        assert files[i] == oracle_file(po, frames[i], o), i


# ---- layouts and limits -----------------------------------------------------------------------------------
def encode_placed(ctx, frames, o, px_off, px_pad, cap):
    n, flen = len(frames), frames[0].size
    src = placed(frames, px_off, flen + px_pad, stripes)
    scan = guarded(n * cap, np.uint8, GUARD8)
    dht = guarded(n * DHT, np.uint8, GUARD8, base=16 + 3, tail=16)
    lens = guarded(n, np.int64, GUARD64, base=2, tail=2)
    ovf = guarded(n, np.int32, GUARD32, base=2, tail=2)
    torch.cuda.synchronize()
    jpeg.encode_dev(src.ptr(px_off), flen + px_pad, n, o, scan.ptr(64), cap, lens.ptr(2), ovf.ptr(2),
                    dht.ptr(19), ctx=ctx)
    ctx.sync()
    s, d, ln, ov = scan.get(), dht.get(), lens.get(), ovf.get()
    assert_guard(s, [(64, n * cap)], GUARD8, "scan slots")
    assert_guard(d, [(19, n * DHT)], GUARD8, "d_dht")
    assert_guard(ln, [(2, n)], GUARD64, "d_scan_len")
    assert_guard(ov, [(2, n)], GUARD32, "d_overflow")
    return ([s[64 + i * cap:64 + (i + 1) * cap] for i in range(n)], d[19:19 + n * DHT].reshape(n, DHT),
            ln[2:2 + n], ov[2:2 + n])


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)])
def test_layouts(po, gpu_ctx, ct, ss):
    """Differing frames at odd pixel offsets and strides, in slots whose size is 4 (mod 16)."""
    w, h = 530, 41
    frames = jpeg_frames(po, w, h, ct, 3, 3 * w)
    o = opts(w, h, ct, 80, ss, 4, 1)
    refs = [oracle_file(po, f, o) for f in frames]
    cap = (max(len(r) for r in refs) + 64 + 15) // 16 * 16 + 4
    for px_off, px_pad in ((0, 0), (3, 0), (0, 5), (5, 4099)):
        slots, tabs, lens, ovf = encode_placed(gpu_ctx, frames, o, px_off, px_pad, cap)
        for i, r in enumerate(refs):
            assert ovf[i] == 0, (px_off, px_pad, i)
            assert jpeg.jpeg_file(o, tabs[i], slots[i][:lens[i]]) == r, (px_off, px_pad, i)


def test_too_small_slot_reports_the_needed_length(po, gpu_ctx):
    w, h = 256, 256
    frames = [po.gen_gradient_rgb(w, h), po.gen_noise(w, h, 3, 4)]
    o = opts(w, h, 2, 90, 1, 7, 1)
    refs = [oracle_file(po, f, o) for f in frames]
    hdr = [len(jpeg.write_headers_dht(o, oracle_dht(po, f, o)[0])) for f in frames]
    need = [len(r) - hl - 2 for r, hl in zip(refs, hdr)]
    cap = (need[0] + 15) // 16 * 16 + 4
    assert need[1] > cap
    slots, tabs, lens, ovf = encode_placed(gpu_ctx, frames, o, 0, 0, cap)
    assert ovf[0] == 0 and ovf[1] & 1 and lens.tolist() == need
    assert jpeg.jpeg_file(o, tabs[0], slots[0][:lens[0]]) == refs[0]
    cap = (int(lens[1]) + 15) // 16 * 16
    slots, tabs, lens, ovf = encode_placed(gpu_ctx, frames, o, 0, 0, cap)
    assert not ovf.any()
    assert [jpeg.jpeg_file(o, tabs[i], slots[i][:lens[i]]) for i in range(2)] == refs


def test_limits_and_options(gpu_ctx):
    lib = _lib.load()
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    before = gpu_ctx.launch_count
    assert lib.pixo_b200_jpeg_encode_dev_opts(gpu_ctx.handle, p, 0, 65536, 8, 8, 2, 80, 1, 0, 1, p, 1024, p, p,
                                              p) == _lib.ERR_INVALID_ARGUMENT
    assert lib.pixo_b200_jpeg_encode_dev_opts(gpu_ctx.handle, p, 192, 1, 8, 8, 2, 80, 1, 65536, 1, p, 1024, p, p,
                                              p) == _lib.ERR_INVALID_RESTART
    assert lib.pixo_b200_jpeg_encode_dev_opts(gpu_ctx.handle, p, 192, 1, 8, 8, 2, 0, 1, 65536, 1, p, 1024, p, p,
                                              p) == _lib.ERR_INVALID_QUALITY
    assert lib.pixo_b200_jpeg_encode_dev_opts(gpu_ctx.handle, p, 192, 1, 8, 8, 2, 80, 1, 0, 1, p + 4, 1024, p, p,
                                              p) == _lib.ERR_INVALID_ARGUMENT
    assert lib.pixo_b200_jpeg_encode_dev_opts(gpu_ctx.handle, p, 192, 0, 8, 8, 2, 80, 1, 0, 1, p, 1024, p, p,
                                              None) == _lib.OK
    assert gpu_ctx.launch_count == before
    with pytest.raises(_lib.PixoError) as e:
        jpeg.encode_dev(buf, 192, 1, JpegOptions(8, 8, progressive=True), buf, 1024, buf, buf, ctx=gpu_ctx)
    assert e.value.code == _lib.ERR_UNSUPPORTED


@pytest.mark.parametrize("opt,with_dht,launches", [(1, True, 4), (1, False, 4), (0, False, 2), (0, True, 3)])
def test_launch_count(po, opt, with_dht, launches):
    """transform, K3, k_huff_tables, k_huff with optimisation; transform and k_huff without (k_huff_tables
    only writes the standard blocks when they are asked for)."""
    ctx = Context(0)
    try:
        f = po.gen_noise(96, 64, 3, 1)
        o = opts(96, 64, 2, 80, 1, 0, opt)
        d_px = torch.from_numpy(f).cuda()
        scan = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
        lens = torch.empty(1, dtype=torch.int64, device="cuda")
        ovf = torch.empty(1, dtype=torch.int32, device="cuda")
        dht = torch.empty(DHT, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        before = ctx.launch_count
        jpeg.encode_dev(d_px, f.size, 1, o, scan, 1 << 16, lens, ovf, dht if with_dht else None, ctx=ctx)
        ctx.sync()
        assert ctx.launch_count - before == launches
        assert int(ovf[0]) == 0
        if with_dht:
            assert jpeg.jpeg_file(o, dht.cpu().numpy(), scan[:int(lens[0])].cpu().numpy()) == oracle_file(po, f, o)
    finally:
        ctx.close()


# ---- stream contract ------------------------------------------------------------------------------------
def opts_case(po, w, h, ct, ss, ri, opt, seed=60):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    o = opts(w, h, ct, 80, ss, ri, opt)
    want = oracle_file(po, real, o)
    cap = (len(want) + 64 + 15) // 16 * 16
    px = c.input(real, stale)
    scan = c.out(poisoned(cap))
    n = c.out(poisoned(1, torch.int64, -1))
    ovf = c.out(poisoned(1, torch.int32, -1))
    dht = c.out(poisoned(DHT))
    c.call("jpeg_encode_dev_opts", lambda ctx: _lib.load().pixo_b200_jpeg_encode_dev_opts(
        ctx.handle, P(px), real.size, 1, w, h, ct, 80, ss, ri, opt, P(scan), cap, P(n), P(ovf), P(dht)))

    def check(out, _):
        assert int(out[2][0]) == 0, int(out[2][0])
        assert jpeg.jpeg_file(o, out[3], out[0][:int(out[1][0])]) == want
    c.check = check
    return c


STREAM_CASES = [(640, 480, 2, 1, 0, 1), (333, 222, 2, 0, 5, 1), (257, 129, 0, 0, 3, 1), (200, 75, 2, 1, 2, 0)]


@pytest.mark.parametrize("w,h,ct,ss,ri,opt", STREAM_CASES)
def test_ordered_on_the_callers_stream(po, lane, w, h, ct, ss, ri, opt):
    """The real input is copied over a stale one on S behind a delay; the output is the real frame's."""
    ctx, s = lane
    run_case(ctx, s, opts_case(po, w, h, ct, ss, ri, opt))


@pytest.mark.parametrize("w,h,ct,ss,ri,opt", STREAM_CASES)
def test_returns_with_its_work_queued(po, lane, w, h, ct, ss, ri, opt):
    """On a context warmed with the same geometry, the call returns while the delay before it still runs."""
    ctx, s = lane
    c = opts_case(po, w, h, ct, ss, ri, opt)
    run_case(ctx, s, c, delay=False)
    busy = run_case(ctx, s, c, probe=True)
    assert busy["jpeg_encode_dev_opts"], "jpeg_encode_dev_opts waited for the device"
