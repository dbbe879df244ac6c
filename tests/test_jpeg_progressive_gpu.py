"""Progressive JPEGs on the GPU (pixo_b200_jpeg_encode_progressive[_batch], progressive_scans_dev) against
real pixo max-preset files (tests/golden/trellis/, tests/golden/progressive/), the C restatement
oracle/jpeg_progressive.c and the scan restatement tests/jpeg_progressive_scans.py.  No frame is finished
by host code."""
import hashlib
import json
import os

import numpy as np
import pytest

import jpeg_progressive_scans as ps
from golden_inputs import make_input
from oracle import jpeg_progressive as jp
from oracle import jpeg_trellis as jt
from progressive_inputs import make_progressive_input
from trellis_inputs import make_trellis_input

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trellis")
GOLDEN_P = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "progressive")
with open(os.path.join(GOLDEN, "manifest.json")) as _f:
    MANIFEST = json.load(_f)["jpeg"]
with open(os.path.join(GOLDEN_P, "manifest.json")) as _f:
    MANIFEST_P = json.load(_f)["jpeg"]


@pytest.fixture(scope="module", autouse=True)
def oracles_built(po):
    jt.build()
    jp.build()


@pytest.fixture(autouse=True)
def no_host_fallback(gpu_ctx):
    from pixo_b200 import _lib
    yield
    assert _lib.load().pixo_b200_ctx_host_fallbacks(gpu_ctx.handle) == 0


def _opts(w, h, ct, ss, q, restart=None, optimize=True, trellis=True):
    from pixo_b200 import ColorType, jpeg
    return jpeg.JpegOptions(w, h, ColorType(ct), q, jpeg.Subsampling(ss), restart, optimize, True, trellis)


def _golden(e):
    img = make_trellis_input(e["kind"], e["w"], e["h"], 1 if e["ct"] == 0 else 3, e["seed"])
    with open(os.path.join(GOLDEN, e["file"]), "rb") as f:
        return img, f.read()


@pytest.mark.parametrize("e", MANIFEST, ids=lambda e: e["file"])
def test_encode_progressive_equals_pixo_max_files(gpu_ctx, e):
    from pixo_b200 import jpeg
    img, want = _golden(e)
    got = jpeg.encode_progressive(img, _opts(e["w"], e["h"], e["ct"], e["s420"], e["q"]), ctx=gpu_ctx)
    assert got == want


@pytest.mark.parametrize("e", MANIFEST_P, ids=lambda e: e["file"])
def test_progressive_fixtures_with_0x7fff_runs(gpu_ctx, e):
    """encode_progressive and progressive_scans_dev (oracle coefficients, the file's tables) against pixo's
    files whose Y AC scans hold EOB runs of 32 766 - 69 999 blocks."""
    from pixo_b200 import ColorType, jpeg
    img = make_progressive_input(e)
    with open(os.path.join(GOLDEN_P, e["file"]), "rb") as f:
        want = f.read()
    assert jpeg.encode_progressive(img, _opts(e["w"], e["h"], e["ct"], e["s420"], e["q"]), ctx=gpu_ctx) == want
    y, cb, cr = jt.jpeg_coefficients(img, e["w"], e["h"], e["ct"], e["s420"], e["q"])
    cap = len(want) + 4096
    r = jpeg.progressive_scans_dev(_dev(y), _dev(cb), _dev(cr), e["w"], e["h"], ColorType(e["ct"]),
                                   jpeg.Subsampling(e["s420"]), tables=ps.dht(want), out_cap_each=cap, ctx=gpu_ctx)
    assert _segments(*r, cap)[0] == [s[5] for s in ps.scans(want)]


def _dev(a):
    import torch
    a = np.ascontiguousarray(a, np.int16).reshape(-1, 64)
    return torch.from_numpy(a if len(a) else np.zeros((1, 64), np.int16)).cuda()


def _segments(d_out, d_len, d_ovf, cap, n=1):
    out = d_out.cpu().numpy()
    lens = d_len.cpu().numpy().reshape(n, 7)
    ovf = d_ovf.cpu().numpy()
    res = []
    for i in range(n):
        assert ovf[i] == 0
        o, segs = i * cap, []
        for s in range(7):
            segs.append(out[o:o + lens[i, s]].tobytes())
            o += lens[i, s]
        res.append(segs)
    return res


@pytest.mark.parametrize("e", MANIFEST[::3], ids=lambda e: e["file"])
def test_scans_dev_on_oracle_coefficients_equal_pixo_segments(gpu_ctx, e):
    from pixo_b200 import ColorType, jpeg
    img, want = _golden(e)
    y, cb, cr = jt.jpeg_coefficients(img, e["w"], e["h"], e["ct"], e["s420"], e["q"])
    cap = jpeg.progressive_capacity(e["w"], e["h"])
    r = jpeg.progressive_scans_dev(_dev(y), _dev(cb), _dev(cr), e["w"], e["h"], ColorType(e["ct"]),
                                   jpeg.Subsampling(e["s420"]), tables=ps.dht(want), out_cap_each=cap, ctx=gpu_ctx)
    assert _segments(*r, cap)[0] == [s[5] for s in ps.scans(want)]


SIZES = [(1, 1), (7, 9), (15, 17), (16, 16), (17, 15), (255, 257), (1297, 35)]
QUALITIES = [1, 50, 80, 100]
KINDS = ["noise", "smooth", "gradient", "primaries"]


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
@pytest.mark.parametrize("trellis", [True, False], ids=["trellis", "plain"])
@pytest.mark.parametrize("optimize", [True, False], ids=["opt", "std"])
@pytest.mark.parametrize("restart", [None, 5], ids=["norst", "rst5"])
def test_option_matrix_matches_reference(gpu_ctx, ct, ss, trellis, optimize, restart):
    from pixo_b200 import jpeg
    for i, (w, h) in enumerate(SIZES):
        for j, q in enumerate(QUALITIES):
            kind = KINDS[(i + j) % len(KINDS)]
            img = make_trellis_input(kind, w, h, 1 if ct == 0 else 3, 10 * i + j)
            got = jpeg.encode_progressive(img, _opts(w, h, ct, ss, q, restart, optimize, trellis), ctx=gpu_ctx)
            want = jp.encode(img, w, h, ct, ss, q, restart, optimize, trellis)
            assert got == want, (w, h, q, kind)


def test_batch_equals_reference_and_repeats(gpu_ctx):
    from pixo_b200 import jpeg
    w, h, n = 333, 217, 7
    frames = np.stack([make_trellis_input(KINDS[i % 4] if i % 3 else "hifreq", w, h, 3, i) for i in range(n)])
    opts = _opts(w, h, 2, 1, 80)
    got = jpeg.encode_progressive_batch(frames, opts, ctx=gpu_ctx)
    again = jpeg.encode_progressive_batch(frames, opts, ctx=gpu_ctx)
    assert got == again
    for i in range(n):
        assert got[i] == jp.encode(frames[i], w, h, 2, 1, 80), i
        assert got[i] == jpeg.encode_progressive(frames[i], opts, ctx=gpu_ctx)


def test_baseline_entry_still_refuses_progressive(gpu_ctx):
    from pixo_b200 import _lib, jpeg
    img = make_input("noise", 16, 16, 3, 0)
    o = _opts(16, 16, 2, 1, 80)
    with pytest.raises(_lib.PixoError) as ei:
        jpeg.encode(img, o, ctx=gpu_ctx)
    assert ei.value.code == _lib.ERR_UNSUPPORTED


# ---- constructed coefficient arrays on the device entry -----------------------------------------------

def _std_tables(po):
    return ps.dht(po.jpeg_encode(np.zeros(64, np.uint8), 8, 8, 0, 80, 0, 0, False))


def _opt_tables():
    with open(os.path.join(GOLDEN, "t008.jpg"), "rb") as f:
        return ps.dht(f.read())


def _gray_frame(nblocks):
    """(w, h) of a gray frame of exactly nblocks blocks (nblocks = bw * bh)."""
    bw = 1
    for c in (512, 256, 128, 64, 32, 16, 8, 4, 2, 1):
        if nblocks % c == 0:
            bw = c
            break
    return 8 * bw, 8 * (nblocks // bw)


def _run_corpus(gpu_ctx, y, tables, cb=None, cr=None, w=None, h=None, ct=0, ss=0):
    from pixo_b200 import ColorType, jpeg
    if w is None:
        w, h = _gray_frame(len(y))
    empty = np.zeros((0, 64), np.int16)
    cb = empty if cb is None else cb
    cr = empty if cr is None else cr
    cap = (sum(len(s) for s in ps.encode_scans(y, cb, cr, tables)) + 4096 + 15) // 16 * 16
    r = jpeg.progressive_scans_dev(_dev(y), _dev(cb), _dev(cr), w, h, ColorType(ct), jpeg.Subsampling(ss),
                                   tables=tables, out_cap_each=cap, ctx=gpu_ctx)
    assert _segments(*r, cap)[0] == ps.encode_scans(y, cb, cr, tables)


def _runs_blocks(gaps, first_nonempty=True, last_nonempty=False, below_se=True, rng=None):
    """Y blocks: non-empty blocks separated by `gaps` empty ones (in every AC band)."""
    rng = rng or np.random.default_rng(0)
    blocks = []

    def busy(i):
        b = np.zeros(64, np.int16)
        b[0] = int(rng.integers(-50, 50))
        b[ps.ZIGZAG[1]] = 3
        b[ps.ZIGZAG[11]] = -2
        if not below_se or i % 2:
            b[ps.ZIGZAG[10]] = 1
            b[ps.ZIGZAG[63]] = 7
        return b

    k = 0
    if first_nonempty:
        blocks.append(busy(k)); k += 1
    for g in gaps:
        blocks += [np.zeros(64, np.int16)] * g
        blocks.append(busy(k)); k += 1
    if not last_nonempty:
        blocks += [np.zeros(64, np.int16)] * 3
    return np.stack(blocks)


@pytest.mark.parametrize("gaps", [[31, 32, 33, 64, 0, 1], [32766], [32767], [32768]], ids=str)
@pytest.mark.parametrize("ends", [(True, False), (False, True)], ids=["first", "last"])
def test_scans_dev_eob_runs_around_chunks_and_0x7fff(po, gpu_ctx, gaps, ends):
    y = _runs_blocks(gaps, *ends)
    pad = (-len(y)) % 8
    y = np.concatenate([y, np.zeros((pad, 64), np.int16)])
    for tables in (_std_tables(po), _opt_tables()):
        _run_corpus(gpu_ctx, y, tables)


def test_scans_dev_eob_run_crossing_0x7fff_twice(po, gpu_ctx):
    y = _runs_blocks([65534, 65535], True, False, below_se=False)
    y = np.concatenate([y, np.zeros(((-len(y)) % 512, 64), np.int16)])
    _run_corpus(gpu_ctx, y, _std_tables(po))


def test_scans_dev_zrl_big_categories_and_ff_bytes(po, gpu_ctx):
    rng = np.random.default_rng(7)
    n = 4096
    y = np.zeros((n, 64), np.int16)
    for i in range(n):
        kind = i % 5
        if kind == 0:      # ZRL: a long zero run before one value
            y[i, ps.ZIGZAG[1 + int(rng.integers(16, 50))]] = int(rng.integers(1, 30))
        elif kind == 1:    # categories 11..15 (the fallback code) in DC and AC
            y[i, 0] = int(rng.choice([-1, 1])) * int(rng.integers(1024, 16384))
            y[i, ps.ZIGZAG[int(rng.integers(1, 64))]] = int(rng.choice([-1, 1])) * int(rng.integers(1024, 16384))
        elif kind == 2:    # long runs of 1-bits -> 0xFF bytes to stuff
            y[i, ps.ZIGZAG[1:20]] = -1
        elif kind == 3:
            y[i] = rng.integers(-300, 300, 64)
    y[:, 0] = np.where(np.arange(n) % 7 == 0, 16383, y[:, 0])   # DC differences up to 32766
    y[1::14, 0] = -16383
    for tables in (_std_tables(po), _opt_tables()):
        _run_corpus(gpu_ctx, y, tables)


@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0)], ids=["420", "444"])
def test_scans_dev_color_constructed(po, gpu_ctx, ct, ss):
    rng = np.random.default_rng(3)
    w, h = 200, 120
    from pixo_b200 import jpeg
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    mk = lambda n: np.where(rng.random((n, 64)) < 0.05, rng.integers(-40, 40, (n, 64)), 0).astype(np.int16)
    _run_corpus(gpu_ctx, mk(ny), _opt_tables(), mk(nc), mk(nc), w, h, ct, ss)


def test_scans_dev_layouts_and_overflow(gpu_ctx):
    """Padded strides with poison between frames, guarded outputs, exact lengths on overflow."""
    import torch
    from pixo_b200 import ColorType, _lib, jpeg
    w, h, n, pad = 40, 24, 3, 64 * 8
    ny, nc = jpeg.block_counts(w, h, 2, 1)
    rng = np.random.default_rng(1)
    frames = [[np.where(rng.random((k, 64)) < 0.2, rng.integers(-60, 60, (k, 64)), 0).astype(np.int16)
               for k in (ny, nc, nc)] for _ in range(n)]
    tables = _opt_tables()
    want = [ps.encode_scans(*f, tables) for f in frames]
    ys, cs = ny * 64 + pad, nc * 64 + pad

    def packed(comp, stride, nb):
        a = np.full(n * stride, 0x7FFF, np.int16)
        for i in range(n):
            a[i * stride:i * stride + nb * 64] = frames[i][comp].reshape(-1)
        return torch.from_numpy(a).cuda()

    d_y, d_cb, d_cr = packed(0, ys, ny), packed(1, cs, nc), packed(2, cs, nc)
    need = [sum(len(s) for s in segs) for segs in want]
    cap = (max(need) + 64 + 15) // 16 * 16
    guard = 0xA5
    d_out = torch.full((n * cap + 64,), guard, dtype=torch.uint8, device="cuda")
    d_len = torch.full((n + 1, 7), -1, dtype=torch.int64, device="cuda")
    d_ovf = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    jpeg.progressive_scans_dev(d_y, d_cb, d_cr, w, h, ColorType.Rgb, jpeg.Subsampling.S420, tables, n, ys, cs,
                               d_out, cap, d_len, d_ovf, ctx=gpu_ctx)
    assert _segments(d_out[:n * cap], d_len[:n], d_ovf[:n], cap, n) == want
    out = d_out.cpu().numpy()
    for i in range(n):
        assert (out[i * cap + need[i]:(i + 1) * cap] == guard).all()
    assert (out[n * cap:] == guard).all() and (d_len[n] == -1).all() and int(d_ovf[n]) == -1

    # a slot one byte too small for frame 1: nothing written for it, lengths are the sizes needed
    cap2 = (need[1] - 1)
    d_out2 = torch.full((n * cap2,), guard, dtype=torch.uint8, device="cuda")
    jpeg.progressive_scans_dev(d_y, d_cb, d_cr, w, h, ColorType.Rgb, jpeg.Subsampling.S420, tables, n, ys, cs,
                               d_out2, cap2, d_len, d_ovf, ctx=gpu_ctx)
    lens = d_len[:n].cpu().numpy()
    assert [list(map(len, s)) for s in want] == lens.tolist()
    ovf = d_ovf[:n].cpu().numpy()
    assert [int(o) for o in ovf] == [int(need[i] > cap2) for i in range(n)]
    o2 = d_out2.cpu().numpy()
    assert (o2[cap2:2 * cap2] == guard).all()

    # refused before anything runs: misaligned arrays, short strides, out-of-range coefficients, bad tables
    launches = _lib.load().pixo_b200_ctx_launch_count(gpu_ctx.handle)
    bad_calls = [
        lambda: jpeg.progressive_scans_dev(d_y[1:], d_cb, d_cr, w, h, ColorType.Rgb, jpeg.Subsampling.S420, tables,
                                           1, ys, cs, d_out, cap, d_len, d_ovf, ctx=gpu_ctx),
        lambda: jpeg.progressive_scans_dev(d_y, d_cb[4:], d_cr, w, h, ColorType.Rgb, jpeg.Subsampling.S420, tables,
                                           1, ys, cs, d_out, cap, d_len, d_ovf, ctx=gpu_ctx),
        lambda: jpeg.progressive_scans_dev(d_y, d_cb, d_cr, w, h, ColorType.Rgb, jpeg.Subsampling.S420, tables,
                                           2, ny * 64 - 8, cs, d_out, cap, d_len, d_ovf, ctx=gpu_ctx),
        lambda: jpeg.progressive_scans_dev(d_y, d_cb, d_cr, w, h, ColorType.Rgb, jpeg.Subsampling.S420, tables,
                                           1, ys + 4, cs, d_out, cap, d_len, d_ovf, ctx=gpu_ctx),
    ]
    big = np.zeros((4, 272), np.uint8)
    big[2, 15] = 255; big[2, 14] = 2   # 257 values
    over = np.zeros((4, 272), np.uint8)
    over[0, 0] = 3                     # three 1-bit codes
    for t in (big, over):
        bad_calls.append(lambda t=t: jpeg.progressive_scans_dev(d_y, d_cb, d_cr, w, h, ColorType.Rgb,
                                                                jpeg.Subsampling.S420, t, 1, ys, cs, d_out, cap,
                                                                d_len, d_ovf, ctx=gpu_ctx))
    before = d_out.cpu().numpy().copy()
    for call in bad_calls:
        with pytest.raises(_lib.PixoError) as ei:
            call()
        assert ei.value.code == _lib.ERR_INVALID_ARGUMENT
    assert _lib.load().pixo_b200_ctx_launch_count(gpu_ctx.handle) == launches
    for v in (16384, -16384):
        y_bad = frames[0][0].copy()
        y_bad[ny // 2, 37] = v
        with pytest.raises(_lib.PixoError) as ei:
            jpeg.progressive_scans_dev(_dev(y_bad), _dev(frames[0][1]), _dev(frames[0][2]), w, h, ColorType.Rgb,
                                       jpeg.Subsampling.S420, tables, 1, None, None, d_out, cap, d_len, d_ovf,
                                       ctx=gpu_ctx)
        assert ei.value.code == _lib.ERR_INVALID_ARGUMENT
    assert (d_out.cpu().numpy() == before).all()


def test_batch_of_32_4k_frames_at_max_preset(gpu_ctx):
    from pixo_b200 import jpeg, synthetic
    w, h, n = 3840, 2160, 32
    frames = np.stack([synthetic.noise(w, h, 3, k) if k % 2 else
                       np.roll(synthetic.gradient_rgb(w, h).reshape(h, w * 3), 7 * k, 0).reshape(-1) for k in range(n)])
    got = jpeg.encode_progressive_batch(frames, jpeg.JpegOptions.max(w, h, 80), ctx=gpu_ctx)
    for i in (0, 1, 16, 31):
        assert got[i] == jp.encode(frames[i], w, h, 2, 1, 80), i


def test_16384_square_frame_without_trellis(gpu_ctx):
    from pixo_b200 import jpeg, synthetic
    w = h = 16384
    img = np.ascontiguousarray(synthetic.gradient_rgb(w, h))
    img.reshape(h, w * 3)[5000:5600, :9000] = synthetic.noise(3000, 600, 3, 1).reshape(600, 9000)
    got = jpeg.encode_progressive(img, _opts(w, h, 2, 1, 80, None, True, False), ctx=gpu_ctx)
    want = jp.encode(img, w, h, 2, 1, 80, 0, True, False)
    assert hashlib.sha256(got).hexdigest() == hashlib.sha256(want).hexdigest()


def test_scans_dev_more_frames_than_one_pass(gpu_ctx):
    """8 193 frames take two passes of the stage; a bad coefficient in the second pass leaves every output
    untouched."""
    import torch
    from pixo_b200 import ColorType, _lib, jpeg
    n = 8193
    rng = np.random.default_rng(5)
    y = np.where(rng.random((n, 64)) < 0.1, rng.integers(-20, 20, (n, 64)), 0).astype(np.int16)
    y[::3] = 0
    tables = _opt_tables()
    cap = 256
    d_y = _dev(y)
    d_out = torch.full((n * cap,), 0xA5, dtype=torch.uint8, device="cuda")
    d_len = torch.full((n, 7), -1, dtype=torch.int64, device="cuda")
    d_ovf = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    jpeg.progressive_scans_dev(d_y, None, None, 8, 8, ColorType.Gray, jpeg.Subsampling.S444, tables, n, 64, 64,
                               d_out, cap, d_len, d_ovf, ctx=gpu_ctx)
    segs = _segments(d_out, d_len, d_ovf, cap, n)
    empty = np.zeros((0, 64), np.int16)
    for i in (0, 1, 2, 8190, 8191, 8192):
        assert segs[i] == ps.encode_scans(y[i:i + 1], empty, empty, tables), i
    y[8192, 5] = -16384
    d_out.fill_(0x5A); d_len.fill_(-1); d_ovf.fill_(-1)
    with pytest.raises(_lib.PixoError) as ei:
        jpeg.progressive_scans_dev(_dev(y), None, None, 8, 8, ColorType.Gray, jpeg.Subsampling.S444, tables, n, 64,
                                   64, d_out, cap, d_len, d_ovf, ctx=gpu_ctx)
    assert ei.value.code == _lib.ERR_INVALID_ARGUMENT
    assert bool((d_out == 0x5A).all()) and bool((d_len == -1).all()) and bool((d_ovf == -1).all())
