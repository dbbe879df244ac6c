"""The GPU decoders on well-formed files at full size, against the C oracles (oracle/png_decode.c,
oracle/jpeg_decode.c) and, where the frame is known from the source, against the source:

  PNG   every colour type and depth through k_png_unfilter's row groups (each filter, random per-row filters, Avg or
        Paeth on the first row of every group) at widths that cross the every-32-pixels progress publish; more row
        groups than resident warps; k_png_inflate on 4K streams of every zlib level and strategy, IDAT chunks around
        the CRC piece size, a stream that runs on past the frame, and bad files among good ones
  JPEG  files written from coefficients over every luma sampling factor 1-4 per axis, chroma factors equal to,
        below and above luma, restart intervals, 16-bit quantisation tables, a file of a million blocks; the
        libjpeg-turbo fixtures; guarded caller offsets; passes split by scratch, where the host's accounting puts them
        (a file that goes alone, behind a caller's queued work; a pass filled to its last file)
"""
import ctypes as C
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import pixo_b200
from pixo_b200 import _lib, decode
from oracle import jpeg_decode as jd
from oracle import png_decode as pd
from decode_inputs import (Coefs, dense_coefs, expand_source, geometry, idat_split, jfif, png_image, qtable,
                           safe_tails, sparse_coefs)
from jpeg_decode_corpus import corrupted
from png_decode_corpus import DEPTHS, png

pytestmark = pytest.mark.gpu
LIBJPEG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "libjpeg")
STATUS = {pd.INVALID: _lib.ERR_INVALID_DECODE, pd.UNSUPPORTED: _lib.ERR_UNSUPPORTED_DECODE,
          pd.DIMENSIONS: _lib.ERR_INVALID_DIMENSIONS, pd.TOO_LARGE: _lib.ERR_IMAGE_TOO_LARGE}


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = pixo_b200.Context(0)
    yield c
    assert c.host_fallbacks == 0
    c.close()


def guarded(ctx, fn, files, sizes, seed):
    """files through a *_decode_to_device entry point at unaligned offsets in shuffled order, 0xA5 guard gaps of odd
    lengths between the slots: (host copy of the buffer, offsets, statuses, launches the call made)"""
    rng = np.random.default_rng(seed)
    n = len(files)
    offs, o = [0] * n, 61
    for i in rng.permutation(n):
        offs[i] = o
        o += sizes[i] + 17 + int(rng.integers(0, 40))
    buf = torch.full((o + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    status = (C.c_int32 * n)()
    before = ctx.launch_count
    _lib.check(ctx.handle, fn(ctx.handle, C.cast((C.c_char_p * n)(*files), C.c_void_p),
                              (C.c_size_t * n)(*map(len, files)), n, buf.data_ptr(), (C.c_size_t * n)(*offs), status))
    launches = ctx.launch_count - before
    ctx.sync()
    return buf.cpu().numpy(), offs, list(status), launches


def check_guarded(host, offs, status, want, codes):
    """want[i]: the frame, or None for a file that fails with codes[i]; nothing outside the frames is written"""
    mask = np.ones(host.size, bool)
    for i, w in enumerate(want):
        if w is None:
            assert status[i] == codes[i] and status[i] != 0, (i, status[i], codes[i])
            continue
        assert status[i] == 0, (i, status[i])
        assert np.array_equal(host[offs[i]:offs[i] + w.size], w), i
        mask[offs[i]:offs[i] + w.size] = False
    assert (host[mask] == 0xA5).all()


# ---- PNG: the unfilter wavefront --------------------------------------------------------------------------

def _width(units: int, depth: int) -> int:
    """a width whose rows are `units` wavefront steps: pixels, or bytes below 8 bits (a part-filled last byte
    where it can be)"""
    return units if depth >= 8 else max(1, units * 8 // depth - (1 if units > 1 else 0))


def unfilter_files():
    """(file, width, depth, ct, seed, raw) over every colour type and depth: random per-row filters at heights
    around one and two row groups and widths around the progress publish; each filter alone; and a tall, wide file
    with Avg or Paeth on the first row of every group"""
    out, seed = [], 0
    for ct, depths in DEPTHS.items():
        for d in depths:
            plans = [(h, u, "random") for h in (31, 32, 33, 64, 65) for u in (1, 31, 32, 33)]
            plans += [(65, 33, (f,)) for f in range(5)]
            tall = np.random.default_rng(seed).integers(0, 5, 1001)
            tall[::32] = np.where(np.arange(len(tall[::32])) % 2, 3, 4)
            plans.append((1001, 4103 + seed % 7, tall))
            for h, u, filters in plans:
                w = _width(u, d)
                f, raw = png_image(w, h, d, ct, seed, filters=filters, level=1)
                out.append((f, w, d, ct, seed, raw))
                seed += 1
    return out


def test_unfilter_every_depth_and_filter_plan(ctx):
    """One guarded batch of every file: 8-bit Gray / GrayAlpha / RGB / RGBA frames equal their source rows; the
    rest equal the oracle, and the frame the source rows make (high bytes, bit replication, the palette)."""
    files = unfilter_files()
    want = []
    for f, w, d, ct, seed, raw in files:
        src = expand_source(raw, w, d, ct, seed)
        if d != 8 or ct == 3:
            r = pd.decode(f)
            assert r.kind == pd.OK and np.array_equal(r.pixels, src), (w, d, ct)
        want.append(src)
    host, offs, status, launches = guarded(ctx, _lib.load().pixo_b200_png_decode_to_device, [f[0] for f in files],
                                           [w.size for w in want], 1)
    assert launches == 4   # one pass: k_png_crc, k_png_inflate, k_png_unfilter, k_png_expand
    check_guarded(host, offs, status, want, None)


def test_unfilter_ticket_loop_past_the_resident_warps(ctx):
    """More 32-row groups than the sm_count * 32 warps launched, in one pass: warps draw further tickets, and a
    group waits on one a running warp drew earlier."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    target = sms * 32 + 700
    files = []
    for i, (ct, d, w) in enumerate(((6, 16, 8), (0, 1, 61), (6, 16, 3), (0, 1, 7))):
        h = 32 * (target // 4) - 5 * i
        filters = "random" if i % 2 else (4,)
        files.append((*png_image(w, h, d, ct, 50 + i, filters=filters, level=1), w, d, ct, 50 + i))
    groups = sum((f[1].shape[0] + 31) // 32 for f in files)
    assert groups > sms * 32
    want = [expand_source(raw, w, d, ct, s) for _, raw, w, d, ct, s in files]
    for (f, *_), wv in zip(files, want):
        assert np.array_equal(pd.decode(f).pixels, wv)
    before = ctx.launch_count
    got = decode.decode_png_batch_dev([f[0] for f in files], ctx=ctx)
    assert ctx.launch_count - before == 4
    host = got.frames.cpu().numpy()
    for i, wv in enumerate(want):
        assert got.errors[i] is None and np.array_equal(host[got.offsets[i]:got.offsets[i] + wv.size], wv), i


# ---- PNG: inflate at 4K -----------------------------------------------------------------------------------

W4, H4 = 3840, 2160
CHUNKS = [1, 4095, 4096, 4097, 65539]


def inflate_files():
    """(name, file, raw): 4K RGB frames, noise and smooth, through every zlib level class and strategy"""
    out = []
    k = 0
    for name, level, strategy in (("stored", 0, zlib.Z_DEFAULT_STRATEGY), ("level9", 9, zlib.Z_DEFAULT_STRATEGY),
                                  ("rle", 6, zlib.Z_RLE), ("fixed", 6, zlib.Z_FIXED),
                                  ("huffman_only", 6, zlib.Z_HUFFMAN_ONLY)):
        for kind in ("noise", "smooth"):
            chunks = CHUNKS if k % 3 == 1 else None
            f, raw = png_image(W4, H4, 8, 2, 300 + k, filters="random", level=level, strategy=strategy,
                               idat_chunks=chunks, kind=kind)
            out.append((f"{name}_{kind}", f, raw))
            k += 1
    return out


@pytest.fixture(scope="module")
def inflated():
    return inflate_files()


def test_inflate_4k_every_level_and_strategy(ctx, inflated):
    files = [f for _, f, _ in inflated]
    assert max(len(f) for f in files[:2]) > W4 * H4 * 3   # stored blocks: the stream is larger than the frame
    assert sum(f.count(b"IDAT") for f in files) > 5 * len(files)
    got = decode.decode_png_batch_dev(files, ctx=ctx)
    ctx.sync()
    for i, (name, f, raw) in enumerate(inflated):
        assert got.errors[i] is None, (name, got.errors[i])
        frame = got.frames[got.offsets[i]:got.offsets[i] + raw.size].cpu().numpy()
        assert np.array_equal(frame, raw.reshape(-1)), name


def _stream(f: bytes) -> bytes:
    o, out = 8, []
    while o < len(f):
        n = int.from_bytes(f[o:o + 4], "big")
        if f[o + 4:o + 8] == b"IDAT":
            out.append(f[o + 8:o + 8 + n])
        o += 12 + n
    return b"".join(out)


def test_stream_past_the_frame(ctx):
    """A stream that produces 100 000 bytes past expected_size, its matches crossing that boundary and reaching
    back through the 32 KiB ring: the single-file message is the oracle's, produced count included."""
    w, h = 997, 61
    period = np.random.default_rng(9).integers(0, 256, 4999, dtype=np.uint8)
    body = np.resize(period, h * (w + 1) + 100_000)
    body[:h * (w + 1):w + 1] = 0   # filter None on every row of the frame
    f = png(w, h, 8, 0, zlib.compress(body.tobytes(), 6))
    want = pd.decode(f)
    assert want.kind == pd.INVALID and want.message.endswith(f"expected {h * (w + 1)}, got {body.size}")
    with pytest.raises(pixo_b200.PixoError) as e:
        decode.decode_png(f, ctx=ctx)
    assert e.value.code == _lib.ERR_INVALID_DECODE and str(e.value).endswith(want.message)


def _rebuild(f: bytes, stream: bytes, chunks=None) -> bytes:
    w, h, d, ct = int.from_bytes(f[16:20], "big"), int.from_bytes(f[20:24], "big"), f[24], f[25]
    return png(w, h, d, ct, stream, idat_split=idat_split(len(stream), chunks))


def test_bad_4k_files_among_good_ones(ctx, inflated):
    """A bad CRC in a middle IDAT chunk, a flipped Adler-32 and filter type 5 at row 2 000, each in a 4K file,
    between good 4K files in one guarded batch: the good frames are right, the bad files get pixo's error and write
    nothing."""
    good = [inflated[i] for i in (2, 5, 8)]
    f0 = good[0][1]
    s = _stream(f0)
    chunked = _rebuild(f0, s, CHUNKS)
    idats = [i for i in range(len(chunked) - 4) if chunked[i:i + 4] == b"IDAT"]
    mid = idats[len(idats) // 2]
    n = int.from_bytes(chunked[mid - 4:mid], "big")
    crc_at = mid + 4 + n
    bad_crc = chunked[:crc_at] + bytes([chunked[crc_at] ^ 0x40]) + chunked[crc_at + 1:]
    bad_adler = _rebuild(f0, s[:-1] + bytes([s[-1] ^ 1]))
    raw = good[1][2]
    filters = np.random.default_rng(301).integers(0, 5, H4)
    filters[2000] = 5
    bad_filter, _ = png_image(W4, H4, 8, 2, 0, filters=filters, level=1, raw=raw)
    bad = [bad_crc, bad_adler, bad_filter]
    wants = [pd.decode(b) for b in bad]
    assert wants[0].message.endswith("CRC mismatch in IDAT chunk")
    assert "Adler32 mismatch" in wants[1].message and wants[2].message.endswith("invalid filter type: 5")
    for b, w in zip(bad, wants):
        with pytest.raises(pixo_b200.PixoError) as e:
            decode.decode_png(b, ctx=ctx)
        assert e.value.code == STATUS[w.kind] and str(e.value).endswith(w.message)
    files = [good[0][1], bad[0], good[1][1], bad[1], bad[2], good[2][1]]
    want = [good[0][2].reshape(-1), None, good[1][2].reshape(-1), None, None, good[2][2].reshape(-1)]
    codes = [0, STATUS[wants[0].kind], 0, STATUS[wants[1].kind], STATUS[wants[2].kind], 0]
    sizes = [w.size if w is not None else 4096 for w in want]
    host, offs, status, _ = guarded(ctx, _lib.load().pixo_b200_png_decode_to_device, files, sizes, 2)
    check_guarded(host, offs, status, want, codes)


# ---- JPEG: sampling factors, restart intervals, tables ------------------------------------------------------

def sampling_files():
    """(file, blocks) written from coefficients: every luma (h, v) in 1-4 x 1-4 with chroma equal to it, at 1x1,
    and above / below it in non-dividing ratios; gray with factors other than 1x1; sizes one pixel either side of
    an MCU edge; restart intervals 1, 7, one MCU row and more than the file holds; dense blocks with 16-bit tables"""
    out, k = [], 0
    luma = [(h, v) for h in range(1, 5) for v in range(1, 5)]
    sets = []
    for (h, v) in luma:
        sets.append([(h, v), (1, 1), (1, 1)])
        sets.append([(h, v), (h, v), (h, v)])
        sets.append([(h, v), (max(1, 4 - h), min(4, v + 1)), (3 if h != 3 else 2, 2 if v != 2 else 3)])
    sets += [[(2, 3)], [(4, 1)], [(3, 3)], [(1, 4)]]
    for s in sets:
        mh, mv = max(a for a, _ in s), max(b for _, b in s)
        w = max(1, 8 * mh * (2 + k % 3) + (k % 3) - 1)
        h = max(1, 8 * mv * (1 + k % 2) + ((k + 1) % 3) - 1)
        mw, mhh, bpm = geometry(w, h, [(a, b, None) for a, b in s])
        rs = [0, 1, 7, mw, mw * mhh + 3][k % 5]
        dense = k % 4 == 3
        tables = "optimal" if k % 2 else "standard"
        comps = [(a, b, qtable(k * 3 + c, 65535 if dense else 255)) for c, (a, b) in enumerate(s)]
        Cf = dense_coefs(mw * mhh * bpm, k, 15 if tables == "optimal" else 10, 16 if tables == "optimal" else 11) \
            if dense else sparse_coefs(mw * mhh * bpm, k)
        Cf = safe_tails(Cf, bpm, rs, mw * mhh, k)
        out.append((jfif(w, h, comps, Cf, restart=rs, tables=tables), Cf.n))
        k += 1
    return out


def check_jpeg_batch(files, ctx, singles=()):
    """decode_jpeg_batch_dev equals the oracle on every file (pixels, or pixo's message); files[i] for i in
    singles also through decode_jpeg"""
    wants = [jd.decode(f, coefs=False) for f in files]
    got = decode.decode_jpeg_batch_dev(files, ctx=ctx)
    ctx.sync()
    host = got.frames.cpu().numpy()
    for i, want in enumerate(wants):
        if want.status != jd.OK:
            assert got.geometries[i] is None and want.message in str(got.errors[i]), (i, want.message)
            continue
        assert got.geometries[i][:2] == (want.width, want.height), i
        assert np.array_equal(host[got.offsets[i]:got.offsets[i] + want.pixels.size], want.pixels), i
    for i in singles:
        if wants[i].status == jd.OK:
            img = decode.decode_jpeg(files[i], ctx=ctx)
            assert np.array_equal(img.pixels, wants[i].pixels), i
        else:
            with pytest.raises(pixo_b200.PixoError) as e:
                decode.decode_jpeg(files[i], ctx=ctx)
            assert str(e.value).endswith(wants[i].message), i
    return wants


def test_jpeg_sampling_factors_and_restarts(ctx):
    files = sampling_files()
    assert len(files) == 52
    wants = check_jpeg_batch([f for f, _ in files], ctx, singles=range(0, 52, 3))
    for (f, n), w in zip(files, wants):
        assert w.status == jd.OK and w.stored == n   # every written block decodes


def test_jpeg_a_million_blocks(ctx):
    """8 016 x 5 328 with luma 3x2 and chroma 1x1 and 2x1, sparse blocks, a restart interval of one MCU row:
    1 000 998 blocks"""
    comps = [(3, 2, qtable(1)), (1, 1, qtable(2)), (2, 1, qtable(3))]
    w, h = 8016, 5328
    mw, mh, bpm = geometry(w, h, comps)
    Cf = safe_tails(sparse_coefs(mw * mh * bpm, 5), bpm, mw, mw * mh)
    assert Cf.n > 1_000_000
    f = jfif(w, h, comps, Cf, restart=mw)
    want = jd.decode(f, coefs=False)
    assert want.status == jd.OK and want.stored == Cf.n
    img = decode.decode_jpeg(f, ctx=ctx)
    assert hashlib.sha256(img.pixels.tobytes()).hexdigest() == hashlib.sha256(want.pixels.tobytes()).hexdigest()


def libjpeg_files():
    m = json.load(open(os.path.join(LIBJPEG, "manifest.json")))
    return [open(os.path.join(LIBJPEG, c["file"]), "rb").read() for c in m]


def test_libjpeg_turbo_files(ctx):
    files = libjpeg_files()
    check_jpeg_batch(files, ctx, singles=range(len(files)))


# ---- JPEG: batches ------------------------------------------------------------------------------------------

def small_jpegs(n, seed):
    """n distinct small 4:2:0 files from the writer"""
    out = []
    for i in range(n):
        comps = [(2, 2, qtable(seed + i)), (1, 1, qtable(seed + i + 1)), (1, 1, qtable(seed + i + 2))]
        w, h = 40 + i % 9, 24 + i % 5
        mw, mh, bpm = geometry(w, h, comps)
        out.append(jfif(w, h, comps, sparse_coefs(mw * mh * bpm, seed + i)))
    return out


def test_jpeg_guarded_offsets_with_bad_files(ctx):
    """pixo_b200_jpeg_decode_to_device at unaligned, shuffled offsets, with refused, truncated and corrupted files
    among good ones: refused files write nothing, and no byte outside a frame changes"""
    good = small_jpegs(12, 70) + libjpeg_files()
    base = good[3]
    comps = [(3, 2, qtable(7)), (1, 1, qtable(8)), (2, 1, qtable(9))]
    mw, mh, bpm = geometry(97, 45, comps)
    odd = jfif(97, 45, comps, sparse_coefs(mw * mh * bpm, 7, nac=6))
    files = [odd[:len(odd) * k // 11] for k in range(3, 11)]   # scans that stop inside an MCU
    for i, g in enumerate(good):
        files.append(g)
        if i % 4 == 0:
            files.append(base[:len(base) * (i % 7 + 1) // 9])     # truncated
        if i % 5 == 1:
            files += corrupted(base, i, 1)
        if i % 6 == 2:
            files.append(b"\xFF\xD8\xFF\xC2" + g[4:])   # SOF2 in the first segment: refused
    files.append(b"not a jpeg")
    wants = [jd.decode(f, coefs=False) for f in files]
    assert sum(w.status != jd.OK for w in wants) >= 8
    want = [w.pixels if w.status == jd.OK else None for w in wants]
    codes = [0 if w.status == jd.OK else
             _lib.ERR_UNSUPPORTED_DECODE if w.status == jd.UNSUPPORTED else _lib.ERR_INVALID_DECODE for w in wants]
    sizes = [x.size if x is not None else 300 for x in want]
    host, offs, status, launches = guarded(ctx, _lib.load().pixo_b200_jpeg_decode_to_device, files, sizes, 3)
    assert launches == 3
    check_guarded(host, offs, status, want, codes)


# The JPEG launcher (jpeg_decode.cu) charges each file blocks * 192 + its entropy bytes + sizeof(JdecFile) +
# kJdecFileTables of scratch (file_scratch), and the pass driver (pass_end, decode_host.hpp) closes a pass before the
# file that would take it past 1 GiB
JDEC_PASS_BYTES = 1 << 30
JDEC_FILE_BYTES = 576 + 8 * 2048


def scan_bytes(f: bytes) -> int:
    """the entropy bytes the decoder copies for a file: from the end of the SOS segment to find_entropy_end"""
    i = 2
    while f[i + 1] != 0xDA:
        i += 2 + int.from_bytes(f[i + 2:i + 4], "big")
    i += 2 + int.from_bytes(f[i + 2:i + 4], "big")
    return jd.find_entropy_end(f[i:])


def jdec_pass_starts(scratch) -> list:
    """the first file of every pass, for files charged the given scratch bytes; a larger file goes alone"""
    starts, need = [], 0
    for i, b in enumerate(scratch):
        if not starts or need + b > JDEC_PASS_BYTES:
            starts.append(i)
            need = 0
        need += b
    return starts


def big_420(side=16384):
    """a side^2 4:2:0 file whose luma DC changes per MCU row and whose AC are all zero; its frame is grey rows"""
    comps = [(2, 2, [8] * 64), (1, 1, [8] * 64), (1, 1, [8] * 64)]
    mw, mh, bpm = geometry(side, side, comps)
    row_dc = ((np.arange(mh) * 37) % 61 - 30) * 4
    dc = np.zeros((mh, mw, bpm), np.int64)
    dc[:, :, :4] = row_dc[:, None, None]
    Cf = Coefs(dc.reshape(-1), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64))
    level = np.array([jd.idct_block(np.array([d] + [0] * 63, np.int16), comps[0][2])[0] for d in row_dc], np.uint8)
    return jfif(side, side, comps, Cf), np.repeat(level, 16)[:side]


def test_jpeg_pass_split_by_scratch_on_a_callers_stream(ctx):
    """40 small files, a 16 384^2 4:2:0 file whose scratch is over 1 GiB, 40 small files, queued behind work on a
    caller's stream: three passes of three launches, the second regrowing the scratch after the first is queued,
    and every frame right"""
    small = small_jpegs(80, 500)
    big, rows = big_420()
    files = small[:40] + [big] + small[40:]
    blocks = [geometry(40 + i % 9, 24 + i % 5, [(2, 2, 0), (1, 1, 0), (1, 1, 0)]) for i in range(80)]
    charge = [mw * mh * bpm * 192 + scan_bytes(f) + JDEC_FILE_BYTES for (mw, mh, bpm), f in zip(blocks, small)]
    assert jdec_pass_starts(charge[:40] + [1024 * 1024 * 6 * 192] + charge[40:]) == [0, 40, 41]
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        before = ctx.launch_count
        with torch.cuda.stream(s):
            torch.cuda._sleep(50_000_000)
            got = decode.decode_jpeg_batch_dev(files, ctx=ctx)
        assert ctx.launch_count - before == 9   # three passes: k_jdec_scan, k_jdec_idct, k_jdec_color
        # the call did not wait for its passes.  The sleep (some 25 ms) has drained by now: growing the scratch for
        # pass 2 waits on the stream.  What keeps the stream busy is pass 2's k_jdec_scan, one thread over the 16 384^2
        # file's 6.3 M blocks: on an H100 80GB HBM3 at 700 W the call returns about 1.9 s before the stream drains.
        assert not s.query()
        s.synchronize()
        frame = got.frames[got.offsets[40]:got.offsets[40] + 16384 * 16384 * 3].view(16384, 16384 * 3)
        assert bool((frame == torch.from_numpy(rows).cuda()[:, None]).all())
        del frame
        host = got.frames.cpu().numpy()
    finally:
        ctx.set_stream(None)
    for i, f in enumerate(files):
        if i == 40:
            continue
        want = jd.decode(f, coefs=False).pixels
        assert np.array_equal(host[got.offsets[i]:got.offsets[i] + want.size], want), i


def test_jpeg_passes_end_at_the_scratch_bound(ctx):
    """One-block files: a pass closes before the file that would take its scratch past 1 GiB, some 62 500 files in.
    That is the only bound: every file is charged at least 16 KiB, so no pass reaches 65 536 files.  A batch that
    fills a pass exactly makes one pass of three launches; one file more makes two."""
    tiny = [jfif(8, 8, [(1, 1, [8] * 64)], Coefs(np.array([k - 140]), *[np.zeros(0, np.int64)] * 3))
            for k in range(300)]
    want = [jd.decode(t, coefs=False).pixels for t in tiny]
    assert len({w.tobytes() for w in want}) > 200
    charge = [64 * 3 + scan_bytes(t) + JDEC_FILE_BYTES for t in tiny]
    full = jdec_pass_starts([charge[i % 300] for i in range(70000)])[1]
    assert 60000 < full < 65536 and sum(charge[i % 300] for i in range(full)) <= JDEC_PASS_BYTES
    for n, passes in ((full, 1), (full + 1, 2)):
        files = [tiny[i % 300] for i in range(n)]
        assert len(jdec_pass_starts([charge[i % 300] for i in range(n)])) == passes
        before = ctx.launch_count
        got = decode.decode_jpeg_batch_dev(files, ctx=ctx)
        assert ctx.launch_count - before == 3 * passes   # k_jdec_scan, k_jdec_idct, k_jdec_color per pass
        host = got.frames.cpu().numpy()
        for i in list(range(0, n, 997)) + list(range(full - 3, n)):
            assert got.errors[i] is None and np.array_equal(host[got.offsets[i]:got.offsets[i] + 64], want[i % 300]), i
