"""The GPU DEFLATE (png_deflate.cu) at its edges, against the oracle: is_high_entropy_data on both sides of 5 %,
bytes past each stream, hash state across a warp's streams and across calls, passes split by bytes, the 2^31-byte
limit, stored-block edges, and whole pixo PNG files built from the device stages with no oracle in the chain."""
import os
import time
import zlib

import numpy as np
import pytest
import torch

from deflate_inputs import (constructed, entropy_cases, families, filtered_frame, golden_pngs, idat, read_past_tail,
                            stored_block_noise)
from oracle import png_deflate as pd

pytestmark = pytest.mark.gpu

READ_PAST = 4096 + 258   # the farthest a census, match or run could read past a stream's end


@pytest.fixture(scope="module", autouse=True)
def _build():
    pd.build()


def _stored_cap(n):
    return 2 + n + (n // 65535 + 1) * 5 + 4


def _run(streams, level, ctx, cap=None, stride=None, tails=None, in_off=0, guard=64, d_src=None):
    """Every stream in one deflate_zlib_packed_dev call: stream i at in_off + i * stride of one device tensor, with
    the rest of its stride (the last slot's too) filled by read_past_tail(stream, ..., tails[i]) when tails is given;
    slot i at guard + i * cap of an output filled with 0xA5.  Checks that the guards before and after the slots and
    every byte past a stream's length in its slot were left alone; returns (outputs, lens, status)."""
    from pixo_b200 import compress
    lens = [len(s) for s in streams]
    stride = stride or max(max(lens, default=0), 1)
    if d_src is None:
        src = np.zeros(in_off + len(streams) * stride, np.uint8)
        for i, s in enumerate(streams):
            at = in_off + i * stride
            src[at:at + len(s)] = np.frombuffer(s, np.uint8)
            if tails is not None:
                src[at + len(s):at + stride] = np.frombuffer(read_past_tail(s, stride - len(s), tails[i]), np.uint8)
        d_src = torch.from_numpy(src).cuda()
    cap = cap or _stored_cap(stride)
    d_out = torch.full((guard + len(streams) * cap + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    out_lens, status = compress.deflate_zlib_packed_dev(d_src[in_off:], stride, lens, level, d_out[guard:], cap,
                                                        ctx=ctx)
    return _slots(d_out, len(streams), cap, guard, out_lens, status), out_lens, status


def _slots(d_out, n, cap, guard, out_lens, status):
    host = d_out.cpu().numpy()
    assert (host[:guard] == 0xA5).all() and (host[guard + n * cap:] == 0xA5).all()
    outs = []
    for i in range(n):
        slot = host[guard + i * cap:guard + (i + 1) * cap]
        k = int(out_lens[i]) if status[i] == 0 else 0
        assert (slot[k:] == 0xA5).all(), i
        outs.append(slot[:k].tobytes())
    return outs


def _same(outs, streams, level, names=None):
    for i, (o, s) in enumerate(zip(outs, streams)):
        assert o == pd.deflate_zlib(s, level), (names[i] if names else i, level)
        assert zlib.decompress(o) == s, (names[i] if names else i, level)


def _btype(z):
    return z[2] >> 1 & 3


# ---- A. is_high_entropy_data on both sides of 5 % -------------------------------------------------------------
@pytest.mark.parametrize("level", range(1, 10))
def test_entropy_bail_on_both_sides(gpu_ctx, level):
    """Streams that bail (stored) and streams just past the threshold (dynamic), mixed into one launch with the
    constructed streams, which parse; and each bail stream alone through the host entry point.  The zlib header's
    FLEVEL differs by level on the stored path too."""
    from pixo_b200 import compress
    cases = entropy_cases()
    items = [(k, v[0]) for k, v in cases.items()] + list(constructed().items())
    rng = np.random.default_rng(level)
    items = [items[i] for i in rng.permutation(len(items))]
    names, streams = [k for k, _ in items], [s for _, s in items]
    outs, _, status = _run(streams, level, gpu_ctx)
    assert (status == 0).all()
    _same(outs, streams, level, names)
    for name, o in zip(names, outs):
        if name in cases:
            assert _btype(o) == (0 if cases[name][2] else 2), name
    for name, (s, _, fires, _) in cases.items():
        z = compress.deflate_zlib_packed(s, level, ctx=gpu_ctx)
        assert z == pd.deflate_zlib(s, level) and _btype(z) == (0 if fires else 2), name


# ---- B. bytes past each stream, odd layouts ------------------------------------------------------------------
@pytest.mark.parametrize("level", range(1, 10))
def test_bytes_past_each_stream_are_not_read(gpu_ctx, level):
    """Every slot's tail (the last slot's too) would change the output if a match, run, 4-byte read, census or
    entropy sample ran past the stream: see read_past_tail and entropy_cases.  Odd stride, input at an odd offset of
    its tensor, odd output slots.  Each output equals the oracle run on the stream alone."""
    cases = entropy_cases()
    items = list(constructed().items()) + [(k, v[0]) for k, v in cases.items()]
    tails = [cases[k][3] if k in cases else b"" for k, _ in items]
    streams = [s for _, s in items]
    stride = max(len(s) for s in streams) + READ_PAST + 1
    stride += 1 - stride % 2
    cap = _stored_cap(stride) | 1
    outs, _, status = _run(streams, level, gpu_ctx, cap=cap, stride=stride, tails=tails, in_off=1, guard=65)
    assert (status == 0).all()
    _same(outs, streams, level, [k for k, _ in items])


# ---- C. hash state across a warp's streams and across calls ---------------------------------------------------
def test_hash_state_across_streams_and_calls(gpu_ctx):
    """About 20 000 streams of 1-4 KiB in families that share content, shuffled, so each resident warp (132 SMs x 16)
    codes about ten streams in turn and a table entry left from its previous stream would find a match.  Level 9
    and then level 1 back to back on the same context, then level 6; every stream against the oracle."""
    streams = families(20000)
    lens = [len(s) for s in streams]
    assert sorted(lens, reverse=True) != lens
    stride = 4096 + READ_PAST + 1
    src = np.zeros(len(streams) * stride, np.uint8)
    for i, s in enumerate(streams):
        src[i * stride:i * stride + len(s)] = np.frombuffer(s, np.uint8)
        src[i * stride + len(s):(i + 1) * stride] = np.frombuffer(read_past_tail(s, stride - len(s)), np.uint8)
    d_src = torch.from_numpy(src).cuda()
    from pixo_b200 import compress
    cap = _stored_cap(4096)
    guard = 64
    outs = {level: torch.full((guard + len(streams) * cap + guard,), 0xA5, dtype=torch.uint8, device="cuda")
            for level in (9, 1)}
    torch.cuda.synchronize()
    runs = [(level, d_out) + compress.deflate_zlib_packed_dev(d_src, stride, lens, level, d_out[guard:], cap, ctx=gpu_ctx)
            for level, d_out in outs.items()]
    for level, d_out, out_lens, status in runs:
        assert (status == 0).all()
        _same(_slots(d_out, len(streams), cap, guard, out_lens, status), streams, level)
    outs, _, status = _run(streams, 6, gpu_ctx, cap=cap, stride=stride, d_src=d_src)
    assert (status == 0).all()
    _same(outs, streams, 6)


# ---- D. passes split by bytes, streams too large for a pass ------------------------------------------------------
def _small(rng, n):
    return bytes(rng.integers(0, 8, n, dtype=np.uint8))


def _check_batch(wants, outs, out_lens, status, cap):
    from pixo_b200 import _lib
    for i, want in enumerate(wants):
        assert int(out_lens[i]) == len(want), i
        if len(want) > cap:
            assert status[i] == _lib.ERR_OUTPUT_TOO_SMALL and outs[i] == b"", i
        else:
            assert status[i] == 0 and outs[i] == want, i


def test_pass_split_by_bytes(gpu_ctx):
    """Seven filtered 4K RGBA frames (33.2 MB each, charged 5 B per byte: 166 MB) between small streams: six frames
    fill the first 1 GiB pass, the seventh goes in a second pass with what follows it, where a noise stream does not
    fit its slot."""
    rng = np.random.default_rng(21)
    frames = [filtered_frame(3840, 2160, 4, seed=k, noise_band=k == 3) for k in range(7)]
    smalls = [_small(rng, n) for n in (3000, 700, 9000)]
    wants = {id(s): pd.deflate_zlib(s, 2) for s in frames + smalls}
    cap = max(len(z) for z in wants.values()) | 1
    noise = rng.integers(0, 256, cap - 5, dtype=np.uint8).tobytes()
    wants[id(noise)] = pd.deflate_zlib(noise, 2)
    streams = [frames[0], smalls[0], frames[1], frames[2], smalls[1], frames[3], frames[4], frames[5], frames[6],
               smalls[2], noise]
    before = gpu_ctx.launch_count
    outs, out_lens, status = _run(streams, 2, gpu_ctx, cap=cap)
    assert gpu_ctx.launch_count - before == 4
    assert int((status != 0).sum()) == 1 and status[-1] != 0
    _check_batch([wants[id(s)] for s in streams], outs, out_lens, status, cap)


def test_stream_too_large_for_a_pass(gpu_ctx):
    """A filtered 16384 x 4096 RGBA frame (268 MB, charged 1.34 GB) goes in a pass alone between small streams:
    three passes, six launches; the last pass's noise stream does not fit its slot."""
    rng = np.random.default_rng(22)
    big = filtered_frame(16384, 4096, 4, seed=5, noise_band=True)
    smalls = [_small(rng, 5000), _small(rng, 100)]
    streams = [smalls[0], big, smalls[1]]
    wants = [pd.deflate_zlib(s, 2) for s in streams]
    cap = max(len(z) for z in wants) | 1
    streams.append(rng.integers(0, 256, cap - 5, dtype=np.uint8).tobytes())
    wants.append(pd.deflate_zlib(streams[-1], 2))
    before = gpu_ctx.launch_count
    outs, out_lens, status = _run(streams, 2, gpu_ctx, cap=cap)
    assert gpu_ctx.launch_count - before == 6
    assert [int(s != 0) for s in status] == [0, 0, 0, 1]
    _check_batch(wants, outs, out_lens, status, cap)


@pytest.mark.parametrize("level", [1, 3, 5, 7, 9])
def test_full_size_frames_at_more_levels(gpu_ctx, level):
    """Filtered 1080p RGB frames, one smooth and one with a band of noise."""
    streams = [filtered_frame(1920, 1080, 3, seed=1), filtered_frame(1920, 1080, 3, seed=2, noise_band=True)]
    outs, _, status = _run(streams, level, gpu_ctx)
    assert (status == 0).all()
    _same(outs, streams, level)


# ---- E. the i32 limit ---------------------------------------------------------------------------------------------
def test_stream_of_2_31_bytes_is_refused(gpu_ctx):
    """A real 2^31 + 1-byte buffer, so that a regression reads inside an allocation: a one-stream batch of exactly
    2^31 bytes returns ERR_UNSUPPORTED with its message before anything is launched, and writes nothing; so does the
    host entry point."""
    import pixo_b200
    from pixo_b200 import _lib, compress
    n = 1 << 31
    d_src = torch.zeros(n + 1, dtype=torch.uint8, device="cuda")
    d_out = torch.full((64 + 4096 + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    before = gpu_ctx.launch_count
    with pytest.raises(pixo_b200.PixoError) as e:
        compress.deflate_zlib_packed_dev(d_src, n, [n], 6, d_out[64:], 4096, ctx=gpu_ctx)
    assert e.value.code == _lib.ERR_UNSUPPORTED and "2^31 bytes or more" in str(e.value)
    assert gpu_ctx.launch_count == before
    assert (d_out.cpu().numpy() == 0xA5).all()
    del d_src
    with pytest.raises(pixo_b200.PixoError) as e:
        compress.deflate_zlib_packed(np.zeros(n, np.uint8), 6, ctx=gpu_ctx)
    assert e.value.code == _lib.ERR_UNSUPPORTED and "2^31 bytes or more" in str(e.value)
    assert gpu_ctx.launch_count == before


def test_largest_stream_is_coded(gpu_ctx):
    """2^31 - 1 bytes: runs of one byte value that changes every 2^20 bytes, at level 6, in a slot of the exact
    length.  32-bit positions, 64-bit token and area offsets and the Adler-32 over 32 pieces of 64 MiB."""
    from pixo_b200 import compress
    n = (1 << 31) - 1
    vals = ((np.arange(2048, dtype=np.uint32) * 157 + 11) & 0xFF).astype(np.uint8)
    host = np.repeat(vals, 1 << 20)[:n]
    t0 = time.time()
    want = pd.deflate_zlib(host, 6)
    t_oracle = time.time() - t0
    d_src = torch.from_numpy(vals).cuda()[:, None].expand(2048, 1 << 20).reshape(-1)[:n]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    guard = 64
    d_out = torch.full((guard + len(want) + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    t0 = time.time()
    out_lens, status = compress.deflate_zlib_packed_dev(d_src, n, [n], 6, d_out[guard:], len(want), ctx=gpu_ctx)
    t_gpu = time.time() - t0
    free1 = torch.cuda.mem_get_info()[0]
    assert status[0] == 0 and int(out_lens[0]) == len(want)
    assert _slots(d_out, 1, len(want), guard, out_lens, status)[0] == want
    assert int.from_bytes(want[-4:], "big") == zlib.adler32(host)
    print(f"2^31-1 bytes at level 6: {len(want)} B; GPU call {t_gpu:.1f} s, oracle {t_oracle:.1f} s; device memory "
          f"in use {(free0 - free1) / 2**30:.1f} GiB more after the call (scratch kept by the context)")


# ---- F. stored-block edges ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("level", [1, 6, 9])
def test_stored_block_edges(gpu_ctx, level):
    """Noise at and beside multiples of 65 535 bytes, each in a slot of its exact size at an odd offset: the block
    count, BFINAL on the last block only, LEN / NLEN, and the bytes against the oracle."""
    from pixo_b200 import compress
    for n, s in stored_block_noise().items():
        want = pd.deflate_zlib(s, level)
        d_src = torch.from_numpy(np.frombuffer(b"\x00" + s, np.uint8).copy()).cuda()
        d_out = torch.full((65 + len(want) + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        out_lens, status = compress.deflate_zlib_packed_dev(d_src[1:], n, [n], level, d_out[65:], len(want),
                                                            ctx=gpu_ctx)
        assert status[0] == 0
        z = _slots(d_out, 1, len(want), 65, out_lens, status)[0]
        assert z == want, n
        blocks, at, left = [], 2, n
        while at < len(z) - 4:
            ln = int.from_bytes(z[at + 1:at + 3], "little")
            assert z[at] & 6 == 0 and int.from_bytes(z[at + 3:at + 5], "little") == ln ^ 0xFFFF
            blocks.append((z[at] & 1, ln))
            at += 5 + ln
        assert at == len(z) - 4 and len(blocks) == -(-n // 65535)
        assert [b for b, _ in blocks] == [0] * (len(blocks) - 1) + [1]
        assert [ln for _, ln in blocks] == [min(65535, n - 65535 * k) for k in range(len(blocks))]


# ---- G. whole pixo PNG files from the device stages ----------------------------------------------------------------
def _golden_jobs():
    """[(path, preset, img, options, palette or None, stage)] for every preset-0/1 golden, with its input
    regenerated as the per-stage golden tests do."""
    import json
    from golden_inputs import make_input
    from pixo_b200 import ColorType, png
    from test_png_quantize import fixture_palette, fixture_parts, quantize_case_input
    from test_png_reduce import reduce_case_input
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    jobs = []
    for sub in ("", "reduce", "quantize"):
        for c in json.load(open(os.path.join(gold, sub, "manifest.json")))["png"]:
            if c["preset"] not in (0, 1):
                continue
            w, h, ct, pal = c["w"], c["h"], c["ct"], None
            if sub == "quantize":
                img = quantize_case_input(c)
                o = png.PngOptions.from_preset_with_lossless(w, h, c["preset"], False)
                if c["kind"] == "trunc":
                    pal = fixture_palette(fixture_parts(c))
            else:
                img = reduce_case_input(c) if sub == "reduce" else make_input(c["kind"], w, h, (1, 2, 3, 4)[ct], c["seed"])
                o = png.PngOptions.from_preset(w, h, c["preset"])
            o.color_type = ColorType(ct)
            jobs.append((os.path.join(gold, sub, c["file"]), c["preset"], img, o, pal, sub))
    return jobs


def test_whole_pngs_from_device_stages(gpu_ctx):
    """Each golden's stage (reduce_and_filter_dev, or quantize_and_filter_dev for quantize/) writes slot i of one
    device buffer per preset; without a synchronisation deflate_zlib_packed_dev then codes that buffer in place at
    the stage's stride, at level 2 (preset 0) or 6 (preset 1).  pd.png_file wraps each stream with the stage's
    IHDR fields, palette and tRNS: the file equals real pixo's, and the stage's Adler-32 the stream's.  The only
    files allowed to differ are the preset-0 ones whose filter stream the library does not reproduce (see below)."""
    from pixo_b200 import compress, png
    jobs = _golden_jobs()
    assert sorted(p for p, *_ in jobs) == sorted(p for p, _ in golden_pngs()) and len(jobs) == 199
    stride = max(o.height * (o.width * int(o.color_type.bytes_per_pixel()) + 1) for _, _, _, o, _, _ in jobs) | 1
    d_imgs = [torch.from_numpy(np.ascontiguousarray(img).reshape(-1).copy()).cuda() for _, _, img, _, _, _ in jobs]
    groups = {}
    for preset in (0, 1):
        idx = [i for i, j in enumerate(jobs) if j[1] == preset]
        groups[preset] = (idx, torch.full((len(idx) * stride,), 0xA5, dtype=torch.uint8, device="cuda"),
                          torch.zeros(len(idx), dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    reds = {}
    for preset, (idx, buf, adl) in groups.items():
        for k, i in enumerate(idx):
            _, _, img, o, pal, stage = jobs[i]
            out = buf[k * stride:]
            if stage == "quantize":
                reds[i] = png.quantize_and_filter_dev(d_imgs[i], img.size, 1, o, out, stride, adl[k:k + 1],
                                                      palettes=None if pal is None else [pal], ctx=gpu_ctx)[0]
            else:
                reds[i] = png.reduce_and_filter_dev(d_imgs[i], img.size, 1, o, out, stride, adl[k:k + 1],
                                                    ctx=gpu_ctx)[0]
    zs, filtered = {}, {}
    for preset, (idx, buf, adl) in groups.items():
        level = {0: 2, 1: 6}[preset]
        lens = [jobs[i][3].height * (1 + reds[i].row_bytes) for i in idx]
        cap = _stored_cap(stride)
        d_z = torch.full((len(idx) * cap,), 0xA5, dtype=torch.uint8, device="cuda")
        out_lens, status = compress.deflate_zlib_packed_dev(buf, stride, lens, level, d_z, cap, ctx=gpu_ctx)
        assert (status == 0).all()
        outs = _slots(d_z, len(idx), cap, 0, out_lens, status)
        sums = adl.cpu().numpy().view(np.uint32)
        host = buf.cpu().numpy()
        for k, i in enumerate(idx):
            zs[i] = outs[k]
            filtered[i] = host[k * stride:k * stride + lens[k]].tobytes()
            assert int(sums[k]) == int.from_bytes(outs[k][-4:], "big"), jobs[i][0]
    bad = []
    for i, (path, preset, _, o, _, _) in enumerate(jobs):
        r = reds[i]
        png_bytes = open(path, "rb").read()
        if pd.png_file(o.width, o.height, r.bit_depth, r.color_type_byte, zs[i], r.palette, r.trns) == png_bytes:
            continue
        # The one known exception is the filter stage's, not DEFLATE's: pixo's wasm build runs AdaptiveFast
        # sequentially, and its filter choice sticks past row 32, where the library implements the default
        # (parallel) build.  Those files' filtered streams differ; their DEFLATE still equals the oracle's.
        name = os.path.relpath(path, os.path.dirname(os.path.abspath(__file__)))
        assert preset == 0 and o.height > 32 and o.width * o.height > 4096 and os.sep not in os.path.relpath(
            path, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")), name
        assert filtered[i] != zlib.decompress(idat(png_bytes)), name
        assert zs[i] == pd.deflate_zlib(filtered[i], 2), name
        bad.append(name)
    print(f"{len(jobs) - len(bad)} of {len(jobs)} goldens reproduced whole; sequential AdaptiveFast: {bad}")
