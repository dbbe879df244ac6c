"""The JPEG transform kernels (k_jpeg_420, k_jpeg_444, k_jpeg_gray) at their edges (tests/transform_inputs.py):
quotients exactly on and one ulp beside the rounding ties at every position and on every route, all 2^24 RGB colours
as flat blocks, flat MCUs and 2x2 quads, every width and height residue and base-pointer phase, unit walks that take
every carry of advance(), the 65 535-frames-per-launch split, and the quantisation tables the kernels refuse.  Every
result is compared with the oracle or with tests/transform_ref.py."""
import numpy as np
import pytest
import torch

import transform_inputs as I
import transform_ref as R
from oracle import jpeg_trellis as jt
from pixo_b200 import _lib, jpeg
from test_dev_layouts_gpu import (GUARD16, ZIGZAG, assert_guard, encode_dev, guarded, placed, run, scan_bytes,
                                  stripes)

pytestmark = pytest.mark.gpu

MODES = {"gray": (0, 0), "444": (2, 0), "420": (2, 1)}   # (colour type, subsampling)
TRELLIS = 2
UNZIG = np.argsort(R.ZIGZAG)
ONES = np.ones(64, np.float32)


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "work was silently done on the host"


def _f32p(a):
    return a.ctypes.data_as(_lib.f32p)


def coefficients_dev(ctx, frames, w, h, mode, lum_q, chr_q, flags=0, px_off=0, px_pad=0, c_pad=8):
    """pixo_b200_jpeg_coefficients_dev on `frames` (stripes around each, `px_pad` bytes between), outputs in guarded
    buffers at padded strides; returns per frame (y, cb, cr) in natural order"""
    ct, ss = MODES[mode]
    n, flen = len(frames), frames[0].size
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    src = placed(frames, px_off, flen + px_pad, stripes)
    ys, cs = ny * 64 + c_pad, max(nc, 1) * 64 + c_pad
    dy = guarded((n - 1) * ys + ny * 64, np.int16, GUARD16)
    dcb = guarded((n - 1) * cs + nc * 64, np.int16, GUARD16)
    dcr = guarded((n - 1) * cs + nc * 64, np.int16, GUARD16)
    run(ctx, _lib.load().pixo_b200_jpeg_coefficients_dev, src.ptr(px_off), flen + px_pad, n, w, h, ct, ss,
        _f32p(lum_q), _f32p(chr_q), dy.ptr(64), ys, dcb.ptr(64) if nc else None, dcr.ptr(64) if nc else None, cs,
        flags, None)
    y, cb, cr = dy.get(), dcb.get(), dcr.get()
    assert_guard(y, [(64 + i * ys, ny * 64) for i in range(n)], GUARD16, "Y")
    assert_guard(cb, [(64 + i * cs, nc * 64) for i in range(n)], GUARD16, "Cb")
    assert_guard(cr, [(64 + i * cs, nc * 64) for i in range(n)], GUARD16, "Cr")
    out = []
    for i in range(n):
        arrs = [y[64 + i * ys:][:ny * 64], cb[64 + i * cs:][:nc * 64], cr[64 + i * cs:][:nc * 64]]
        arrs = [a.reshape(-1, 64) for a in arrs]
        if flags & ZIGZAG:
            arrs = [a[:, UNZIG] for a in arrs]
        out.append(arrs)
    return out


def _same(got, want, what):
    for a, b, name in zip(got, want, ("Y", "Cb", "Cr")):
        assert a.shape == b.shape and np.array_equal(a, b), (what, name, np.argwhere(a != b)[:4].tolist())


def _case_values(fr, arrs):
    for c in fr.cases:
        nb = 4 if fr.mode == "420" and c.comp == 0 else 1
        got = int(arrs[c.comp][c.block * nb + c.sub][c.pos])
        assert got == c.want, (c, got)


# ---- quantiser cases ----------------------------------------------------------------------------------
@pytest.mark.parametrize("route", I.ROUTES)
@pytest.mark.parametrize("zigzag", [False, True])
def test_quantiser_cases_host(po, gpu_ctx, route, zigzag):
    """compute_all_coefficients with each frame's own tables, natural and zig-zag order"""
    for fr in I.quantiser_frames(route):
        ct, ss = MODES[fr.mode]
        want = po.jpeg_coefficients(fr.pixels, fr.w, fr.h, ct, ss, lum_q=fr.lum_q, chr_q=fr.chr_q)
        got = jpeg.compute_all_coefficients(fr.pixels, fr.w, fr.h, ct, ss, lum_q=fr.lum_q, chr_q=fr.chr_q,
                                            zigzag=zigzag, ctx=gpu_ctx)
        got = [g[:, UNZIG] if zigzag else g for g in got]
        _same(got, want, (route, fr.w))
        _case_values(fr, got)


def _mirrored(fr):
    """the frame with its blocks (MCUs) in reverse order: the same cases in other lanes and units"""
    ch = 1 if fr.mode == "gray" else 3
    px = fr.h
    t = fr.pixels.reshape(px, fr.w // px, px, ch)[:, ::-1]
    return np.ascontiguousarray(t).reshape(-1)


@pytest.mark.parametrize("route", I.ROUTES)
def test_quantiser_cases_dev(po, gpu_ctx, route):
    """pixo_b200_jpeg_coefficients_dev, each frame batched with its mirror image, natural and zig-zag, aligned (TMA
    where the pitch allows) and at an odd pixel offset"""
    for fr in I.quantiser_frames(route):
        ct, ss = MODES[fr.mode]
        frames = [fr.pixels, _mirrored(fr)]
        want = [po.jpeg_coefficients(f, fr.w, fr.h, ct, ss, lum_q=fr.lum_q, chr_q=fr.chr_q) for f in frames]
        for flags, px_off in ((0, 0), (ZIGZAG, 0), (0, 3), (ZIGZAG, 1)):
            got = coefficients_dev(gpu_ctx, frames, fr.w, fr.h, fr.mode, fr.lum_q, fr.chr_q, flags, px_off, 5)
            for g, wnt in zip(got, want):
                _same(g, wnt, (route, fr.w, flags, px_off))
            _case_values(fr, got[0])


# ---- every colour -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def colour_luts():
    ycc = torch.from_numpy(R.all_colours_ycbcr().astype(np.int64)).cuda()
    dc = torch.from_numpy(R.flat_dc(np.arange(256)).astype(np.int64)).cuda()
    qdc = torch.from_numpy(R.flat_dc(np.arange(1021, dtype=np.float32) / 4).astype(np.int64)).cuda()
    return ycc, dc, qdc


def _rgb(cols):
    return torch.stack([cols >> 16, (cols >> 8) & 255, cols & 255], -1).to(torch.uint8)


def _dev_tensors(ctx, px, n, w, h, mode, offset=0):
    """one coefficients_dev call on device frames `px` [n, frame bytes] (copied to byte `offset` of a fresh buffer);
    returns (y, cb, cr) int16 tensors [blocks, 64] over all frames"""
    ct, ss = MODES[mode]
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    flen = px.shape[1]
    if offset:
        buf = torch.empty(n * flen + 16, dtype=torch.uint8, device="cuda")
        buf[offset:offset + n * flen] = px.reshape(-1)
        ptr = buf.data_ptr() + offset
    else:
        buf, ptr = px, px.data_ptr()
    y = torch.empty(n * ny * 64, dtype=torch.int16, device="cuda")
    cb = torch.empty(n * nc * 64, dtype=torch.int16, device="cuda")
    cr = torch.empty(n * nc * 64, dtype=torch.int16, device="cuda")
    run(ctx, _lib.load().pixo_b200_jpeg_coefficients_dev, ptr, flen, n, w, h, ct, ss, _f32p(ONES), _f32p(ONES),
        y.data_ptr(), ny * 64, cb.data_ptr(), cr.data_ptr(), nc * 64, 0, None)
    del buf
    return y.view(-1, 64), cb.view(-1, 64), cr.view(-1, 64)


def _flat_check(arr, want_dc, what):
    bad = int((arr[:, 0].long() != want_dc).sum())
    assert bad == 0, (what, bad, torch.nonzero(arr[:, 0].long() != want_dc)[:4].flatten().tolist())
    assert not bool(arr[:, 1:].any()), (what, "AC")


def _flat_run(ctx, luts, mode, chunk, fw, offset=0):
    ycc, dc, _ = luts
    px = 8 if mode == "444" else 16
    per = fw // px
    for c0 in range(0, 1 << 24, chunk):
        cols = torch.arange(c0, c0 + chunk, dtype=torch.int64, device="cuda")
        n = chunk // per
        f = _rgb(cols).view(n, 1, per, 1, 3).expand(n, px, per, px, 3).reshape(n, -1)
        y, cb, cr = _dev_tensors(ctx, f, n, fw, px, mode, offset)
        del f
        nyb = 1 if mode == "444" else 4
        yy = ycc[cols]
        _flat_check(y, dc[yy[:, 0]].repeat_interleave(nyb), (mode, c0, "Y"))
        _flat_check(cb, dc[yy[:, 1]], (mode, c0, "Cb"))
        _flat_check(cr, dc[yy[:, 2]], (mode, c0, "Cr"))
        del y, cb, cr, yy
        if offset:
            return
    torch.cuda.empty_cache()


def test_every_colour_flat_444(gpu_ctx, colour_luts):
    """k_jpeg_444: each of the 2^24 colours as a flat 8x8 block; with all-ones tables every DC is a known,
    value-injective function of Y, Cb or Cr and every AC is 0.  One chunk again through the clamped loader."""
    _flat_run(gpu_ctx, colour_luts, "444", I.CHUNK444, I.FLAT444_W)
    _flat_run(gpu_ctx, colour_luts, "444", 1 << 16, I.FLAT444_W, offset=1)


def test_every_colour_flat_420(gpu_ctx, colour_luts):
    """k_jpeg_420: each colour as a flat 16x16 MCU (its quad sums are 4 c)"""
    _flat_run(gpu_ctx, colour_luts, "420", I.CHUNK420, I.FLAT420_W)
    _flat_run(gpu_ctx, colour_luts, "420", 1 << 16, I.FLAT420_W, offset=1)


def _quad_frames(quads):
    """[m, 4] colour indices (TL, TR, BL, BR) -> frames of 512 MCUs, each MCU one quad tiled: [m / 512, bytes]"""
    rgb = _rgb(quads)                                   # [m, 4, 3]
    n = quads.shape[0] // 512
    q = rgb.view(n, 512, 2, 2, 3).permute(0, 2, 1, 3, 4)        # [n, ry, mcu, rx, 3]
    q = q.reshape(n, 1, 2, 512, 1, 2, 3).expand(n, 8, 2, 512, 8, 2, 3)
    return q.reshape(n, -1).contiguous()


def _quad_check(luts, quads, y, cb, cr, what):
    ycc, _, qdc = luts
    yy = ycc[quads]                                     # [m, 4, 3]
    _flat_check(cb, qdc[yy[:, :, 1].sum(1)], (what, "Cb"))
    _flat_check(cr, qdc[yy[:, :, 2].sum(1)], (what, "Cr"))
    y4 = y.view(-1, 4, 64)
    assert bool((y4 == y4[:, :1]).all()), (what, "the four Y blocks of an MCU differ")
    got = y4[:, 0].cpu().numpy()
    yv = yy[:, :, 0].cpu().numpy()
    for s in range(0, len(yv), 1 << 17):                # the restated DCT of the tiled quad, on the host
        v = yv[s:s + (1 << 17)]
        blocks = v[:, [0, 1] * 4 + [2, 3] * 4][:, np.tile(np.arange(16), 4)]
        want = R.quantize(R.dct_2d(R.gray_block(blocks)), ONES)
        bad = np.flatnonzero((got[s:s + len(v)] != want).any(1))
        assert bad.size == 0, (what, "Y", s + bad[:4])


def test_every_colour_in_a_quad_420(gpu_ctx, colour_luts):
    """k_jpeg_420: every colour once in a 2x2 quad (a seeded permutation), one quad tiled per MCU, and quads at the
    ends of the chroma sums' range.  Chroma DC against the quad sums, Y blocks against the restated DCT."""
    perm = torch.from_numpy(I.quad_permutation().astype(np.int64))
    for q0 in range(0, perm.shape[0], I.CHUNK_QUAD):
        quads = perm[q0:q0 + I.CHUNK_QUAD].cuda()
        f = _quad_frames(quads)
        y, cb, cr = _dev_tensors(gpu_ctx, f, f.shape[0], I.QUAD_W, 16, "420")
        del f
        _quad_check(colour_luts, quads, y, cb, cr, ("quads", q0))
        if q0 == 0:   # again through the clamped loader
            g = _quad_frames(quads[:1 << 15])
            y1, cb1, cr1 = _dev_tensors(gpu_ctx, g, g.shape[0], I.QUAD_W, 16, "420", offset=1)
            assert all(bool(torch.equal(a, b[:len(a)])) for a, b in ((y1, y), (cb1, cb), (cr1, cr)))
        del y, cb, cr, quads
    ext = torch.from_numpy(I.extreme_quads().astype(np.int64)).cuda()
    ext = ext.repeat(128, 1)                            # 512 quads: one frame
    f = _quad_frames(ext)
    y, cb, cr = _dev_tensors(gpu_ctx, f, 1, I.QUAD_W, 16, "420")
    _quad_check(colour_luts, ext, y, cb, cr, "extremes")
    s = colour_luts[0][ext[:4]].sum(1)                 # the four quads' (Y, Cb, Cr) sums
    assert [int(s[0, 1]), int(s[1, 1]), int(s[2, 2]), int(s[3, 2])] == [1020, 4, 1020, 4]
    torch.cuda.empty_cache()


# ---- geometry ----------------------------------------------------------------------------------------
def _trellis_ref(frame, w, h, mode):
    ct, ss = MODES[mode]
    return jt.jpeg_coefficients(frame, w, h, ct, ss, 80)


@pytest.mark.parametrize("mode", ["420", "444", "gray"])
def test_geometry_sweep(po, gpu_ctx, mode):
    """Every width and height residue and the tile boundaries, two frames per call with poison between them:
    natural and zig-zag coefficients, coefficient records (through jpeg_encode_dev files) and COEF_TRELLIS"""
    ct, ss = MODES[mode]
    ch = 1 if mode == "gray" else 3
    _, _, lq, cq = jpeg.quant_tables(80)
    for i, (w, h) in enumerate(I.geometry_shapes(mode)):
        frames = [I.geometry_frame(w, h, ch, 7 * i + k) for k in range(2)]
        want = [po.jpeg_coefficients(f, w, h, ct, ss, 80) for f in frames]
        for flags, off, pad in ((0, 0, 0), (ZIGZAG, i % 16, 5)):
            got = coefficients_dev(gpu_ctx, frames, w, h, mode, lq, cq, flags, off, pad)
            for g, wnt in zip(got, want):
                _same(g, wnt, (mode, w, h, flags, off))
        refs = [scan_bytes(po.jpeg_encode(f, w, h, ct, 80, ss)) for f in frames]
        cap = (max(len(r) for r in refs) + 64 + 15) // 16 * 16
        slots, lens, ovf = encode_dev(gpu_ctx, frames, w, h, ct, ss, 80, i % 5, 3, cap)
        for k, r in enumerate(refs):
            assert ovf[k] == 0 and lens[k] == len(r) and slots[k][:len(r)].tobytes() == r, (mode, w, h, k)
        got = coefficients_dev(gpu_ctx, frames, w, h, mode, lq, cq, TRELLIS, 1, 3)
        for g, f in zip(got, frames):
            _same(g, _trellis_ref(f, w, h, mode), (mode, w, h, "trellis"))


@pytest.mark.parametrize("mode", ["420", "444"])
def test_base_pointer_phases(po, gpu_ctx, mode):
    """Widths whose pitch is a multiple of 16 at pixel offsets 0-15: TMA at 0, the funnel-shift loader at every
    other byte phase (and the byte loader near the buffer's ends)"""
    ct, ss = MODES[mode]
    _, _, lq, cq = jpeg.quant_tables(80)
    for w, h in ((16, 16), (48, 23), (256, 17), (528, 40)):
        frames = [I.geometry_frame(w, h, 3, w + k) for k in range(3)]
        want = [po.jpeg_coefficients(f, w, h, ct, ss, 80) for f in frames]
        for off in range(16):
            got = coefficients_dev(gpu_ctx, frames, w, h, mode, lq, cq, 0, off, 0)
            for g, wnt in zip(got, want):
                _same(g, wnt, (mode, w, h, off))


# ---- the unit walk -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["420", "444"])
def test_walk_shapes(po, gpu_ctx, mode):
    """Batches of at least three grid strides of units, with 1, 2, 3, 15, 16 and 17 units per MCU row: the warps'
    steps carry ux into my, wrap my into the next frame, and do both at once.  Frames are whole MCU rows, so the
    batch stacked vertically is one image for the oracle."""
    ct, ss = MODES[mode]
    _, _, lq, cq = jpeg.quant_tables(80)
    g = torch.Generator(device="cuda").manual_seed(11)
    for w, h, n, ux, my in I.walk_shapes(mode):
        px = torch.randint(0, 256, (n, w * h * 3), dtype=torch.uint8, device="cuda", generator=g)
        y, cb, cr = _dev_tensors_q(gpu_ctx, px, n, w, h, mode, lq, cq)
        want = po.jpeg_coefficients(px.cpu().numpy().reshape(-1), w, h * n, ct, ss, 80)
        _same([y.cpu().numpy(), cb.cpu().numpy(), cr.cpu().numpy()], want, (mode, w, h, n))


def _dev_tensors_q(ctx, px, n, w, h, mode, lq, cq):
    ct, ss = MODES[mode]
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    y = torch.empty(n * ny * 64, dtype=torch.int16, device="cuda")
    cb = torch.empty(n * nc * 64, dtype=torch.int16, device="cuda")
    cr = torch.empty(n * nc * 64, dtype=torch.int16, device="cuda")
    run(ctx, _lib.load().pixo_b200_jpeg_coefficients_dev, px.data_ptr(), px.shape[1], n, w, h, ct, ss, _f32p(lq),
        _f32p(cq), y.data_ptr(), ny * 64, cb.data_ptr(), cr.data_ptr(), nc * 64, 0, None)
    return y.view(-1, 64), cb.view(-1, 64), cr.view(-1, 64)


@pytest.mark.parametrize("mode,px", [("420", 16), ("444", 8)])
def test_rgb_launch_split(po, gpu_ctx, mode, px):
    """65 537 distinct px x px RGB frames: K1 and K2 run 65 535 frames per launch"""
    ct, ss = MODES[mode]
    _, _, lq, cq = jpeg.quant_tables(80)
    n = 65537
    g = torch.Generator(device="cuda").manual_seed(5)
    f = torch.randint(0, 256, (n, px * px * 3), dtype=torch.uint8, device="cuda", generator=g)
    f[::5] = f[::5] // 64 * 64                         # some coarser frames, shorter blocks
    l0 = gpu_ctx.launch_count
    y, cb, cr = _dev_tensors_q(gpu_ctx, f, n, px, px, mode, lq, cq)
    assert gpu_ctx.launch_count - l0 == 2
    want = po.jpeg_coefficients(f.cpu().numpy().reshape(-1), px, px * n, ct, ss, 80)
    _same([y.cpu().numpy(), cb.cpu().numpy(), cr.cpu().numpy()], want, (mode, "split"))


# ---- table validation --------------------------------------------------------------------------------
BAD_ENTRIES = [0.0, -1.0, 0.5, 255.5, 256.0, np.inf, -np.inf, np.nan, -0.0, 1e-45, 2.0 ** 31]


@pytest.mark.parametrize("mode", ["420", "444", "gray"])
def test_tables_outside_1_to_255_are_refused(po, gpu_ctx, mode):
    """Every table entry the exact division is not proved for is refused before any launch, in either table and at
    any position, with the outputs untouched; 1.0 and 255.0 are accepted"""
    lib = _lib.load()
    ct, ss = MODES[mode]
    w, h = 40, 24
    frame = I.geometry_frame(w, h, 1 if mode == "gray" else 3, 3)
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    src = placed([frame], 0, 0, stripes)
    dy, dcb, dcr = (guarded(n * 64, np.int16, GUARD16) for n in (ny, nc, nc))
    _, _, lq, cq = jpeg.quant_tables(80)
    torch.cuda.synchronize()
    for k, bad in enumerate(BAD_ENTRIES):
        for which in range(2):
            tabs = [lq.copy(), cq.copy()]
            tabs[which][(11 * k + 63 * which) % 64] = np.float32(bad)
            for flags in (0, ZIGZAG, TRELLIS):
                l0 = gpu_ctx.launch_count
                rc = lib.pixo_b200_jpeg_coefficients_dev(gpu_ctx.handle, src.ptr(), frame.size, 1, w, h, ct, ss,
                                                         _f32p(tabs[0]), _f32p(tabs[1]), dy.ptr(64), ny * 64,
                                                         dcb.ptr(64), dcr.ptr(64), nc * 64, flags, None)
                assert rc == _lib.ERR_INVALID_ARGUMENT, (bad, which, flags, rc)
                assert gpu_ctx.launch_count == l0, (bad, which, flags)
            with pytest.raises(_lib.PixoError):
                jpeg.compute_all_coefficients(frame, w, h, ct, ss, lum_q=tabs[0], chr_q=tabs[1], ctx=gpu_ctx)
    gpu_ctx.sync()
    for b, name in ((dy, "Y"), (dcb, "Cb"), (dcr, "Cr")):
        assert_guard(b.get(), [], GUARD16, name + " of refused calls")
    for v in (1.0, 255.0):
        t = np.full(64, v, np.float32)
        t2 = np.where(np.arange(64) % 2 == 0, np.float32(1.0), np.float32(255.0)).astype(np.float32)
        for lt, ctab in ((t, t), (t2, t2[::-1].copy())):
            got = coefficients_dev(gpu_ctx, [frame], w, h, mode, lt, ctab)
            _same(got[0], po.jpeg_coefficients(frame, w, h, ct, ss, lum_q=lt, chr_q=ctab), (mode, v))
