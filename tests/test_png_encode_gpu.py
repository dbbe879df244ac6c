"""Whole PNG files on the GPU (pixo_b200_png_encode*, png_encode.cu) against real pixo's files and the oracle
composition in png_encode_ref.py: every preset-0/1 golden through both calls, IDAT chunk boundaries, a batch that
mixes every route, passes, stream order after the decoder and resizer, the 2^31-byte limit and launch counts."""
import zlib

import numpy as np
import pytest
import torch

import png_encode_ref as R
from oracle import png_deflate as pd
from test_png_encode import SEQUENTIAL_ADAPTIVE_FAST

pytestmark = pytest.mark.gpu

GUARD = 0xA5


@pytest.fixture(scope="module", autouse=True)
def _build():
    pd.build()


def _want(name, img, o, pal):
    """pixo's file, or for the sequential-AdaptiveFast goldens the oracle with pixo's default (parallel) filter."""
    if name in SEQUENTIAL_ADAPTIVE_FAST:
        return R.encode(img, o, pal, parallel_feature=True)
    return R.golden_bytes(name)


def _frames(imgs, stride):
    """The frames at stride bytes (odd or not) in one device tensor, the gaps filled with GUARD."""
    buf = np.full(len(imgs) * stride, GUARD, np.uint8)
    for i, img in enumerate(imgs):
        buf[i * stride:i * stride + img.size] = np.asarray(img, np.uint8).reshape(-1)
    return torch.from_numpy(buf).cuda()


def _slots(d_out, n, cap, lens, status, guard=64):
    """The files in their slots; every byte after a file in its slot (the whole slot if it has none) and the guards
    before and after the slots hold GUARD."""
    host = d_out.cpu().numpy()
    assert (host[:guard] == GUARD).all() and (host[guard + n * cap:] == GUARD).all()
    outs = []
    for i in range(n):
        slot = host[guard + i * cap:guard + (i + 1) * cap]
        k = int(lens[i]) if status[i] == 0 else 0
        assert (slot[k:] == GUARD).all(), i
        outs.append(slot[:k].tobytes())
    return outs


def _encode_dev(imgs, o, ctx, cap, in_stride=None, palettes=None, guard=64):
    in_stride = in_stride or imgs[0].size
    d_in = _frames(imgs, in_stride)
    d_out = torch.full((guard + len(imgs) * cap + guard,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()   # the fill runs on torch's stream, the encode on the context's
    from pixo_b200 import png
    lens, status, infos = png.encode_on_device(d_in, in_stride, len(imgs), o, d_out[guard:], cap, palettes=palettes,
                                               ctx=ctx)
    return _slots(d_out, len(imgs), cap, lens, status, guard), lens, status, infos


# ---- the goldens -----------------------------------------------------------------------------------------------
def test_goldens_through_the_host_call(gpu_ctx):
    """187 goldens equal pixo's file; the 12 sequential-AdaptiveFast ones equal the oracle with the parallel filter,
    and they are exactly those the oracle's sequential filter reproduces and the parallel one does not."""
    from pixo_b200 import png
    differ = []
    for name, preset, img, o, pal in R.golden_jobs():
        got = png.encode(img, o, pal, ctx=gpu_ctx)
        if got != R.golden_bytes(name):
            differ.append(name)
        assert got == _want(name, img, o, pal), name
        out = bytearray(b"stale")
        png.encode_into(out, img, o, pal, ctx=gpu_ctx)
        assert out == got
    assert differ == SEQUENTIAL_ADAPTIVE_FAST


def test_goldens_through_the_device_call(gpu_ctx):
    """One encode_on_device call per geometry, preset and route, frames at an odd in_stride, files in guarded slots of
    odd out_cap_each."""
    from pixo_b200 import png
    groups = {}
    for name, preset, img, o, pal in R.golden_jobs():
        key = (o.width, o.height, int(o.color_type), preset, int(o.quantization_mode))
        groups.setdefault(key, []).append((name, img, o, pal))
    for key, jobs in groups.items():
        o = jobs[0][2]
        imgs = [np.asarray(j[1], np.uint8).reshape(-1) for j in jobs]
        stride = imgs[0].size + 1 + imgs[0].size % 2
        cap = png.encode_capacity(o.width, o.height, o.color_type) | 1
        pals = [j[3] for j in jobs] if any(j[3] is not None for j in jobs) else None
        outs, lens, status, _ = _encode_dev(imgs, o, gpu_ctx, cap, stride, pals, guard=65)
        assert (status == 0).all(), key
        for (name, img, oo, pal), got in zip(jobs, outs):
            assert got == _want(name, img, oo, pal), name


# ---- IDAT chunk boundaries ---------------------------------------------------------------------------------------
def _stored_len(n):
    return 2 + n + -(-n // 65535) * 5 + 4


def _geometry_for(zlen):
    """A Gray geometry whose unfiltered rows (strategy None) make a stored zlib stream of exactly zlen bytes."""
    for h in (1, 2, 3, 5, 7):
        for n in range(zlen - 6 - 5 * (zlen // 65535 + 2), zlen):
            if n % h == 0 and n // h > 1 and _stored_len(n) == zlen:
                return n // h - 1, h
    raise AssertionError(zlen)


@pytest.mark.parametrize("k", [1, 2])
def test_idat_chunk_boundaries(gpu_ctx, k):
    from pixo_b200 import decode, png
    from pixo_b200.color import ColorType
    for zlen in (k * pd.IDAT_CHUNK - 1, k * pd.IDAT_CHUNK, k * pd.IDAT_CHUNK + 1):
        w, h = _geometry_for(zlen)
        img = np.random.default_rng(zlen).integers(0, 256, (h, w), dtype=np.uint8)
        o = png.PngOptions(w, h, ColorType.Gray, png.FilterStrategy.NoFilter, compression_level=6)
        want = R.encode(img, o, parallel_feature=True)
        got = png.encode(img, o, ctx=gpu_ctx)
        assert got == want, zlen
        chunks = pd.chunks(got)
        idats = [(t, p) for t, p in chunks if t == b"IDAT"]
        assert len(idats) == -(-zlen // pd.IDAT_CHUNK)
        assert [len(p) for _, p in idats] == [min(pd.IDAT_CHUNK, zlen - pd.IDAT_CHUNK * i) for i in range(len(idats))]
        at = 8
        for t, p in chunks:
            assert int.from_bytes(got[at + 8 + len(p):at + 12 + len(p)], "big") == zlib.crc32(t + p)
            at += 12 + len(p)
        raw = zlib.decompress(b"".join(p for _, p in idats))
        assert raw == np.concatenate([np.zeros((h, 1), np.uint8), img], 1).tobytes()
        assert np.array_equal(np.asarray(decode.decode_png(got, ctx=gpu_ctx).pixels).reshape(h, w), img)


# ---- one batch through every route ------------------------------------------------------------------------------
W, H = 256, 200


def _mixed_frames():
    """RGBA frames of one geometry: {name: img}."""
    rng = np.random.default_rng(77)
    n = W * H

    def from_colors(cols, idx):
        return cols[idx].reshape(H, W, 4).astype(np.uint8)

    def gray(vmax):
        v = rng.integers(0, vmax + 1, n, dtype=np.uint8)
        return np.stack([v, v, v, np.full(n, 255, np.uint8)], 1).reshape(H, W, 4)

    f = {}
    cols = rng.integers(0, 256, (1000, 4), dtype=np.uint8)
    cols[:, 3] = rng.choice([255, 128], 1000)
    f["quantise"] = from_colors(cols, rng.integers(0, 1000, n))
    # the decision samples (every 2nd pixel) see 300 colours, the histogram (every pixel) far more than 8192
    t = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    t[:, 3] = 255
    t[::2] = cols[:300][rng.integers(0, 300, n // 2)]
    f["truncation"] = t.reshape(H, W, 4)
    pal = rng.integers(0, 256, (40, 4), dtype=np.uint8)
    pal[:, 3] = 255
    f["palette"] = from_colors(pal, rng.integers(0, 40, n))
    pal[5, 3] = 0
    f["palette_trns"] = from_colors(pal, rng.integers(0, 40, n))
    for vmax in (1, 3, 15, 255):
        f[f"gray{vmax}"] = gray(vmax)
    rgb = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    rgb[:, 3] = 255
    f["rgb"] = rgb.reshape(H, W, 4)
    ga = rng.integers(0, 256, n, dtype=np.uint8)
    f["gray_alpha"] = np.stack([ga, ga, ga, rng.integers(0, 256, n, dtype=np.uint8)], 1).reshape(H, W, 4)
    f["rgba"] = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    return f


@pytest.mark.parametrize("reduce_palette", [True, False])
def test_mixed_batch(gpu_ctx, reduce_palette):
    """Preset 1 lossy (Auto + dither), and the same without palette reduction (where gray frames keep their bit
    depths instead of becoming palettes): one slot one byte too small, one exactly full, info[] as
    quantize_and_filter_dev's."""
    from pixo_b200 import _lib, png
    frames = _mixed_frames()
    names, imgs = list(frames), list(frames.values())
    o = png.PngOptions.from_preset_with_lossless(W, H, 1, False)
    o.reduce_palette = reduce_palette
    given = np.random.default_rng(3).integers(0, 256, (256, 4), dtype=np.uint8)
    pals = [given if nm == "truncation" else None for nm in names]
    wants = [R.encode(img, o, p, parallel_feature=True) for img, p in zip(imgs, pals)]
    order = sorted(range(len(wants)), key=lambda i: len(wants[i]))
    big, fit = order[-1], order[-2]
    assert len(wants[big]) > len(wants[fit])
    cap = len(wants[fit])
    outs, lens, status, infos = _encode_dev(imgs, o, gpu_ctx, cap, palettes=pals)
    for i, nm in enumerate(names):
        assert int(lens[i]) == len(wants[i]), nm
        if i == big:
            assert status[i] == _lib.ERR_OUTPUT_TOO_SMALL and outs[i] == b"", nm
        else:
            assert status[i] == 0 and outs[i] == wants[i], nm
    kinds = {(r.color_type_byte, r.bit_depth, r.trns is not None) for r in infos}
    if reduce_palette:
        assert {(3, 1, False), (3, 2, False), (3, 4, False), (3, 8, False), (3, 8, True), (2, 8, False),
                (4, 8, False), (6, 8, False)} <= kinds, kinds
    else:
        assert {(0, 1, False), (0, 2, False), (0, 4, False), (0, 8, False), (3, 8, True), (2, 8, False),
                (4, 8, False), (6, 8, False)} <= kinds, kinds
    d_in = _frames(imgs, imgs[0].size)
    d_f = torch.empty(len(imgs) * H * (W * 4 + 1), dtype=torch.uint8, device="cuda")
    ref = png.quantize_and_filter_dev(d_in, imgs[0].size, len(imgs), o, d_f, H * (W * 4 + 1), palettes=pals,
                                      ctx=gpu_ctx)
    for a, b in zip(infos, ref):
        assert (a.color_type_byte, a.bit_depth, a.effective_color_type, a.bytes_per_pixel, a.row_bytes, a.trns) == \
            (b.color_type_byte, b.bit_depth, b.effective_color_type, b.bytes_per_pixel, b.row_bytes, b.trns)
        assert (a.palette is None and b.palette is None) or np.array_equal(a.palette, b.palette)


# ---- passes --------------------------------------------------------------------------------------------------------
def test_passes(gpu_ctx):
    """34 4K RGBA frames (33.2 MB of unreduced filtered rows each, 32 to a 1 GiB pass) at preset 0: the second pass
    holds a frame that is written and a noise frame whose slot is too small."""
    from pixo_b200 import _lib, png
    w, h = 3840, 2160
    rng = np.random.default_rng(4)
    kinds = []
    for k in range(3):
        img = np.zeros((h, w, 4), np.uint8)
        img[100 * k:100 * k + 64, 200:264] = rng.integers(0, 256, (64, 64, 4), dtype=np.uint8)
        kinds.append(img)
    noise = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    o = png.PngOptions.from_preset(w, h, 0)
    wants = [R.encode(img, o, parallel_feature=True) for img in kinds]
    want_noise = R.encode(noise, o, parallel_feature=True)
    imgs = [kinds[i % 3] for i in range(33)] + [noise]
    cap = max(len(x) for x in wants) | 1
    assert len(want_noise) > cap
    outs, lens, status, _ = _encode_dev(imgs, o, gpu_ctx, cap)
    for i in range(33):
        assert status[i] == 0 and outs[i] == wants[i % 3], i
    assert status[33] == _lib.ERR_OUTPUT_TOO_SMALL and int(lens[33]) == len(want_noise)


# ---- stream order ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("callers_stream", [False, True])
def test_decode_resize_encode_in_stream_order(gpu_ctx, callers_stream):
    """PNG files decoded into HBM, resized and encoded again on one context with no host synchronisation between
    the calls; the files equal the oracle's encode of the resized pixels."""
    from oracle import png_decode as odec
    from oracle import resize as rz
    from pixo_b200 import decode, png, resize
    from pixo_b200.color import ColorType
    rng = np.random.default_rng(8)
    sw, sh, dw, dh = 301, 203, 160, 120
    srcs = []
    for k in range(4):
        g = (np.arange(sw)[None, :, None] * (k + 1) + np.arange(sh)[:, None, None] * 2 + np.arange(4) * 40) % 256
        img = g.astype(np.uint8).copy()
        img[rng.integers(0, sh, 50), rng.integers(0, sw, 50)] = rng.integers(0, 256, (50, 4), dtype=np.uint8)
        srcs.append(img)
    so = png.PngOptions.from_preset(sw, sh, 1)
    files = [R.encode(img, so, parallel_feature=True) for img in srcs]
    o = png.PngOptions.from_preset(dw, dh, 1)
    # pixo's decode of each file (optimize_alpha cleared the colour of transparent pixels), resized, encoded
    decoded = [np.asarray(odec.decode(f).pixels, np.uint8) for f in files]
    wants = [R.encode(rz.resize(img, sw, sh, dw, dh, 3, 1), o, parallel_feature=True) for img in decoded]
    cap = png.encode_capacity(dw, dh, ColorType.Rgba)
    d_small = torch.empty(4 * dw * dh * 4, dtype=torch.uint8, device="cuda")
    d_out = torch.full((64 + 4 * cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    if callers_stream:
        gpu_ctx.set_stream(s.cuda_stream)
    try:
        batch = decode.decode_png_batch_dev(files, ctx=gpu_ctx, align=1)
        assert batch.offsets == [i * sw * sh * 4 for i in range(4)]
        resize.resize_dev(batch.frames, sw * sh * 4, 4, resize.ResizeOptions(sw, sh, dw, dh, ColorType.Rgba),
                          d_small, dw * dh * 4, ctx=gpu_ctx)
        lens, status, _ = png.encode_on_device(d_small, dw * dh * 4, 4, o, d_out[64:], cap, ctx=gpu_ctx)
    finally:
        if callers_stream:
            gpu_ctx.set_stream(None)
    assert (status == 0).all()
    assert _slots(d_out, 4, cap, lens, status) == wants


# ---- the 2^31-byte limit --------------------------------------------------------------------------------------------
def test_stream_of_2_31_bytes_is_refused_per_frame():
    """Two RGB 65 535 x 32 769 frames with colour-type reduction only: one all gray, whose Gray 8-bit filtered stream
    is 2^31 + 65 536 bytes, gets ERR_UNSUPPORTED and an untouched slot; the other, black, reduces to 1-bit gray
    (268 MB) and is written.  On a context of its own, closed after the test, since its scratch is large."""
    import pixo_b200
    from pixo_b200 import _lib, png
    from pixo_b200.color import ColorType
    w, h = 65535, 32769
    fb = w * h * 3
    d_in = torch.zeros(2 * fb, dtype=torch.uint8, device="cuda")
    d_in[:fb].view(h, w, 3).copy_((torch.arange(w, device="cuda", dtype=torch.int32) % 251).to(torch.uint8)[None, :, None]
                                  .expand(h, w, 3))
    o = png.PngOptions(w, h, ColorType.Rgb, png.FilterStrategy.NoFilter, reduce_color_type=True, compression_level=1)
    small = np.zeros((1, w, 3), np.uint8)
    so = png.PngOptions(w, 1, ColorType.Rgb, png.FilterStrategy.NoFilter, reduce_color_type=True, compression_level=1)
    rows = R.stages(small, so, parallel_feature=True)[4]
    z = pd.deflate_zlib(np.tile(rows, h), 1)
    want = pd.png_file(w, h, 1, 0, z)
    cap = len(want) + 1
    d_out = torch.full((64 + 2 * cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    with pixo_b200.Context(0) as ctx:
        lens, status, infos = png.encode_on_device(d_in, fb, 2, o, d_out[64:], cap, ctx=ctx)
    assert status[0] == _lib.ERR_UNSUPPORTED and int(lens[0]) == 0
    assert h * (infos[0].row_bytes + 1) == (1 << 31) + 65536
    assert status[1] == 0 and (infos[1].color_type_byte, infos[1].bit_depth) == (0, 1)
    assert _slots(d_out, 2, cap, lens, status) == [b"", want]


# ---- launch counts ----------------------------------------------------------------------------------------------------
def test_launch_counts(gpu_ctx):
    """One pass: the filter stage's launches (as quantize_and_filter_dev makes them), DEFLATE's two and the
    container's two.  A refused call launches nothing."""
    from pixo_b200 import PixoError, png
    frames = _mixed_frames()
    imgs = [frames[k] for k in ("quantise", "palette", "gray3", "rgb", "gray_alpha", "rgba")]
    o = png.PngOptions.from_preset_with_lossless(W, H, 1, False)
    d_in = _frames(imgs, imgs[0].size)
    d_f = torch.empty(len(imgs) * H * (W * 4 + 1), dtype=torch.uint8, device="cuda")
    cap = png.encode_capacity(W, H, o.color_type)
    d_out = torch.empty(len(imgs) * cap, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    png.encode_on_device(d_in, imgs[0].size, len(imgs), o, d_out, cap, ctx=gpu_ctx)   # scratch grown
    b0 = gpu_ctx.launch_count
    png.quantize_and_filter_dev(d_in, imgs[0].size, len(imgs), o, d_f, H * (W * 4 + 1), ctx=gpu_ctx)
    stage = gpu_ctx.launch_count - b0
    b1 = gpu_ctx.launch_count
    png.encode_on_device(d_in, imgs[0].size, len(imgs), o, d_out, cap, ctx=gpu_ctx)
    assert gpu_ctx.launch_count - b1 == stage + 2 + 2
    o.optimal_compression = True
    b2 = gpu_ctx.launch_count
    with pytest.raises(PixoError):
        png.encode_on_device(d_in, imgs[0].size, len(imgs), o, d_out, cap, ctx=gpu_ctx)
    with pytest.raises(PixoError):
        png.encode_on_device(d_in, imgs[0].size, len(imgs), o, d_in[1:], cap, ctx=gpu_ctx)
    assert gpu_ctx.launch_count == b2
