"""A short tour of every kernel on small inputs, for compute-sanitizer (memcheck / racecheck):
    compute-sanitizer --tool memcheck python tools/sanitize_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import pixo_b200
from pixo_b200 import jpeg, png, synthetic, ColorType
from pixo_b200.jpeg import JpegOptions, Subsampling
from pixo_b200.png import FilterStrategy, PngOptions

ctx = pixo_b200.Context(0)
rng = np.random.default_rng(3)
for (w, h) in [(333, 222), (640, 480), (1000, 70)]:
    img = synthetic.noise(w, h, 3, 9)
    for ss in (Subsampling.S420, Subsampling.S444):
        for q, opt in ((80, False), (100, True)):
            out = jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, q, ss, None, opt), ctx=ctx)
            assert out[:2] == b"\xff\xd8" and out[-2:] == b"\xff\xd9"
    g = synthetic.noise(w, h, 1, 4)
    jpeg.encode(g, JpegOptions(w, h, ColorType.Gray, 85, Subsampling.S444), ctx=ctx)
    frames = np.stack([synthetic.noise(w, h, 3, k) for k in range(5)])
    jpeg.encode_batch(frames, JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420), ctx=ctx)
    for bpp, ct in ((4, 3), (2, 1), (3, 2)):
        px = rng.integers(0, 256, (h, w, bpp), dtype=np.uint8)
        if bpp in (2, 4):
            px[..., -1] = np.where(rng.random((h, w)) < 0.3, 0, px[..., -1])
        for st in (FilterStrategy.Adaptive, FilterStrategy.AdaptiveFast, FilterStrategy.Bigrams, FilterStrategy.Paeth):
            png.apply_filters(px.reshape(-1), w, h, bpp, PngOptions(w, h, ColorType(ct), st, True), with_adler=True, ctx=ctx)
    png.adler32(img, ctx=ctx)
# ---- round 2: restart intervals, segmented coding (k_huff<RAW> + k_seg_*), bands of one frame (band entropy +
# splice, also segmented), the PNG row-band entry point and the mixed-row scoring paths ----------------------
import torch
from pixo_b200 import _lib, parallel
lib = _lib.load()
w, h = 1024, 512
img = synthetic.noise(w, h, 3, 11)
img.reshape(h, w * 3)[100:300] = synthetic.gradient_rgb(w, h).reshape(h, w * 3)[100:300]
plain = jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420), ctx=ctx)
jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420, 7), ctx=ctx)          # restart interval
for S in ("1", "3", "16", "200"):
    os.environ["PIXO_B200_SEGMENTS"] = S
    seg = jpeg.encode(img, JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420), ctx=ctx)
    assert seg == plain, S
    # bands of the frame, each band's raw string itself segmented
    dev = torch.device("cuda", 0)
    _, _, lq, cq = jpeg.quant_tables(80)
    coders, keep = [], []
    for b in parallel.plan_bands(w, h, 3):
        bh = b.px_row1 - b.px_row0
        d_y = torch.empty((max(b.y_blocks, 1), 64), dtype=torch.int16, device=dev)
        d_cb = torch.empty((max(b.c_blocks, 1), 64), dtype=torch.int16, device=dev)
        d_cr = torch.empty_like(d_cb)
        px = torch.from_numpy(np.ascontiguousarray(parallel.band_pixels(img, w, h, 3, b)).reshape(-1)).to(dev)
        keep.append(px)
        torch.cuda.synchronize(dev)
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
            ctx.handle, px.data_ptr(), px.numel(), 1, w, bh, 2, 1, lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p),
            d_y.data_ptr(), b.y_blocks * 64, d_cb.data_ptr(), d_cr.data_ptr(), b.c_blocks * 64, 0, None))
        coders.append(parallel.DeviceBandCoder(ctx, d_y, d_cb, d_cr, w, bh, 2, 1, b.y_blocks, b.c_blocks))
    ctx.sync()
    tiled = parallel.encode_tiled_local(coders, w, h, 2, 80, 1)
    assert tiled == plain, ("bands", S)
del os.environ["PIXO_B200_SEGMENTS"]
# PNG: flat rows next to noise rows (both scoring routes and their switches), and a row band with the row above
hh, ww, bpp = 70, 1024, 4
rows = rng.integers(0, 256, (hh, ww * bpp), dtype=np.uint8)
rows[::3] = 17
for st in (FilterStrategy.Adaptive, FilterStrategy.AdaptiveFast, FilterStrategy.MinSum):
    whole, _ = png.apply_filters(rows.reshape(-1), ww, hh, bpp, PngOptions(ww, hh, ColorType.Rgba, st), with_adler=True, ctx=ctx)
    d_rows = torch.from_numpy(rows).to(dev)
    torch.cuda.synchronize(dev)
    d_out = torch.empty(30 * (ww * bpp + 1), dtype=torch.uint8, device=dev)
    d_ad = torch.zeros(1, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    png.apply_filters_rows_dev(d_rows[20:50].contiguous().reshape(-1), d_rows[19].contiguous(), ww, hh, 30, ww * bpp, bpp, st,
                               d_out, d_ad, ctx=ctx)
    ctx.sync()
    assert np.array_equal(d_out.cpu().numpy(), whole.reshape(hh, ww * bpp + 1)[20:50].reshape(-1)), st
# PNG colour-type / palette reduction: every branch of the analysis, index, pack and filter kernels
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from reduce_inputs import make_reduce_input  # noqa: E402
for kind, ch, n, (ww, hh) in (("pal", 3, 2, (9, 5)), ("pal", 4, 3, (7, 6)), ("pal", 4, 17, (65, 9)),
                              ("palblk", 4, 256, (300, 40)), ("pal", 3, 257, (300, 40)), ("graypal", 3, 4, (33, 7)),
                              ("graypal", 4, 200, (33, 7)), ("opaque", 4, 0, (70, 33)), ("grayalpha", 4, 0, (70, 33)),
                              ("noise", 4, 0, (70, 33)), ("noise", 1, 0, (20, 9)), ("noise", 2, 0, (20, 9))):
    px = make_reduce_input(kind, ww, hh, ch, 1, n)
    for rct, rpal in ((True, True), (True, False), (False, True)):
        for st in (FilterStrategy.Adaptive, FilterStrategy.Bigrams):
            png.reduce_and_filter(px, PngOptions(ww, hh, ColorType(ch - 1), st, True, rct, rpal), ctx=ctx)
frames = [make_reduce_input(k, 300, 40, 4, 2, n) for k, n in (("pal", 5), ("opaque", 0), ("pal", 300), ("grayalpha", 0))]
d_in = torch.from_numpy(np.concatenate(frames)).to(dev)
d_out = torch.empty(4 * 40 * (300 * 4 + 1), dtype=torch.uint8, device=dev)
d_ad = torch.zeros(4, dtype=torch.int32, device=dev)
torch.cuda.synchronize(dev)
png.reduce_and_filter_dev(d_in, 300 * 40 * 4, 4, PngOptions.from_preset(300, 40, 1), d_out, 40 * (300 * 4 + 1), d_ad, ctx=ctx)
ctx.sync()
# JPEG progressive scans with the tables and raw strings from the host (the wait for the bit counts): the
# measuring kernels, k_prog_place, k_prog_emit_at and the splice with k_seg_fit, with trellis and plain
# coefficients, optimised and standard tables, gray / 4:4:4 / 4:2:0, a batch and caller arrays
for (ww, hh) in ((333, 222), (17, 9)):
    for ct, ss in ((2, Subsampling.S420), (2, Subsampling.S444), (0, Subsampling.S444)):
        ch = 1 if ct == 0 else 3
        im = synthetic.noise(ww, hh, ch, 5)
        for opt, tr, rst in ((True, True, None), (False, False, 3)):
            jpeg.encode_progressive(im, JpegOptions(ww, hh, ColorType(ct), 80, ss, rst, opt, True, tr), ctx=ctx)
frames = np.stack([synthetic.noise(200, 120, 3, k) for k in range(3)])
jpeg.encode_progressive_batch(frames, JpegOptions.max(200, 120, 80), ctx=ctx)
yb = np.zeros((40000, 64), np.int16)
yb[::9000, 1] = 5
yb[7, 63] = -3
d_yb = torch.from_numpy(yb).to(dev)
jpeg.progressive_scans_dev(d_yb, None, None, 8 * 400, 8 * 100, ColorType.Gray, Subsampling.S444, ctx=ctx)
ctx.sync()
# the queued progressive stage (encode_progressive_dev): k_prog_dht_tables, k_prog_place, k_prog_emit_at and
# k_seg_fit, with a frame that fits, one whose stuffed bytes do not and one whose raw bytes do not
d_fr = torch.from_numpy(np.stack([np.full(64 * 48 * 3, 90, np.uint8), synthetic.noise(64, 48, 3, 6),
                                  synthetic.noise(64, 48, 3, 7)])).to(dev)
for cap, (opt, tr) in ((16384, (True, True)), (16384, (False, False)), (2048, (True, False))):
    d_o = torch.empty(3 * cap, dtype=torch.uint8, device=dev)
    d_l = torch.empty((3, 7), dtype=torch.int64, device=dev)
    d_f = torch.empty(3, dtype=torch.int32, device=dev)
    d_t = torch.empty((3, jpeg.DHT_BYTES), dtype=torch.uint8, device=dev)
    jpeg.encode_progressive_dev(d_fr, 64 * 48 * 3, 3, JpegOptions(64, 48, ColorType.Rgb, 100, Subsampling.S420, None,
                                                                  opt, True, tr), d_o, cap, d_l, d_f, d_t, ctx=ctx)
    ctx.sync()
# resize: every kernel at every pixel size, the wide and byte nearest copies, and Lanczos3 in one band and,
# for a tall frame whose one destination row needs 280 MB of intermediate, in column chunks
from pixo_b200 import resize as rs  # noqa: E402
for ct in range(4):
    for alg in range(3):
        for (sw, sh, dw, dh) in ((37, 29, 100, 71), (97, 61, 37, 29), (1, 1, 3, 2), (1024, 5, 3, 2)):
            px = rng.integers(0, 256, sw * sh * (ct + 1), dtype=np.uint8)
            o = rs.ResizeOptions.builder(sw, sh).dst(dw, dh).color_type(ColorType(ct)).algorithm(rs.ResizeAlgorithm(alg)).build()
            rs.resize(px, o, ctx=ctx)
            d_px = torch.from_numpy(np.concatenate([px, px])).to(dev)
            d_o = torch.empty(2 * dw * dh * (ct + 1) + 1, dtype=torch.uint8, device=dev)
            torch.cuda.synchronize(dev)
            rs.resize_dev(d_px if ct % 2 else d_px[1:], px.size, 2 if ct % 2 else 1, o, d_o[1:], dw * dh * (ct + 1),
                          ctx=ctx)
            ctx.sync()
tall = rng.integers(0, 256, 16 * 70000 * 4, dtype=np.uint8)
rs.resize(tall, rs.ResizeOptions.builder(16, 70000).dst(1000, 3).algorithm(rs.ResizeAlgorithm.Lanczos3).build(), ctx=ctx)
# ---- the stages whose scratch layouts go through pixo::Layout and no earlier part reaches: PNG quantisation
# (Auto, Force, dither, a given palette; host and device entry points), COEF_TRELLIS and the trellis entry
# point, device encodes with optimised tables and a restart interval, the device entropy entry point with
# optimised tables, and the stream-ordered band flow on one rank ---------------------------------------------
from pixo_b200.png import QuantizationMode  # noqa: E402
for (ww, hh) in ((70, 33), (300, 40)):
    cols = rng.integers(0, 256, (500, 4), dtype=np.uint8)
    px = cols[rng.integers(0, 500, ww * hh)].reshape(-1)
    pal = rng.integers(0, 256, (16, 4), dtype=np.uint8)
    for mode, dith in ((QuantizationMode.Auto, False), (QuantizationMode.Force, False), (QuantizationMode.Force, True)):
        o = PngOptions(ww, hh, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, mode, 64, dith)
        png.quantize_and_filter(px, o, ctx=ctx)
        png.quantize_and_filter(px, o, palette=pal, ctx=ctx)
    d_px = torch.from_numpy(np.concatenate([px, px])).to(dev)
    d_out = torch.empty(2 * hh * (ww * 4 + 1), dtype=torch.uint8, device=dev)
    d_ad = torch.zeros(2, dtype=torch.int32, device=dev)
    torch.cuda.synchronize(dev)
    o = PngOptions(ww, hh, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, QuantizationMode.Force, 64, True)
    png.quantize_and_filter_dev(d_px, px.size, 2, o, d_out, hh * (ww * 4 + 1), d_ad, palettes=[None, pal], ctx=ctx)
    ctx.sync()
im = synthetic.noise(333, 222, 3, 6)
jpeg.compute_all_coefficients(im, 333, 222, ColorType.Rgb, Subsampling.S420, 80, ctx=ctx, use_trellis=True)
jpeg.compute_all_coefficients(im[: 333 * 222], 333, 222, ColorType.Gray, Subsampling.S444, 90, ctx=ctx, use_trellis=True)
d_dct = torch.from_numpy(rng.normal(0, 200, (5000, 64)).astype(np.float32)).to(dev)
torch.cuda.synchronize(dev)
jpeg.trellis_quantize_dev(d_dct, np.full(64, 16, np.float32), ctx=ctx)
ctx.sync()
ww, hh, nf, cap = 640, 480, 3, 2 << 20
d_fr = torch.from_numpy(np.stack([synthetic.noise(ww, hh, 3, k) for k in range(nf)]).reshape(-1)).to(dev)
d_scan = torch.empty(nf * cap, dtype=torch.uint8, device=dev)
d_len = torch.zeros(nf, dtype=torch.int64, device=dev)
d_ovf = torch.zeros(nf, dtype=torch.int32, device=dev)
d_dht = torch.empty(nf * jpeg.DHT_BYTES, dtype=torch.uint8, device=dev)
torch.cuda.synchronize(dev)
for rst, opt in ((5, True), (None, True), (5, False)):
    jpeg.encode_dev(d_fr, ww * hh * 3, nf, JpegOptions(ww, hh, ColorType.Rgb, 80, Subsampling.S420, rst, opt), d_scan, cap,
                    d_len, d_ovf, d_dht, ctx=ctx)
ctx.sync()
coef = [torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        for a in jpeg.compute_all_coefficients(im, 333, 222, ColorType.Rgb, Subsampling.S420, 80, ctx=ctx)]
torch.cuda.synchronize(dev)
for rst in (None, 4):
    jpeg.entropy_encode_dev(*coef, JpegOptions(333, 222, ColorType.Rgb, 80, Subsampling.S420, rst, True), ctx=ctx)
fw, fh = 1024, 512
frame = synthetic.noise(fw, fh, 3, 12)
want = jpeg.encode(frame, JpegOptions(fw, fh, ColorType.Rgb, 80, Subsampling.S420), ctx=ctx)
for S in ("1", "3"):
    os.environ["PIXO_B200_SEGMENTS"] = S
    b = parallel.plan_bands(fw, fh, 1)[0]
    d_y = torch.empty((b.y_blocks, 64), dtype=torch.int16, device=dev)
    d_cb = torch.empty((b.c_blocks, 64), dtype=torch.int16, device=dev)
    d_cr = torch.empty_like(d_cb)
    px = torch.from_numpy(np.ascontiguousarray(frame).reshape(-1)).to(dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.synchronize(dev)
    with torch.cuda.stream(stream):
        ctx.set_stream(stream.cuda_stream)
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
            ctx.handle, px.data_ptr(), px.numel(), 1, fw, fh, 2, 1, lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p),
            d_y.data_ptr(), b.y_blocks * 64, d_cb.data_ptr(), d_cr.data_ptr(), b.c_blocks * 64, 0, None))
        coder = parallel.DeviceBandCoder(ctx, d_y, d_cb, d_cr, fw, fh, 2, 1, b.y_blocks, b.c_blocks)
        parts, _ = parallel.tiled_scan_parts_async(coder, [True], 0, 1)
        got = parallel.assemble_tiled(parts, None, fw, fh, 2, 80, 1)
        stream.synchronize()
    ctx.set_stream(None)
    assert got == want, ("stream-ordered band", S)
del os.environ["PIXO_B200_SEGMENTS"]
# ---- baseline JPEG decoding: k_jdec_scan / k_jdec_idct / k_jdec_color over real, truncated, corrupt and constructed
# files, gray, 4:4:4, 4:2:0 and odd sampling factors ----------------------------------------------------------
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from pixo_b200 import decode as jdec  # noqa: E402
from jpeg_decode_corpus import constructed, corrupted, truncations  # noqa: E402
small = jpeg.encode(synthetic.noise(37, 21, 3, 2), JpegOptions(37, 21, ColorType.Rgb, 90, Subsampling.S420, 3), ctx=ctx)
gray = jpeg.encode(synthetic.noise(w, h, 1, 4), JpegOptions(w, h, ColorType.Gray, 85, Subsampling.S444), ctx=ctx)
files = [plain, small, gray]
files += truncations(small) + corrupted(small, 5, 50) + [constructed(k) for k in range(100)]
jdec.decode_jpeg_batch_dev(files, ctx=ctx)
jdec.decode_jpeg(plain, ctx=ctx)
ctx.sync()
# ---- PNG decoding: k_png_crc / k_png_inflate / k_png_unfilter / k_png_expand over real, truncated, bit-flipped and
# constructed files: every colour type and depth, hand-built DEFLATE, failing files between good ones ------------------
import glob  # noqa: E402
from png_decode_corpus import bit_flips, corpus  # noqa: E402
from png_decode_corpus import truncations as png_truncations  # noqa: E402
gold = sorted(glob.glob(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                                     "p*.png")))[:12]
pngs = [open(p, "rb").read() for p in gold]
pngs += [f for n, f in corpus() if n != "huge_claim_small_idat"] + png_truncations(pngs[0]) + bit_flips(pngs[1], 20, 3)
jdec.decode_png_batch_dev(pngs, ctx=ctx)
jdec.decode_png(pngs[0], ctx=ctx)
ctx.sync()
# ---- well-formed files past one row group and with odd sampling: a tall Paeth RGBA16 PNG (bpp 8 at every group's
# first row) and a 3x2-sampled JPEG with restart intervals ------------------------------------------------------
from decode_inputs import geometry, jfif, png_image, qtable, safe_tails, sparse_coefs  # noqa: E402
tall, _ = png_image(45, 200, 16, 6, 1, filters=(4,))
jdec.decode_png(tall, ctx=ctx)
comps = [(3, 2, qtable(1)), (1, 1, qtable(2)), (2, 1, qtable(3))]
mw, mh, bpm = geometry(101, 53, comps)
odd = jfif(101, 53, comps, safe_tails(sparse_coefs(mw * mh * bpm, 4), bpm, 3, mw * mh), restart=3)
jdec.decode_jpeg(odd, ctx=ctx)
ctx.sync()
print("tour done")
