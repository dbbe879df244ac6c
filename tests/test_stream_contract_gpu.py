"""When the device entry points run: every `_dev` call is ordered on the context's stream, after the caller's
earlier work on that stream and before its later work, and either returns with its work still queued or
waits for the device, as include/pixo_b200.h lists.  pixo_b200_ctx_set_stream orders a context's work
across a switch, and contexts on one GPU do not disturb each other.

The rest of the suite calls each entry point between two full synchronisations, so it cannot see a call
that reads its input before the stream has written it, writes its output on another stream, leaves the
context's scratch half-written for the next queued call, or starts to block the host.  Here a context
works on one torch stream S.  Inputs are uploaded once at set-up; after that the only synchronisation is
the one under test.  A bounded spin (torch.cuda._sleep) on S holds the stream while the real input is
copied over an input buffer that starts out holding another valid input (another frame of the same
geometry, another frame's oracle coefficients): a call that runs early codes the wrong frame, which shows
as wrong bytes, never as a fault or a range status.  Every output is copied on S and compared byte for
byte with the oracle, whose results are computed before any GPU work is queued.

Every tensor the library touches stays referenced until its stream has drained: torch's caching
allocator does not know about work the library queues."""
import ctypes as C
import os
import re
import threading
import zlib

import numpy as np
import pytest
import torch

import jpeg_progressive_scans as ps
from oracle import jpeg_progressive as jp
from oracle import jpeg_trellis as jt
from oracle import resize as rz
from pixo_b200 import Context, _lib, jpeg, png
from quantize_inputs import make_quantize_input
from reduce_inputs import make_reduce_input
from test_dev_layouts_gpu import GUARD8, POISON16, png_frames, png_ref, scan_bytes
from test_dev_layouts_lossy_gpu import (DITHER, QFORCE, RCT, RPAL, quantize_ref, reduce_ref, same_lossless,
                                        same_quantized)
from test_resize_gpu import frame as resize_frame

pytestmark = pytest.mark.gpu

# A spin of 2^29 SM cycles: about 0.27 s at the H100's 1.98 GHz boost clock, longer at any lower clock.
# Far longer than the host side of any call here, so a call that returns while it runs did not wait.
DELAY = 1 << 29
COEF_TRELLIS = 2

# The spec of include/pixo_b200.h: entry points that return while the work queued before them is still
# running, and entry points that wait for it (and for part of their own work) before they return.
QUEUED = {"jpeg_coefficients_dev", "jpeg_encode_dev", "png_filter_dev", "png_filter_rows_dev", "adler32_dev",
          "resize_dev", "jpeg_band_histogram_dev", "jpeg_band_entropy_dev_async", "jpeg_band_splice_dev_async"}
WAITS = {"jpeg_coefficients_dev+trellis", "jpeg_trellis_quantize_dev", "jpeg_progressive_scans_dev",
         "jpeg_entropy_encode_dev", "jpeg_band_last_dc", "jpeg_band_entropy_dev", "jpeg_band_splice_dev",
         "png_reduce_filter_dev", "png_quantize_filter_dev"}


def lib():
    return _lib.load()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def P(t):
    return None if t is None else t.data_ptr()


def sleep_on(s, cycles=DELAY):
    with torch.cuda.stream(s):
        torch.cuda._sleep(cycles)


# ---- cases: staged inputs, named calls, device outputs, a check ------------------------------------------
class Case:
    def __init__(self):
        self.stage = []   # (dst, src): dst holds another valid input until src is copied over it on the stream
        self.calls = []   # (entry point, fn(ctx) -> status)
        self.outs = []    # device tensors the calls write
        self.host = {}    # what the calls return in host memory
        self.check = None   # fn(host copies of outs, self.host)

    def input(self, real, stale):
        assert real.shape == stale.shape and not np.array_equal(real, stale)
        dst, src = dev(stale), dev(real)
        self.stage.append((dst, src))
        return dst

    def out(self, t):
        self.outs.append(t)
        return t

    def call(self, name, fn):
        self.calls.append((name, fn))


def poisoned(n, dtype=torch.uint8, value=GUARD8):
    return torch.full((n,), value, dtype=dtype, device="cuda")


def jpeg_frame(po, w, h, ct, kind, seed):
    ch = 3 if ct == 2 else 1
    if kind == "noise":
        return po.gen_noise(w, h, ch, seed)
    g = np.roll(po.gen_gradient_rgb(w, h).reshape(h, w * 3), seed, axis=0).reshape(-1)
    return g if ch == 3 else g[seed % 3::3].copy()


def quant(q=80):
    _, _, lq, cq = jpeg.quant_tables(q)
    return lq, cq


def staged_coefficients(c, real, stale):
    """The three arrays as staged inputs (None for an empty chroma array: Gray)."""
    return [c.input(np.ascontiguousarray(a, np.int16).reshape(-1), np.ascontiguousarray(b, np.int16).reshape(-1))
            if len(a) else None for a, b in zip(real, stale)]


def same_arrays(got, want, what):
    for g, w_, name in zip(got, want, ("Y", "Cb", "Cr")):
        g = g.reshape(-1, 64)
        assert g.shape == w_.shape and np.array_equal(g, w_), (what, name, int((g != w_).sum()))


def coef_case(po, w, h, ct, ss, hist=True, seed=1):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    want = po.jpeg_coefficients(real, w, h, ct, ss, 80)
    want_hist = po.jpeg_histograms(*want, w, h, ct, ss)
    ny, nc = len(want[0]), len(want[1])
    px = c.input(real, stale)
    dy = c.out(poisoned(ny * 64, torch.int16, POISON16))
    dcb, dcr = (c.out(poisoned(nc * 64, torch.int16, POISON16)) for _ in range(2)) if nc else (None, None)
    dh = c.out(poisoned(536, torch.int64, -1)) if hist else None
    lq, cq = quant()
    c.call("jpeg_coefficients_dev", lambda ctx: lib().pixo_b200_jpeg_coefficients_dev(
        ctx.handle, P(px), real.size, 1, w, h, ct, ss, lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p),
        P(dy), ny * 64, P(dcb), P(dcr), nc * 64, 0, P(dh)))

    def check(o, _):
        same_arrays(o[:1 + 2 * bool(nc)], want, (w, h, ct, ss))
        if hist:
            assert np.array_equal(o[-1].view(np.uint64), want_hist)
    c.check = check
    return c


def trellis_case(po, w, h, ct, ss, q=90, seed=2):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    want = jt.jpeg_coefficients(real, w, h, ct, ss, q)[:3]
    ny, nc = len(want[0]), len(want[1])
    px = c.input(real, stale)
    dy = c.out(poisoned(ny * 64, torch.int16, POISON16))
    dcb, dcr = (c.out(poisoned(nc * 64, torch.int16, POISON16)) for _ in range(2)) if nc else (None, None)
    lq, cq = quant(q)
    c.call("jpeg_coefficients_dev+trellis", lambda ctx: lib().pixo_b200_jpeg_coefficients_dev(
        ctx.handle, P(px), real.size, 1, w, h, ct, ss, lq.ctypes.data_as(_lib.f32p), cq.ctypes.data_as(_lib.f32p),
        P(dy), ny * 64, P(dcb), P(dcr), nc * 64, COEF_TRELLIS, None))
    c.check = lambda o, _: same_arrays(o, want, (w, h, ct, ss, q))
    return c


def trellis_quantize_case(nb=300, seed=3):
    c = Case()
    rng = np.random.default_rng(seed)
    blocks = [(rng.laplace(0, 40, (nb, 64)) * (rng.random((nb, 64)) < 0.6)).astype(np.float32) for _ in range(2)]
    q = rng.integers(1, 100, 64).astype(np.float32)
    want = jt.trellis_quantize_blocks(blocks[0], q, 0.75)
    d = c.input(blocks[0].reshape(-1), blocks[1].reshape(-1))
    out = c.out(poisoned(nb * 64, torch.int16, POISON16))
    c.call("jpeg_trellis_quantize_dev", lambda ctx: lib().pixo_b200_jpeg_trellis_quantize_dev(
        ctx.handle, P(d), nb, q.ctypes.data_as(_lib.f32p), 0.75, P(out), 0))
    c.check = lambda o, _: same_arrays(o, [want], "trellis_quantize_dev")
    return c


def encode_case(po, w, h, ct, ss, q=80, segments=None, seed=4):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    want = scan_bytes(po.jpeg_encode(real, w, h, ct, q, ss))
    cap = (len(want) + 64 + 15) // 16 * 16
    px = c.input(real, stale)
    scan = c.out(poisoned(cap))
    n = c.out(poisoned(1, torch.int64, -1))
    ovf = c.out(poisoned(1, torch.int32, -1))

    def call(ctx):
        old = os.environ.get("PIXO_B200_SEGMENTS")
        if segments:
            os.environ["PIXO_B200_SEGMENTS"] = str(segments)
        try:
            return lib().pixo_b200_jpeg_encode_dev(ctx.handle, P(px), real.size, 1, w, h, ct, q, ss, P(scan), cap,
                                                  P(n), P(ovf))
        finally:
            if segments:
                if old is None:
                    del os.environ["PIXO_B200_SEGMENTS"]
                else:
                    os.environ["PIXO_B200_SEGMENTS"] = old
    c.call("jpeg_encode_dev", call)

    def check(o, _):
        assert int(o[2][0]) == 0 and int(o[1][0]) == len(want), (w, h, ct, ss, q, int(o[2][0]), int(o[1][0]))
        assert o[0][:len(want)].tobytes() == want, (w, h, ct, ss, q)
    c.check = check
    return c


def progressive_case(po, w, h, ct, ss, q=80, seed=5):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    file = jp.encode(real, w, h, ct, ss, q)
    want = [s[5] for s in ps.scans(file)]
    dy, dcb, dcr = staged_coefficients(c, jt.jpeg_coefficients(real, w, h, ct, ss, q)[:3],
                                       jt.jpeg_coefficients(stale, w, h, ct, ss, q)[:3])
    dht = jpeg.dht_array(ps.dht(file))
    ny, nc = jpeg.block_counts(w, h, ct, ss)
    cap = (jpeg.progressive_capacity(w, h) + 15) // 16 * 16
    out = c.out(poisoned(cap))
    lens = c.out(poisoned(7, torch.int64, -1))
    ovf = c.out(poisoned(1, torch.int32, -1))
    c.call("jpeg_progressive_scans_dev", lambda ctx: lib().pixo_b200_jpeg_progressive_scans_dev(
        ctx.handle, P(dy), ny * 64, P(dcb), P(dcr), nc * 64, 1, w, h, ct, ss, dht.ctypes.data, P(out), cap, P(lens),
        P(ovf)))

    def check(o, _):
        assert int(o[2][0]) == 0
        got, k = [], 0
        for n in o[1].tolist():
            got.append(o[0][k:k + n].tobytes())
            k += n
        assert got == want, (w, h, ct, ss)
    c.check = check
    return c


def entropy_encode_case(po, w, h, ct, ss, ri, opt, seed=6):
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    coef = po.jpeg_coefficients(real, w, h, ct, ss, 80)
    want = po.jpeg_encode_from_coefficients(*coef, w, h, ct, 80, ss, ri, opt)
    dy, dcb, dcr = staged_coefficients(c, coef, po.jpeg_coefficients(stale, w, h, ct, ss, 80))
    buf = np.zeros(len(want) + 4096, np.uint8)
    n = C.c_size_t()

    def call(ctx):
        rc = lib().pixo_b200_jpeg_entropy_encode_dev(ctx.handle, P(dy), P(dcb), P(dcr), w, h, ct, 80, ss, ri, int(opt),
                                                     buf.ctypes.data, buf.size, C.byref(n))
        c.host["jpeg"] = buf[:n.value].tobytes()
        return rc
    c.call("jpeg_entropy_encode_dev", call)

    def check(o, host):
        assert host["jpeg"] == want, (w, h, ct, ss, ri, opt)
    c.check = check
    return c


def band_case(po, w, h, ct, ss, seed=7):
    """The host-synchronised band flow: last DC, coding, splice of a whole frame as one band."""
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    coef = po.jpeg_coefficients(real, w, h, ct, ss, 80)
    want = scan_bytes(po.jpeg_encode_from_coefficients(*coef, w, h, ct, 80, ss))
    want_dc = [int(a[-1, 0]) if len(a) else 0 for a in coef]
    dy, dcb, dcr = staged_coefficients(c, coef, po.jpeg_coefficients(stale, w, h, ct, ss, 80))
    ny, nc = len(coef[0]), len(coef[1])
    raw_cap = (w * h * 3 + (2 << 20)) // 16 * 16
    raw = c.out(poisoned(raw_cap))
    out = c.out(poisoned(len(want) + 4096))
    last = (C.c_int32 * 3)(-1, -1, -1)
    zero = (C.c_int32 * 3)(0, 0, 0)
    nbits, tail, out_len = C.c_uint64(), C.c_uint32(), C.c_uint64()

    def last_dc(ctx):
        rc = lib().pixo_b200_jpeg_band_last_dc(ctx.handle, P(dy), P(dcb), P(dcr), ny, nc, last)
        c.host["last_dc"] = list(last)
        return rc
    c.call("jpeg_band_last_dc", last_dc)
    c.call("jpeg_band_entropy_dev", lambda ctx: lib().pixo_b200_jpeg_band_entropy_dev(
        ctx.handle, P(dy), P(dcb), P(dcr), w, h, ct, ss, zero, None, P(raw), raw_cap, C.byref(nbits), C.byref(tail)))

    def splice(ctx):
        rc = lib().pixo_b200_jpeg_band_splice_dev(ctx.handle, P(raw), nbits.value, 0, 0, 1, P(out), out.numel(),
                                                  C.byref(out_len))
        c.host["len"] = out_len.value
        return rc
    c.call("jpeg_band_splice_dev", splice)

    def check(o, host):
        assert host["last_dc"] == want_dc
        assert host["len"] == len(want) and o[1][:len(want)].tobytes() == want, (w, h, ct, ss)
    c.check = check
    return c


def band_async_case(po, w, h, ct, ss, seed=8):
    """The stream-ordered band flow with optimised tables: histogram -> coding -> splice, no host round trip
    (the tables come from the oracle's statistics, known before anything is queued)."""
    c = Case()
    real, stale = jpeg_frame(po, w, h, ct, "noise", seed), jpeg_frame(po, w, h, ct, "smooth", seed)
    coef = po.jpeg_coefficients(real, w, h, ct, ss, 80)
    hist = np.ascontiguousarray(po.jpeg_histograms(*coef, w, h, ct, ss), np.uint64)
    want = scan_bytes(po.jpeg_encode_from_coefficients(*coef, w, h, ct, 80, ss, 0, True))
    dy, dcb, dcr = staged_coefficients(c, coef, po.jpeg_coefficients(stale, w, h, ct, ss, 80))
    zero = (C.c_int32 * 3)(0, 0, 0)
    dh = c.out(poisoned(536, torch.int64, -1))
    seed_dev = torch.zeros(3, dtype=torch.int32, device="cuda")
    raw_cap = (w * h * 3 + (2 << 20)) // 16 * 16
    raw = c.out(poisoned(raw_cap))
    bits_tail = c.out(poisoned(2, torch.int64, -1))
    flags = c.out(torch.zeros(1, dtype=torch.int32, device="cuda"))
    offset = torch.tensor([0, 0, 1], dtype=torch.int64, device="cuda")
    out = c.out(poisoned(len(want) + 4096))
    out_len = c.out(poisoned(1, torch.int64, -1))
    c.keep = (seed_dev, offset)
    c.call("jpeg_band_histogram_dev", lambda ctx: lib().pixo_b200_jpeg_band_histogram_dev(
        ctx.handle, P(dy), P(dcb), P(dcr), w, h, ct, ss, zero, P(dh)))
    c.call("jpeg_band_entropy_dev_async", lambda ctx: lib().pixo_b200_jpeg_band_entropy_dev_async(
        ctx.handle, P(dy), P(dcb), P(dcr), w, h, ct, ss, P(seed_dev), hist.ctypes.data_as(_lib.u64p), P(raw), raw_cap,
        P(bits_tail), P(flags)))
    c.call("jpeg_band_splice_dev_async", lambda ctx: lib().pixo_b200_jpeg_band_splice_dev_async(
        ctx.handle, P(raw), P(offset), P(out), out.numel(), P(out_len), P(flags)))

    def check(o, _):
        assert np.array_equal(o[0].view(np.uint64), hist)
        assert int(o[3][0]) == 0 and int(o[5][0]) == len(want), (int(o[3][0]), int(o[5][0]), len(want))
        assert o[4][:len(want)].tobytes() == want, (w, h, ct, ss)
    c.check = check
    return c


def png_filter_case(po, w, h, bpp, word, seed=9):
    c = Case()
    rb = w * bpp
    real, stale = png_frames(w, h, rb, bpp, 2, seed)
    want = png_ref(po, real, w, h, rb, bpp, word)
    src = c.input(real, stale)
    out = c.out(poisoned(h * (rb + 1)))
    ad = c.out(poisoned(1, torch.int32, -1))
    c.call("png_filter_dev", lambda ctx: lib().pixo_b200_png_filter_dev(
        ctx.handle, P(src), real.size, 1, w, h, rb, bpp, word, P(out), h * (rb + 1), P(ad)))

    def check(o, _):
        assert np.array_equal(o[0], want), (w, h, bpp, word)
        assert int(o[1].view(np.uint32)[0]) == zlib.adler32(want.tobytes())
    c.check = check
    return c


def png_rows_case(po, w, h, bpp, word, r0, r1, seed=10):
    c = Case()
    rb = w * bpp
    real, stale = (f.reshape(h, rb) for f in png_frames(w, h, rb, bpp, 2, seed))
    want = png_ref(po, real.reshape(-1), w, h, rb, bpp, word)[r0 * (rb + 1):r1 * (rb + 1)]
    rows = c.input(real[r0:r1].reshape(-1), stale[r0:r1].reshape(-1))
    above = c.input(real[r0 - 1], stale[r0 - 1])
    out = c.out(poisoned((r1 - r0) * (rb + 1)))
    ad = c.out(poisoned(1, torch.int32, -1))
    c.call("png_filter_rows_dev", lambda ctx: lib().pixo_b200_png_filter_rows_dev(
        ctx.handle, P(rows), P(above), w, h, r1 - r0, rb, bpp, word, P(out), P(ad)))

    def check(o, _):
        assert np.array_equal(o[0], want), (w, h, bpp, word, r0, r1)
        assert int(o[1].view(np.uint32)[0]) == zlib.adler32(want.tobytes())
    c.check = check
    return c


def adler_case(n=(1 << 20) + 3, seed=11):
    c = Case()
    rng = np.random.default_rng(seed)
    real, stale = rng.integers(0, 256, n, dtype=np.uint8), rng.integers(0, 256, n, dtype=np.uint8)
    src = c.input(real, stale)
    out = c.out(poisoned(1, torch.int32, -1))
    c.call("adler32_dev", lambda ctx: lib().pixo_b200_adler32_dev(ctx.handle, P(src), n, P(out)))

    def check(o, _):
        assert int(o[0].view(np.uint32)[0]) == zlib.adler32(real.tobytes())
    c.check = check
    return c


def resize_case(sw, sh, dw, dh, ct, alg, seed=12):
    c = Case()
    real, stale = resize_frame(sw, sh, ct, seed, "noise"), resize_frame(sw, sh, ct, seed, "edges")
    want = rz.resize(real, sw, sh, dw, dh, ct, alg)
    src = c.input(real, stale)
    out = c.out(poisoned(want.size))
    c.call("resize_dev", lambda ctx: lib().pixo_b200_resize_dev(
        ctx.handle, P(src), real.size, 1, sw, sh, dw, dh, ct, alg, P(out), want.size))

    def check(o, _):
        assert np.array_equal(o[0], want), (sw, sh, dw, dh, ct, alg, int((o[0] != want).sum()))
    c.check = check
    return c


def reduce_case(po, w, h, ct, word, seed=13):
    """A palette frame: the stale one has other colours, so reading it changes the palette."""
    c = Case()
    real, stale = make_reduce_input("pal", w, h, ct + 1, seed, 16), make_reduce_input("pal", w, h, ct + 1, seed + 1, 5)
    want, wf = reduce_ref(po, real, w, h, ct, word)
    assert want.color_type_byte == 3
    src = c.input(real, stale)
    out = c.out(poisoned(h * (w * (ct + 1) + 1)))
    ad = c.out(poisoned(1, torch.int32, -1))
    infos = (png._Reduced * 1)()
    c.call("png_reduce_filter_dev", lambda ctx: lib().pixo_b200_png_reduce_filter_dev(
        ctx.handle, P(src), real.size, 1, w, h, ct, word, infos, P(out), out.numel(), P(ad)))
    c.check = lambda o, _: same_lossless(png.ReducedImage._from_c(infos[0]), want, o[0][:wf.size], wf,
                                         o[1].view(np.uint32)[0], (w, h, ct, hex(word)))
    return c


def quantize_case(po, w, h, ct, word, m=16, seed=14):
    """A quantised frame of 3 m colours (Force, so the stale frame, of other colours, quantises too)."""
    c = Case()
    real = make_quantize_input("pal", w, h, ct + 1, seed, 3 * m)
    stale = make_quantize_input("pal", w, h, ct + 1, seed + 1, 3 * m)
    want = quantize_ref(po, real, w, h, ct, word, m)
    assert want[0]
    src = c.input(real, stale)
    out = c.out(poisoned(h * (w * (ct + 1) + 1)))
    ad = c.out(poisoned(1, torch.int32, -1))
    infos = (png._Reduced * 1)()
    c.call("png_quantize_filter_dev", lambda ctx: lib().pixo_b200_png_quantize_filter_dev(
        ctx.handle, P(src), real.size, 1, w, h, ct, word, m, None, None, infos, P(out), out.numel(), P(ad)))
    c.check = lambda o, _: same_quantized(png.ReducedImage._from_c(infos[0]), want, o[0][:h * (w + 1)],
                                          o[1].view(np.uint32)[0], (w, h, ct, hex(word)))
    return c


CASES = {
    "coef-420-tma": lambda po: coef_case(po, 256, 256, 2, 1),
    "coef-444-clamped": lambda po: coef_case(po, 530, 41, 2, 0),
    "coef-gray-tma": lambda po: coef_case(po, 256, 256, 0, 0),
    "coef-gray-clamped": lambda po: coef_case(po, 530, 41, 0, 0, hist=False),
    "trellis-420": lambda po: trellis_case(po, 530, 41, 2, 1),
    "trellis-444": lambda po: trellis_case(po, 256, 256, 2, 0),
    "trellis-gray": lambda po: trellis_case(po, 530, 41, 0, 0),
    "tquant": lambda po: trellis_quantize_case(),
    "encode-420-tma": lambda po: encode_case(po, 256, 256, 2, 1),
    "encode-420-clamped": lambda po: encode_case(po, 530, 41, 2, 1),
    "encode-444-tma": lambda po: encode_case(po, 256, 256, 2, 0),
    "encode-gray-clamped": lambda po: encode_case(po, 530, 41, 0, 0),
    "encode-420-segments": lambda po: encode_case(po, 1000, 600, 2, 1, segments=5),
    "progressive-420": lambda po: progressive_case(po, 333, 217, 2, 1),
    "progressive-gray": lambda po: progressive_case(po, 200, 75, 0, 0),
    "entropy-420-opt-rst": lambda po: entropy_encode_case(po, 333, 222, 2, 1, 7, True),
    "entropy-444": lambda po: entropy_encode_case(po, 200, 75, 2, 0, 0, False),
    "entropy-gray-opt": lambda po: entropy_encode_case(po, 257, 129, 0, 0, 0, True),
    "band-420": lambda po: band_case(po, 333, 222, 2, 1),
    "band-gray": lambda po: band_case(po, 257, 129, 0, 0),
    "bandasync-420": lambda po: band_async_case(po, 333, 222, 2, 1),
    "bandasync-444": lambda po: band_async_case(po, 200, 75, 2, 0),
    "filter-rgba-adaptive": lambda po: png_filter_case(po, 1000, 70, 4, 6 | 0x100),
    "filter-gray-bigrams": lambda po: png_filter_case(po, 999, 70, 1, 8),
    "rows-rgb": lambda po: png_rows_case(po, 1001, 70, 3, 5, 17, 50),
    "adler32": lambda po: adler_case(),
    "resize-nearest": lambda po: resize_case(1297, 35, 640, 71, 3, 0),
    "resize-bilinear": lambda po: resize_case(200, 100, 333, 77, 2, 1),
    "resize-lanczos3-small": lambda po: resize_case(256, 256, 97, 61, 3, 2),
    "resize-lanczos3-large": lambda po: resize_case(16384, 64, 12000, 64, 3, 2),        # 0.7 MB of tables
    "resize-lanczos3-tables": lambda po: resize_case(262144, 1, 65535, 1, 0, 2),        # 7.9 MB of tables
    "reduce-palette": lambda po: reduce_case(po, 131, 70, 3, 6 | RCT | RPAL),
    "quantize-dither": lambda po: quantize_case(po, 160, 130, 3, 4 | QFORCE | DITHER),
}
# the entry points each kind of case calls, in order
ENTRIES = {
    "coef": ["jpeg_coefficients_dev"], "trellis": ["jpeg_coefficients_dev+trellis"],
    "tquant": ["jpeg_trellis_quantize_dev"], "encode": ["jpeg_encode_dev"],
    "progressive": ["jpeg_progressive_scans_dev"], "entropy": ["jpeg_entropy_encode_dev"],
    "band": ["jpeg_band_last_dc", "jpeg_band_entropy_dev", "jpeg_band_splice_dev"],
    "bandasync": ["jpeg_band_histogram_dev", "jpeg_band_entropy_dev_async", "jpeg_band_splice_dev_async"],
    "filter": ["png_filter_dev"], "rows": ["png_filter_rows_dev"], "adler32": ["adler32_dev"],
    "resize": ["resize_dev"], "reduce": ["png_reduce_filter_dev"], "quantize": ["png_quantize_filter_dev"],
}


def make_case(po, name):
    c = CASES[name](po)
    assert [n for n, _ in c.calls] == ENTRIES[name.split("-")[0]], name
    return c


@pytest.fixture(scope="module")
def lane():
    """A context of its own whose work goes on the torch stream S (the shared test context keeps its own)."""
    ctx, s = Context(0), torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    yield ctx, s
    s.synchronize()
    ctx.set_stream(None)
    ctx.close()


def run_case(ctx, s, c, delay=True, probe=False):
    """Stage c's inputs on s (behind the delay), make its calls, copy its outputs on s, synchronise once
    and check.  probe: a delay before every call instead, and {entry point: the delay queued before it was
    still running when it returned}."""
    torch.cuda.synchronize()   # the set-up uploads (default stream) have landed
    with torch.cuda.stream(s):
        if delay and not probe:
            torch.cuda._sleep(DELAY)
        for dst, src in c.stage:
            dst.copy_(src)
    busy = {}
    for name, fn in c.calls:
        if probe:
            sleep_on(s)
            delayed = torch.cuda.Event()
            delayed.record(s)
        _lib.check(ctx.handle, fn(ctx))
        if probe:
            busy[name] = not delayed.query()
    with torch.cuda.stream(s):
        res = [o.clone() for o in c.outs]
    s.synchronize()
    c.check([r.cpu().numpy() for r in res], c.host)
    return busy


# ---- 1. producer -> entry point -> consumer on one stream -----------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_entry_point_ordered_on_the_callers_stream(po, lane, name):
    """The input is written on S behind the delay, the call reads it, S copies the outputs: the outputs
    equal the oracle only if the call ran in between, on S."""
    ctx, s = lane
    before = ctx.host_fallbacks
    run_case(ctx, s, make_case(po, name))
    assert ctx.host_fallbacks == before


# ---- 2. which entry points block ------------------------------------------------------------------------
def test_the_spec_lists_name_every_device_entry_point():
    """QUEUED and WAITS together hold every device-pointer entry point of the header (and band_last_dc,
    which reads device arrays), once, and the cases below call each of them."""
    with open(os.path.join(os.path.dirname(__file__), "..", "include", "pixo_b200.h")) as f:
        declared = set(re.findall(r"\bint pixo_b200_(\w+_dev(?:_async)?)\(", f.read())) | {"jpeg_band_last_dc"}
    assert {n.split("+")[0] for n in QUEUED | WAITS} == declared
    assert not QUEUED & WAITS
    called = {e for name in CASES for e in ENTRIES[name.split("-")[0]]}
    assert called == QUEUED | WAITS, called ^ (QUEUED | WAITS)


@pytest.mark.parametrize("name", list(CASES))
def test_entry_point_returns_queued_or_waits_as_documented(po, lane, name):
    """On a context already warmed with the same geometry (growing scratch synchronises by design), a call
    queued behind the delay returns while the delay still runs, or only once it has finished, as QUEUED
    and WAITS say.  Two warm-up runs: Lanczos3 stages its tables in two pinned buffers in turn."""
    ctx, s = lane
    c = make_case(po, name)
    run_case(ctx, s, c, delay=False)
    run_case(ctx, s, c, delay=False)
    busy = run_case(ctx, s, c, probe=True)
    for entry, b in busy.items():
        assert entry in QUEUED | WAITS, entry
        if entry in QUEUED:
            assert b, f"{entry} ({name}) waited for the device"
        else:
            assert not b, f"{entry} ({name}) returned with work still queued"


# ---- 3. a queue of mixed calls on one context -----------------------------------------------------------
def test_mixed_queue_without_synchronisation(po):
    """Twelve calls on a fresh context behind one delay, one synchronisation at the end; every output is the
    oracle's.  The first call of each kind allocates its scratch (the context has none yet, so nothing is
    freed and nothing waits); after that no call before the trellis grows a buffer it shares with an
    earlier one: the 333 x 222 encode reuses the 1000 x 600 encode's coefficient and entropy scratch, the
    97 x 61 Lanczos3 call uploads its tables into the region the 640 x 71 call's kernels read (and reuses
    its intermediate), and the second PNG filter and the Adler-32 reuse the first filter's accumulators,
    all while the delay still holds the stream, which the test checks.  The trellis and the PNG reduction
    then wait for the device, and the last encode reuses the first one's scratch."""
    builds = [lambda: encode_case(po, 1000, 600, 2, 1, seed=41), lambda: encode_case(po, 333, 222, 2, 1, seed=42),
              lambda: resize_case(300, 200, 640, 71, 2, 2, seed=44), lambda: resize_case(256, 256, 97, 61, 3, 2, seed=43),
              lambda: png_filter_case(po, 1000, 70, 4, 6, seed=45), lambda: adler_case(5553, seed=46),
              lambda: png_filter_case(po, 500, 40, 3, 8, seed=47), lambda: coef_case(po, 530, 41, 2, 1, hist=False, seed=48),
              lambda: coef_case(po, 256, 256, 2, 0, seed=49), lambda: trellis_case(po, 256, 256, 2, 1, seed=50),
              lambda: reduce_case(po, 131, 70, 3, 6 | RCT | RPAL, seed=51), lambda: encode_case(po, 640, 480, 2, 0, seed=52)]
    cases = [b() for b in builds]
    ctx, s = Context(0), torch.cuda.Stream()
    try:
        ctx.set_stream(s.cuda_stream)
        torch.cuda.synchronize()
        sleep_on(s, 2 * DELAY)
        delayed = torch.cuda.Event()
        delayed.record(s)
        with torch.cuda.stream(s):
            for c in cases:
                for dst, src in c.stage:
                    dst.copy_(src)
        for c in cases:
            for name, fn in c.calls:
                if name == "jpeg_coefficients_dev+trellis":
                    assert not delayed.query(), "a call queued before the trellis waited for the stream"
                _lib.check(ctx.handle, fn(ctx))
        with torch.cuda.stream(s):
            res = [[o.clone() for o in c.outs] for c in cases]
        s.synchronize()
        for c, r in zip(cases, res):
            c.check([x.cpu().numpy() for x in r], c.host)
        assert ctx.host_fallbacks == 0
    finally:
        s.synchronize()
        ctx.close()


# ---- 4. stream switch -----------------------------------------------------------------------------------
@pytest.fixture
def switching(po):
    """A context on stream A, warmed with the geometry of the PNG case it then gets, and a second stream B."""
    ctx, a, b = Context(0), torch.cuda.Stream(), torch.cuda.Stream()
    ctx.set_stream(a.cuda_stream)
    run_case(ctx, a, png_filter_case(po, 1000, 70, 4, 6, seed=60), delay=False)
    c = png_filter_case(po, 1000, 70, 4, 6, seed=61)
    yield ctx, a, b, c
    a.synchronize()
    b.synchronize()
    ctx.close()


def queue_behind_delay(ctx, a, c):
    """The delay, c's input and c's call on A; A is still busy when this returns."""
    torch.cuda.synchronize()
    sleep_on(a)
    with torch.cuda.stream(a):
        for dst, src in c.stage:
            dst.copy_(src)
    for _, fn in c.calls:
        _lib.check(ctx.handle, fn(ctx))
    assert not a.query()


def download(ctx, t):
    host = np.empty(t.numel() * t.element_size(), np.uint8)
    _lib.check(ctx.handle, lib().pixo_b200_download(ctx.handle, host.ctypes.data, P(t), host.size))
    return host


@pytest.mark.parametrize("to", ["other", "own"])
def test_download_after_a_stream_switch_returns_the_finished_bytes(switching, to):
    """png_filter_dev on A behind the delay into a poisoned output, then a switch to B (or back to the
    context's own stream) that does not block the host, then pixo_b200_download through the context: it
    syncs the context's current stream, which must be ordered after A's work."""
    ctx, a, b, c = switching
    queue_behind_delay(ctx, a, c)
    ctx.set_stream(b.cuda_stream if to == "other" else None)
    assert not a.query(), "set_stream blocked the host"
    out = download(ctx, c.outs[0])
    ad = download(ctx, c.outs[1]).view(np.int32)
    c.check([out, ad], c.host)


def test_sync_after_a_stream_switch_covers_the_old_stream(switching):
    ctx, a, b, c = switching
    queue_behind_delay(ctx, a, c)
    ctx.set_stream(b.cuda_stream)
    ctx.sync()
    assert a.query(), "ctx.sync() after the switch returned while the old stream still held the context's work"
    c.check([o.cpu().numpy() for o in c.outs], c.host)


def test_switch_to_the_current_stream_changes_nothing(switching):
    ctx, a, b, c = switching
    queue_behind_delay(ctx, a, c)
    ctx.set_stream(a.cuda_stream)
    assert not a.query(), "set_stream to the current stream blocked the host"
    c.check([download(ctx, c.outs[0]), download(ctx, c.outs[1]).view(np.int32)], c.host)


def test_calls_on_both_sides_of_a_switch(po):
    """jpeg_encode_dev on A behind the delay, a switch, jpeg_encode_dev of another frame of the same
    geometry on B (the same transform and entropy scratch): both scans are the oracle's.  This checks the
    spec, not the switch's ordering: without it B's call runs to the end inside A's delay and A's call
    after it, so the shared scratch is never used by both at once and the scans are right either way.
    The download and sync tests above are the ones that fail when the new stream does not wait."""
    ctx, a, b = Context(0), torch.cuda.Stream(), torch.cuda.Stream()
    try:
        ctx.set_stream(a.cuda_stream)
        run_case(ctx, a, encode_case(po, 1000, 600, 2, 1, seed=70), delay=False)
        first, second = encode_case(po, 1000, 600, 2, 1, seed=71), encode_case(po, 1000, 600, 2, 1, seed=72)
        queue_behind_delay(ctx, a, first)
        ctx.set_stream(b.cuda_stream)
        with torch.cuda.stream(b):
            for dst, src in second.stage:
                dst.copy_(src)
        for _, fn in second.calls:
            _lib.check(ctx.handle, fn(ctx))
        with torch.cuda.stream(a):
            ra = [o.clone() for o in first.outs]
        with torch.cuda.stream(b):
            rb = [o.clone() for o in second.outs]
        a.synchronize()
        b.synchronize()
        first.check([x.cpu().numpy() for x in ra], first.host)
        second.check([x.cpu().numpy() for x in rb], second.host)
        assert ctx.host_fallbacks == 0
    finally:
        a.synchronize()
        b.synchronize()
        ctx.close()


# ---- 5. concurrent contexts on one GPU ------------------------------------------------------------------
def test_concurrent_contexts_on_one_gpu(po):
    """Three host threads, each with its own context and stream on device 0, start together and run the
    same short sequence twice: q100 noise encode (dense k_huff units and look-back chains), a dithered
    quantisation (k_quant_dither's row hand-off between CTAs), COEF_TRELLIS, Lanczos3 and the progressive
    scans.  The bounded waits must not run out while another context's kernels share the SMs: every output
    is the oracle's, no call fails, no frame goes to the host coder."""
    def sequence(seed):
        return [encode_case(po, 640, 480, 2, 1, q=100, seed=seed),
                quantize_case(po, 160, 130, 3, 4 | QFORCE | DITHER, seed=seed),
                trellis_case(po, 530, 41, 2, 1, seed=seed),
                resize_case(256, 256, 97, 61, 3, 2, seed=seed),
                progressive_case(po, 333, 217, 2, 1, seed=seed)]
    workers = [(Context(0), torch.cuda.Stream(), sequence(80 + t) + sequence(90 + t)) for t in range(3)]
    for _, _, cases in workers:
        for c in cases:
            for dst, src in c.stage:
                dst.copy_(src)
    torch.cuda.synchronize()
    barrier = threading.Barrier(len(workers), timeout=120)
    errors = []

    def work(ctx, s, cases):
        try:
            ctx.set_stream(s.cuda_stream)
            barrier.wait()
            for c in cases:
                for name, fn in c.calls:
                    rc = fn(ctx)
                    if rc:
                        errors.append((name, rc, lib().pixo_b200_last_error(ctx.handle)))
                        return
            s.synchronize()
        except Exception as e:   # reported below, after every thread has finished
            errors.append(e)

    threads = [threading.Thread(target=work, args=w) for w in workers]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    try:
        assert not errors, errors
        for ctx, _, cases in workers:
            assert ctx.host_fallbacks == 0
            for c in cases:
                c.check([o.cpu().numpy() for o in c.outs], c.host)
    finally:
        for ctx, s, _ in workers:
            s.synchronize()
            ctx.close()
