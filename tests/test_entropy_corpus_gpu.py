"""The device entropy stage (k_huff, k_huff<RAW> + k_seg_*, K3) on constructed coefficients
(tests/coef_corpus.py): byte-identical to the oracle, round-tripped by the independent decoder
(tests/jpeg_scan_decode.py), and rejecting coefficients that have no baseline code."""
import ctypes as C
import threading

import numpy as np
import pytest

import coef_corpus as cc
import jpeg_scan_decode as jd
import pixo_b200
from pixo_b200 import ColorType, _lib, jpeg, parallel
from pixo_b200.jpeg import JpegOptions, Subsampling
from test_entropy_corpus import band_border_straddle, band_slices, restart_intervals, straddling

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was silently finished by the host entropy coder"


def upload(case):
    import torch
    y, cb, cr = case[:3]
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() if len(a) else None for a in (y, cb, cr)]
    torch.cuda.synchronize()
    return d


def opts(case, ri=0, opt=False):
    w, h, ct, ss = case[3:7]
    return JpegOptions(w, h, ColorType(ct), 80, Subsampling(ss), ri or None, opt)


def oracle(po, case, ri=0, opt=False):
    y, cb, cr, w, h, ct, ss = case
    return po.jpeg_encode_from_coefficients(y, cb, cr, w, h, ct, 80, ss, ri, opt)


def check_decodes(jpg, case, seen):
    if jpg not in seen:
        d = jd.decode(jpg)
        assert np.array_equal(d.y, case[0]) and np.array_equal(d.cb, case[1]) and np.array_equal(d.cr, case[2])
        seen.add(jpg)


@pytest.mark.parametrize("segments", [None, "2", "5"])
@pytest.mark.parametrize("name", sorted(cc.MATRIX))
def test_device_coder_on_the_corpus(po, gpu_ctx, monkeypatch, name, segments):
    if segments:
        monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
    seen = set()
    for ct, ss in cc.geometries():
        case = cc.MATRIX[name](ct, ss)
        d = upload(case)
        for ri in restart_intervals(case):
            if ri and name in cc.NO_RESTART:
                continue
            for opt in (False, True):
                ref = oracle(po, case, ri, opt)
                assert jpeg.entropy_encode_dev(*d, opts(case, ri, opt), ctx=gpu_ctx) == ref, (ct, ss, ri, opt)
                if segments is None:
                    check_decodes(ref, case, seen)


@pytest.mark.parametrize("segments", [None, "2"])
def test_device_coder_block_lengths_stuffing_and_borders(po, gpu_ctx, monkeypatch, segments):
    """Blocks of 511..545 and 1658 bits at chunk lanes 0/15/31; an all-0xFF scan; 0xFF bytes across
    the chunk border and (two segments) the segment border; restart padding completing 0xFF bytes.
    (The band border: test_ff_byte_across_a_band_border.)"""
    if segments:
        monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
    case, _ = cc.block_lengths()
    cases = [(case, 0), (cc.stuffing_gray(), 0), cc.restart_padding()]
    cases += [(straddling(po, 64, 32)[0], 0), (straddling(po, 96, 48)[0], 0)]   # 96 MCUs in 2 segments: 48
    for case, ri in cases:
        for opt in (False, True):
            assert jpeg.entropy_encode_dev(*upload(case), opts(case, ri, opt), ctx=gpu_ctx) == oracle(po, case, ri, opt)


@pytest.mark.parametrize("ct,ss", cc.geometries())
def test_dense_frames_recode_on_the_gpu(po, monkeypatch, ct, ss):
    """Every block near 1658 bits: a scan of 2x (4:2:0) to 4x (gray) the pixel bytes, beyond the first
    pass's buffer.  Unsegmented: k_huff twice (bit 0, then the exact size).  Forced segments: the
    segments outgrow their shares (bit 2), then the frame is coded unsegmented.  No host coder; an
    output that holds the headers but not the scan is reported, nothing written past it."""
    case = cc.dense(ct, ss)
    w, h = case[3:5]
    ref = oracle(po, case)
    pixels = w * h * (3 if ct == 2 else 1)
    assert len(ref) > 1.5 * pixels
    d = upload(case)
    with pixo_b200.Context(0) as ctx:
        # unsegmented: k_huff twice; segmented: k_huff<RAW> + 4 splice kernels, then k_huff twice
        for segments, least in ((None, 2), ("4", 5 + 2)):
            if segments:
                monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
            l0 = ctx.launch_count
            assert jpeg.entropy_encode_dev(*d, opts(case), ctx=ctx) == ref
            assert ctx.launch_count - l0 >= least, segments
            for opt in (False, True):
                assert jpeg.entropy_encode_dev(*d, opts(case, 0, opt), ctx=ctx) == oracle(po, case, 0, opt)
        assert ctx.host_fallbacks == 0
        out_cap = len(ref) // 2
        buf = np.full(out_cap + 256, 0xA5, np.uint8)
        n = C.c_size_t(0)
        ptr = lambda t: None if t is None else t.data_ptr()
        rc = _lib.load().pixo_b200_jpeg_entropy_encode_dev(ctx.handle, ptr(d[0]), ptr(d[1]), ptr(d[2]), w, h, ct, 80,
                                                           ss, 0, 0, buf.ctypes.data, out_cap, C.byref(n))
        assert rc == _lib.ERR_OUTPUT_TOO_SMALL
        assert (buf[out_cap:] == 0xA5).all()


def device_coders(ctx, case, world):
    import torch
    y, cb, cr, w, h, ct, ss = case
    coders, keep = [], []
    for b, by, bcb, bcr in band_slices(case, world):
        t = [torch.from_numpy(np.ascontiguousarray(a if len(a) else np.zeros((1, 64), np.int16))).cuda()
             for a in (by, bcb, bcr)]
        keep.append(t)
        coders.append(parallel.DeviceBandCoder(ctx, t[0], t[1] if ct else None, t[2] if ct else None, w,
                                               max(b.px_row1 - b.px_row0, 1), ct, ss, len(by), len(bcb)))
    torch.cuda.synchronize()
    return coders, keep


@pytest.mark.parametrize("name,ct,ss,world,segments", [("dc_chains", 2, 1, 3, None), ("symbol_sweep", 2, 0, 2, "2"),
                                                       ("dc_climb", 0, 0, 4, None), ("dc_chains", 0, 0, 3, "3")])
def test_bands_on_one_gpu(po, gpu_ctx, monkeypatch, name, ct, ss, world, segments):
    """Constructed bands (+-2047 DC differences across every band border, the seeds carry them):
    parallel.encode_tiled_local equals the oracle, with standard and optimised tables."""
    if segments:
        monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
    case = cc.MATRIX[name](ct, ss)
    coders, _keep = device_coders(gpu_ctx, case, world)
    for opt in (False, True):
        got = parallel.encode_tiled_local(coders, *case[3:5], ct, 80, ss, opt)
        assert got == oracle(po, case, 0, opt), opt


@pytest.mark.parametrize("segments", [None, "2"])
def test_ff_byte_across_a_band_border(po, gpu_ctx, monkeypatch, segments):
    """The byte holding the last bits of band 0 and the first of band 1 is 0xFF: k_huff<RAW> and the
    splice kernels (inherited bits, stuffing) must produce the bytes one coder would."""
    if segments:
        monkeypatch.setenv("PIXO_B200_SEGMENTS", segments)
    case, ref, _ = band_border_straddle(po)
    coders, _keep = device_coders(gpu_ctx, case, 2)
    assert len(coders) == 2 and coders[0].ny == 48
    for opt in (False, True):
        assert parallel.encode_tiled_local(coders, *case[3:5], 0, 80, 0, opt) == oracle(po, case, 0, opt), opt
    assert parallel.encode_tiled_local(coders, *case[3:5], 0, 80, 0) == ref


@pytest.mark.parametrize("ct,ss", [(2, 1), (0, 0)])
def test_dense_band_coded_in_segments(po, gpu_ctx, monkeypatch, ct, ss):
    """A dense band whose segments outgrow their shares (pixel bytes + 4 KiB each) is coded again as
    one string in the same synchronous call: two passes of k_huff<RAW> + k_band_totals.  With a raw_cap
    too small for that string the call reports the bits it needs and writes nothing past raw_cap; a
    second call with those bytes (rounded up to 256) + 512 succeeds."""
    import torch
    monkeypatch.setenv("PIXO_B200_SEGMENTS", "2")
    case = cc.dense(ct, ss)
    coders, _keep = device_coders(gpu_ctx, case, 2)
    lib = _lib.load()
    c = coders[1]
    seed = (C.c_int32 * 3)(*[int(v) for v in coders[0].last_dc()])

    def code(cap):
        raw = torch.full((cap + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
        nbits, tail = C.c_uint64(), C.c_uint32()
        l0 = gpu_ctx.launch_count
        rc = lib.pixo_b200_jpeg_band_entropy_dev(gpu_ctx.handle, c._p(c.d_y), c._p(c.d_cb), c._p(c.d_cr), *c.geo, seed,
                                                 None, raw.data_ptr(), cap, C.byref(nbits), C.byref(tail))
        assert (raw[cap:].cpu().numpy() == 0xA5).all()
        return rc, nbits.value, gpu_ctx.launch_count - l0

    w, bh = c.geo[:2]
    rc, nbits, launches = code((w * bh * 3 + (1 << 20)) // 16 * 16)      # DeviceBandCoder's first capacity
    assert rc == 0 and launches == 4, (rc, launches)                      # the segmented pass overflowed
    need = (nbits + 7) // 8
    rc, n2, launches = code((need - 4096) // 16 * 16)    # room for the segments' shares, not for one string
    assert rc == _lib.ERR_OUTPUT_TOO_SMALL and n2 == nbits and launches == 4, (rc, launches)
    rc, n3, _ = code((need + 255) // 256 * 256 + 512)
    assert rc == 0 and n3 == nbits
    assert parallel.encode_tiled_local(coders, *case[3:5], ct, 80, ss) == oracle(po, case)


def test_stream_ordered_band_flow_on_the_corpus(po, monkeypatch):
    """One constructed frame through pixo_b200_jpeg_band_*_async with three thread ranks."""
    import torch
    monkeypatch.setenv("PIXO_B200_SEGMENTS", "2")
    case = cc.dc_chains(2, 1)
    world = 3
    nonempty = [len(s[1]) > 0 for s in band_slices(case, world)]
    comm = parallel.ThreadComm(world)
    res, errs = {}, []

    def work(rank):
        try:
            torch.cuda.set_device(0)
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                ctx = pixo_b200.Context(0)
                ctx.set_stream(stream.cuda_stream)
                coders, _keep = device_coders(ctx, case, world)
                parts, _ = parallel.tiled_scan_parts_async(coders[rank], nonempty, rank, world, comm=comm)
                if rank == 0:
                    res["jpg"] = parallel.assemble_tiled(parts, None, *case[3:5], 2, 80, 1)
                assert ctx.host_fallbacks == 0
        except BaseException as e:   # noqa: BLE001 - re-raised in the main thread
            errs.append(e)
            comm.barrier.abort()

    ths = [threading.Thread(target=work, args=(r,)) for r in range(world)]
    for t in ths: t.start()
    for t in ths: t.join()
    assert not errs, errs
    assert res["jpg"] == oracle(po, case)


def test_band_histograms_on_the_symbol_sweep(po, gpu_ctx):
    """K3 per band (pixo_b200_jpeg_band_histogram_dev, seeded with the previous band's last DCs)
    equals the host twin band by band, and the bands sum to the oracle's whole-frame histogram."""
    for ct, ss in cc.geometries():
        case = cc.symbol_sweep(ct, ss)
        coders, _keep = device_coders(gpu_ctx, case, 3)
        hosts = [parallel.HostBandCoder(by, bcb, bcr, case[3], max(b.px_row1 - b.px_row0, 1), ct, ss)
                 for b, by, bcb, bcr in band_slices(case, 3)]
        last = np.stack([c.last_dc() for c in hosts])
        total = np.zeros(536, np.uint64)
        for r, (dc, hc) in enumerate(zip(coders, hosts)):
            seed = parallel.dc_seeds(last, [True] * 3, r)
            got = dc.histogram(seed).cpu().numpy().astype(np.uint64)
            assert np.array_equal(got, hc.histogram(seed).numpy().astype(np.uint64)), r
            total += got
        assert np.array_equal(total, po.jpeg_histograms(*case))


def test_out_of_range_coefficients_on_the_device(po, gpu_ctx, monkeypatch):
    """Every device entry point that takes coefficients: ERR_INVALID_ARGUMENT from the synchronous ones
    (nothing written past the output), bit 3 in the stream-ordered flags, and the context codes the next
    valid input correctly.  A segmented pass passes bit 3 on, so it is not retried unsegmented."""
    import torch
    lib = _lib.load()
    good = cc.zero_runs(2, 1)
    w, h = good[3:5]
    bads = []
    for arr, idx, val in ((0, (3, 1), 1024), (2, (1, 12), -32768), (1, (2, 0), 2500), (0, (5, 63), -1024)):
        b = [a.copy() for a in good[:3]]
        b[arr][idx] = val
        bads.append((tuple(b) + good[3:], 0))
    reset = [a.copy() for a in good[:3]]
    reset[1][1, 0] = 2000
    reset[1][2:, 0] = 3000                      # differences of 2000, 1000, 0...; 3000 after a reset at MCU 2
    reset = tuple(reset) + good[3:]
    bads.append((reset, 2))
    assert jpeg.entropy_encode_dev(*upload(reset), opts(reset), ctx=gpu_ctx) == oracle(po, reset)
    ref = oracle(po, good)
    for case, ri in bads:
        d = upload(case)
        for opt in (False, True):
            out_cap = 1 << 16
            buf = np.full(out_cap + 256, 0xA5, np.uint8)
            n = C.c_size_t(0)
            rc = lib.pixo_b200_jpeg_entropy_encode_dev(gpu_ctx.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                                       w, h, 2, 80, 1, ri, int(opt), buf.ctypes.data, out_cap, C.byref(n))
            assert rc == _lib.ERR_INVALID_ARGUMENT, (ri, opt)
            assert (buf[out_cap:] == 0xA5).all()
        assert jpeg.entropy_encode_dev(*upload(good), opts(good), ctx=gpu_ctx) == ref
        if ri:
            continue
        # bands: the synchronous call, the stream-ordered one (flag bit 3), K3 (clamps, no error)
        coder = device_coders(gpu_ctx, case, 1)[0][0]
        s = (C.c_int32 * 3)(0, 0, 0)
        raw = torch.full((1 << 20,), 0xA5, dtype=torch.uint8, device="cuda")
        nbits, tail = C.c_uint64(), C.c_uint32()
        cap = (1 << 20) - 4096
        rc = lib.pixo_b200_jpeg_band_entropy_dev(gpu_ctx.handle, coder._p(coder.d_y), coder._p(coder.d_cb),
                                                 coder._p(coder.d_cr), *coder.geo, s, None, raw.data_ptr(), cap,
                                                 C.byref(nbits), C.byref(tail))
        assert rc == _lib.ERR_INVALID_ARGUMENT
        assert (raw[cap:].cpu().numpy() == 0xA5).all()
        flags = torch.zeros(1, dtype=torch.int32, device="cuda")
        bt = torch.zeros(2, dtype=torch.int64, device="cuda")
        seed = torch.zeros(3, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        _lib.check(gpu_ctx.handle, lib.pixo_b200_jpeg_band_entropy_dev_async(
            gpu_ctx.handle, coder._p(coder.d_y), coder._p(coder.d_cb), coder._p(coder.d_cr), *coder.geo,
            seed.data_ptr(), None, raw.data_ptr(), raw.numel(), bt.data_ptr(), flags.data_ptr()))
        gpu_ctx.sync()
        assert int(flags.item()) & 8
        hist = coder.histogram(np.zeros(3, np.int32)).cpu().numpy()
        assert hist.sum() > 0
    coders, _keep = device_coders(gpu_ctx, good, 2)
    assert parallel.encode_tiled_local(coders, w, h, 2, 80, 1) == ref
    monkeypatch.setenv("PIXO_B200_SEGMENTS", "5")
    d = upload(bads[0][0])
    buf = np.zeros(1 << 16, np.uint8)
    n = C.c_size_t(0)
    l0 = gpu_ctx.launch_count
    rc = lib.pixo_b200_jpeg_entropy_encode_dev(gpu_ctx.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                               w, h, 2, 80, 1, 0, 0, buf.ctypes.data, buf.size, C.byref(n))
    assert rc == _lib.ERR_INVALID_ARGUMENT
    assert gpu_ctx.launch_count - l0 == 5      # k_huff<RAW> + four splice kernels, once
    assert jpeg.entropy_encode_dev(*upload(good), opts(good), ctx=gpu_ctx) == ref
