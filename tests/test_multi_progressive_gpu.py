"""One frame's progressive scans (pixo's max preset) tiled over several ranks in MCU-row bands: every band is
transformed, trellis-quantised and coded on its own (pixo_b200_jpeg_band_dev_progressive*), and the file is byte for
byte the one a single GPU - and pixo - writes.  Ranks are bands of this process on one GPU, or threads with a
context each (ThreadComm); with >= 2 devices the same frame also goes through NCCL, one process per GPU."""
import ctypes as C
import hashlib
import json
import os
import socket
import sys
import threading

import numpy as np
import pytest
import torch

from conftest import ROOT
from pixo_b200 import ColorType, _lib, jpeg, parallel
from pixo_b200.jpeg import JpegOptions, Subsampling
from progressive_inputs import make_progressive_input
from trellis_inputs import make_trellis_input

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
M = 0x7FFF
C_i32, C_u32 = C.c_int32, C.c_uint32


@pytest.fixture(autouse=True)
def _no_silent_host_fallback(gpu_ctx):
    before = gpu_ctx.host_fallbacks
    yield
    assert gpu_ctx.host_fallbacks == before, "a frame was finished by the host entropy coder"


def opts(w, h, ct, q, ss, opt=True, trellis=True):
    return JpegOptions(w, h, ColorType(ct), q, Subsampling(ss), None, bool(opt), True, bool(trellis))


def coders_for(ctx, frame, o, world):
    """The frame's bands (plan_bands) as ProgressiveBandCoders on ctx's device."""
    w, h, ct, ss = o.width, o.height, int(o.color_type), int(o.subsampling)
    bpp = 1 if ct == 0 else 3
    bands = parallel.plan_bands(w, h, world, gray=ct == 0, s420=ss == 1)
    rows = torch.from_numpy(np.ascontiguousarray(frame, np.uint8).reshape(h, w * bpp)).to(f"cuda:{ctx.device}")
    return [parallel.progressive_band_coder(ctx, rows[b.px_row0:b.px_row1].contiguous().reshape(-1), w, h, ct, ss,
                                            o.quality, o.trellis_quant, bands, r) for r, b in enumerate(bands)]


def tiled(ctx, frame, o, world):
    return parallel.encode_progressive_tiled_local(coders_for(ctx, frame, o, world), o)


def _manifest(sub):
    with open(os.path.join(GOLD, sub, "manifest.json")) as f:
        return json.load(f)["jpeg"]


# ---- real pixo -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("e", _manifest("trellis"), ids=lambda e: e["file"])
def test_pixo_max_preset_goldens(gpu_ctx, e):
    img = make_trellis_input(e["kind"], e["w"], e["h"], 1 if e["ct"] == 0 else 3, e["seed"])
    o = opts(e["w"], e["h"], e["ct"], e["q"], e["s420"])
    want = open(os.path.join(GOLD, "trellis", e["file"]), "rb").read()
    for world in (2, 3, 5, 8):
        assert tiled(gpu_ctx, img, o, world) == want, world


@pytest.mark.parametrize("e", _manifest("progressive"), ids=lambda e: e["file"])
def test_eob_run_fixtures(gpu_ctx, e):
    """Y AC EOB runs of 32 766 - 69 999 blocks, carried across the bands."""
    o = opts(e["w"], e["h"], e["ct"], e["q"], e["s420"])
    img = make_progressive_input(e)
    want = open(os.path.join(GOLD, "progressive", e["file"]), "rb").read()
    for world in (2, 3, 5, 8):
        assert tiled(gpu_ctx, img, o, world) == want, world


# ---- against the single-GPU path -------------------------------------------------------------------------------
@pytest.mark.parametrize("opt,trellis", [(1, 1), (1, 0), (0, 1), (0, 0)])
@pytest.mark.parametrize("ct,ss", [(2, 1), (2, 0), (0, 0)], ids=["420", "444", "gray"])
def test_option_matrix(po, gpu_ctx, ct, ss, opt, trellis):
    for w, h in ((1, 1), (17, 9), (333, 217), (1297, 35)):
        for q in (1, 50, 100):
            o = opts(w, h, ct, q, ss, opt, trellis)
            frame = po.gen_noise(w, h, 1 if ct == 0 else 3, 7 * w + q).reshape(-1)
            want = jpeg.encode_progressive(frame, o, ctx=gpu_ctx)
            for world in range(1, 9):
                assert tiled(gpu_ctx, frame, o, world) == want, (w, h, q, world)


def test_thread_ranks_with_collectives(po):
    """The collective flow (tiled_progressive_parts) with every rank a thread of this process, a context each:
    all-gathers, the all-reduce of the statistics and the gather to dst are real exchanges of device tensors."""
    import pixo_b200
    for (w, h, ct, ss, world, dst) in ((640, 400, 2, 1, 4, 0), (333, 217, 0, 0, 3, 2), (100, 40, 2, 0, 5, 1)):
        o = opts(w, h, ct, 85, ss)
        frame = po.gen_noise(w, h, 1 if ct == 0 else 3, w + world).reshape(-1)
        comm = parallel.ThreadComm(world)
        res, errs = {}, []

        def work(rank):
            try:
                torch.cuda.set_device(0)
                ctx = pixo_b200.Context(0)
                coder = coders_for(ctx, frame, o, world)[rank]
                got = parallel.encode_progressive_tiled(coder, o, rank, world, dst=dst, comm=comm)
                assert (got is None) == (rank != dst)
                if got is not None:
                    res["jpg"] = got
                assert ctx.host_fallbacks == 0
            except BaseException as e:   # noqa: BLE001 - re-raised in the main thread
                errs.append(e)
                comm.barrier.abort()

        ths = [threading.Thread(target=work, args=(r,)) for r in range(world)]
        for t in ths: t.start()
        for t in ths: t.join()
        assert not errs, errs
        assert res["jpg"] == jpeg.encode_progressive(frame, o), (w, h, ct)


# ---- constructed coefficient arrays ------------------------------------------------------------------------------
def constructed(nb, busy, rng):
    """nb Y blocks, empty but for the DC and the AC of the blocks in `busy`."""
    y = np.zeros((nb, 64), np.int16)
    y[:, 0] = rng.integers(-300, 300, nb)
    for b in busy:
        y[b, 1:] = rng.integers(-40, 40, 63) * (rng.random(63) < 0.3)
        y[b, 5] = 7
    return y


def band_coders(ctx, y, cuts):
    d = torch.from_numpy(y).cuda()
    n = y.shape[0]
    return [parallel.ProgressiveBandCoder(ctx, (d[lo:max(hi, lo + 1)], d[:1], d[:1]), hi - lo, 0, lo, 0, n, 0)
            for lo, hi in zip(cuts, cuts[1:])]


@pytest.mark.parametrize("run", [M - 1, M, M + 1])
def test_runs_ending_on_band_edges(gpu_ctx, run):
    """Gray frames whose Y AC runs of 0x7FFF - 1, 0x7FFF and 0x7FFF + 1 empty blocks end exactly on a band's first
    and on its last block, coded band by band and compared with progressive_scans_dev on the whole arrays."""
    rng = np.random.default_rng(run)
    w = 8 * 256
    first, second = 3, 3 + run + 1
    nb = ((second + 2 * run + 40) // 256 + 1) * 256
    h = 8 * (nb // 256)
    busy = [first, second, nb - 1]
    y = constructed(nb, busy, rng)
    o = JpegOptions(w, h, ColorType.Gray, 80, Subsampling.S444, None, False, True, False)
    d = torch.from_numpy(y).cuda()
    out, lens, ovf = jpeg.progressive_scans_dev(d, None, None, w, h, ColorType.Gray, Subsampling.S444, ctx=gpu_ctx)
    gpu_ctx.sync()
    assert not ovf.cpu().numpy().any()
    lens = lens.cpu().numpy()[0]
    want = jpeg.progressive_file(o, None, out.cpu().numpy(), lens)
    edges = [second, second + 1, first + 1, second - 1, nb - 1, nb - 2]   # runs end on a first or a last block
    for cuts in ([0, second, nb], [0, first + 1, second, nb], [0, first + 1, second + 1, nb],
                 [0, 2, first + 1, first + 1, second, second + M, nb - 1, nb], [0] + sorted(edges) + [nb]):
        seg, ln, dht = parallel.tiled_progressive_parts_local(band_coders(gpu_ctx, y, cuts))
        assert ln == [int(v) for v in lens], cuts
        assert jpeg.progressive_file(o, dht, seg.cpu().numpy(), ln) == want, cuts


def test_band_calls_are_ordered_on_the_callers_stream_and_wait():
    """The three band calls run in order on the context's stream and wait for it before they return: each reads an
    input that a copy queued behind a spin on that stream writes (one that runs early codes other coefficients), and
    returns with the stream drained.  Outputs are compared with a fully synchronised run."""
    import pixo_b200
    from test_stream_contract_gpu import sleep_on
    nb = 4096
    real = constructed(nb, [3, 100, 2000, nb - 1], np.random.default_rng(5))
    stale = constructed(nb, [7, 50], np.random.default_rng(6))
    ref = parallel.ProgressiveBandCoder(pixo_b200.Context(0), (torch.from_numpy(real).cuda(),) * 3, nb, 0, 0, 0, nb, 0)
    want_sum = ref.summary()
    want_bits, want_tails = ref.code([0, 0, 0], [0] * 4)
    want = [ref.splice(k, want_bits[k], 0, 0, True).cpu().numpy() for k in range(7)]
    want_dht = ref.dht.cpu().numpy()
    s = torch.cuda.Stream()
    ctx = pixo_b200.Context(0)
    ctx.set_stream(s.cuda_stream)
    d, src = torch.from_numpy(stale).cuda(), torch.from_numpy(real).cuda()
    coder = parallel.ProgressiveBandCoder(ctx, (d, d, d), nb, 0, 0, 0, nb, 0)

    def real_behind_a_spin():
        d.copy_(torch.from_numpy(stale))
        torch.cuda.synchronize()
        sleep_on(s)
        with torch.cuda.stream(s):
            d.copy_(src)

    real_behind_a_spin()
    assert coder.summary() == want_sum and s.query()
    real_behind_a_spin()
    assert coder.code([0, 0, 0], [0] * 4) == (want_bits, want_tails) and s.query()
    assert np.array_equal(coder.dht.cpu().numpy(), want_dht)
    for k in range(7):
        sleep_on(s)
        out = coder.splice(k, want_bits[k], 0, 0, True)
        assert s.query()
        assert np.array_equal(out.cpu().numpy(), want[k]), k
    ctx.set_stream(None)


# ---- a 16 384^2 frame in 8 bands ---------------------------------------------------------------------------------
def test_16k_frame_in_8_bands(po, gpu_ctx):
    from test_jpeg_encode_dev_opts_gpu import big_frames
    w = h = 16384
    f = big_frames(po, w, h, [3], 500)[0]
    o = opts(w, h, 2, 80, 1)
    cap = (w * h * 3 // 2 + 65536) // 16 * 16
    d_px = torch.from_numpy(f).cuda()
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    lens = torch.empty((1, 7), dtype=torch.int64, device="cuda")
    ovf = torch.empty(1, dtype=torch.int32, device="cuda")
    dht = torch.empty((1, jpeg.DHT_BYTES), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    jpeg.encode_progressive_dev(d_px, f.size, 1, o, out, cap, lens, ovf, dht, ctx=gpu_ctx)
    gpu_ctx.sync()
    assert not ovf.cpu().numpy().any()
    whole = jpeg.progressive_file(o, dht.cpu().numpy()[0], out.cpu().numpy(), lens.cpu().numpy()[0])
    del d_px, out
    got = tiled(gpu_ctx, f, o, 8)
    assert hashlib.sha256(got).hexdigest() == hashlib.sha256(whole).hexdigest()


# ---- refusals ------------------------------------------------------------------------------------------------
def test_refusals(gpu_ctx):
    lib = _lib.load()
    h = gpu_ctx.handle
    d = torch.zeros((64, 64), dtype=torch.int16, device="cuda")
    raw = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    seed, carry = (C_i32 * 3)(), (C_u32 * 4)()
    need, nbits, tails = C.c_size_t(), (C.c_uint64 * 7)(), (C.c_uint32 * 7)()
    dc, enc = (C_i32 * 3)(), (C_u32 * 4)()
    p = d.data_ptr()

    def band(y=p, ny=64, raw_ptr=raw.data_ptr(), cap=raw.numel(), s=seed, c=carry, y_base=0, frame=64):
        return lib.pixo_b200_jpeg_band_dev_progressive(h, y, None, None, ny, 0, y_base, 0, frame, 0, s, c, None, None,
                                                       raw_ptr, cap, C.byref(need), nbits, tails)

    def summary(y=p, ny=64):
        return lib.pixo_b200_jpeg_band_dev_progressive_summary(h, y, None, None, ny, 0, 0, 0, dc, enc)

    inv = _lib.ERR_INVALID_ARGUMENT
    assert band(y=None) == inv and summary(y=None) == inv
    assert band(y=p + 2) == inv and summary(y=p + 8) == inv
    assert band(raw_ptr=raw.data_ptr() + 4) == inv and band(raw_ptr=None) == inv
    assert band(frame=63) == inv
    assert band(s=(C_i32 * 3)(20000, 0, 0)) == inv
    assert band(c=(C_u32 * 4)(2 * 10 + 1, 0, 0, 0), y_base=0) == inv   # a carry past the band's first block
    d[17, 9] = 16384
    assert band() == inv and summary() == inv
    d[17, 9] = -16383
    assert summary() == 0 and list(enc) == [(18 << 1) | 1, 0, 0, 0]   # block 17, its last non-zero below Se 10
    # too small a raw capacity: the bits needed, then the retry
    assert band(cap=256) == _lib.ERR_OUTPUT_TOO_SMALL
    small = list(nbits)
    assert need.value > 256 and small[0] > 0
    assert band(cap=need.value) == 0 and list(nbits) == small
    coder = parallel.ProgressiveBandCoder(gpu_ctx, (d, d, d), 64, 0, 0, 0, 64, 0)
    coder.raw = torch.empty(256, dtype=torch.uint8, device="cuda")
    assert coder.code([0, 0, 0], [0] * 4)[0] == small and coder.raw.numel() >= need.value
    assert lib.pixo_b200_jpeg_band_dev_progressive_splice(h, raw.data_ptr() + 256, 0, 5, 0, 0, 1, raw.data_ptr(), 64,
                                                          C.byref(C.c_uint64())) == inv   # not a coded buffer
    with pytest.raises(_lib.PixoError) as e:
        parallel.encode_progressive_tiled_local([coder], JpegOptions(8, 512, ColorType.Gray, 80, Subsampling.S444, 4,
                                                                     False, True, False))
    assert e.value.code == _lib.ERR_UNSUPPORTED


# ---- NCCL ----------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _nccl_worker(rank, world, port, w, h, q, out_path):
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import pixo_b200
    from pixo_b200 import synthetic
    ctx = pixo_b200.Context(rank)
    o = opts(w, h, 2, q, 1)
    coder = coders_for(ctx, synthetic.noise(w, h, 3, 42), o, world)[rank]
    jpg = parallel.encode_progressive_tiled(coder, o, rank, world)
    assert ctx.host_fallbacks == 0
    if rank == 0:
        open(out_path, "wb").write(jpg)
    dist.destroy_process_group()


def test_tiled_progressive_frame_over_nccl_on_real_devices(lib, tmp_path):
    """>= 2 GPUs: one process per GPU, its band's transform, trellis and scans on its own device."""
    import torch.multiprocessing as mp
    from pixo_b200 import synthetic
    ndev = lib.pixo_b200_device_count()
    if ndev < 2:
        pytest.skip("needs at least two CUDA devices")
    world = min(ndev, 8)
    w, h, q = 2048, 1024, 80
    out = str(tmp_path / "nccl.jpg")
    mp.spawn(_nccl_worker, args=(world, _free_port(), w, h, q, out), nprocs=world, join=True)
    assert open(out, "rb").read() == jpeg.encode_progressive(synthetic.noise(w, h, 3, 42), opts(w, h, 2, q, 1))
