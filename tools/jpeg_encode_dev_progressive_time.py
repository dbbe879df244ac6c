"""Times pixo_b200_jpeg_encode_dev_progressive (pixo's max preset queued on the context's stream) and writes
profiles/h100_jpeg_encode_dev_progressive.json: the card's name and power limit, read in the same run, then
(CUDA events around REPS calls after one warm-up call; host clock around calls that end in a synchronise)
  - 32 4K RGB frames at 4:2:0 q80, max preset (optimised tables, trellis): encode_dev_progressive on the
    device, against pixo_b200_jpeg_encode_progressive_batch from pinned memory on the same frames (host clock:
    the call returns with its files in host memory);
  - the scan stage alone on the same frames' coefficients: the queued stage (encode_dev_progressive without
    trellis and with the standard tables, minus the transform and k_huff_tables, timed on their own) against
    pixo_b200_jpeg_progressive_scans_dev, which waits for the device for the bit counts;
  - a small-batch pipeline: CALLS calls of FEW 1080p frames each, queued back to back with one synchronisation
    at the end, against the same files through the waiting routes (encode_progressive_batch per call, from pinned
    memory), host clock around each whole pipeline;
  - per-kernel device time from torch.profiler, one call of the 4K batch, in a run of its own.
Content: bench.py's ring of frames (half gradients, half noise).  The 4K files and the pipeline's files are
checked against the host batch call's.

    python tools/jpeg_encode_dev_progressive_time.py [out.json]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pixo_b200  # noqa: E402
from pixo_b200 import ColorType, _lib, jpeg  # noqa: E402
from pixo_b200.jpeg import JpegOptions, Subsampling  # noqa: E402

REPS = 5
W, H, N = 3840, 2160, 32
SW, SH, FEW, CALLS = 1920, 1080, 3, 8
fp = C.POINTER(C.c_float)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frames(dev, n, w, h, seed):
    """Even frames: a horizontal + vertical gradient with a per-frame offset; odd frames: uniform noise."""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
    x = torch.arange(w, device=dev)[None, :, None]
    y = torch.arange(h, device=dev)[:, None, None]
    c = torch.arange(3, device=dev)[None, None, :]
    for i in range(n):
        if i % 2:
            out[i] = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device=dev, generator=g)
        else:
            out[i] = ((x * (c + 1) + y * (3 - c) + 17 * i) % 256).to(torch.uint8)
    return out


def events_ms(fn, stream):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(REPS):
        fn()
    b.record(stream)
    b.synchronize()
    return round(a.elapsed_time(b) / REPS, 3)


def host_ms(fn):
    fn()
    t = time.perf_counter()
    for _ in range(REPS):
        fn()
    return round((time.perf_counter() - t) * 1e3 / REPS, 3)


def kernel_ms(fn, ctx):
    from torch.profiler import ProfilerActivity, profile
    ctx.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        ctx.sync()
    kt = {}
    for e in prof.key_averages():
        if e.key.startswith("void pixo::") or "k_" in e.key:
            name = e.key.replace("void ", "").replace("pixo::(anonymous namespace)::", "").split("(")[0]
            kt[name] = kt.get(name, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
    return {k: round(v, 3) for k, v in sorted(kt.items())}


class Dev:
    """Device outputs of encode_dev_progressive for n frames of cap bytes each."""

    def __init__(self, dev, n, cap):
        self.n, self.cap = n, cap
        self.out = torch.empty(n * cap, dtype=torch.uint8, device=dev)
        self.lens = torch.empty((n, 7), dtype=torch.int64, device=dev)
        self.ovf = torch.empty(n, dtype=torch.int32, device=dev)
        self.dht = torch.empty((n, jpeg.DHT_BYTES), dtype=torch.uint8, device=dev)

    def call(self, ctx, px, each, o):
        jpeg.encode_progressive_dev(px, each, self.n, o, self.out, self.cap, self.lens, self.ovf, self.dht, ctx=ctx)

    def files(self, o):
        assert not self.ovf.any().item(), "a frame did not fit"
        out, lens, tabs = self.out.cpu().numpy(), self.lens.cpu().numpy(), self.dht.cpu().numpy()
        return [jpeg.progressive_file(o, tabs[i], out[i * self.cap:(i + 1) * self.cap], lens[i]) for i in range(self.n)]


def host_batch(ctx, pinned, n, each, o, out, cap, lens):
    _lib.check(ctx.handle, _lib.load().pixo_b200_jpeg_encode_progressive_batch(
        ctx.handle, pinned.data_ptr(), each, n, o.width, o.height, int(o.color_type), o.quality, int(o.subsampling),
        o.restart_interval or 0, int(o.optimize_huffman), int(o.trellis_quant), out.ctypes.data, cap, lens))


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles",
                                                                 "h100_jpeg_encode_dev_progressive.json")
    lib = _lib.load()
    ctx = pixo_b200.Context(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)
    rec = {"card": gpu_info(), "note": f"ms; CUDA events (device) or host clock around calls ending in a "
                                       f"synchronise, mean of {REPS} after one warm-up call; kernels from "
                                       "torch.profiler, one call, in a run of its own", "configs": {}}

    # ---- 32 4K frames, max preset ---------------------------------------------------------------------------
    mx = JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420, None, True, True, True)
    px = frames(dev, N, W, H, 7)
    each = W * H * 3
    cap = (each + 65536) // 256 * 256   # room for the noise frames
    d = Dev(dev, N, cap)
    pinned = px.cpu().pin_memory()
    hout = np.empty(N * cap, np.uint8)
    hlens = (C.c_size_t * N)()
    d.call(ctx, px, each, mx)
    got = d.files(mx)
    host_batch(ctx, pinned, N, each, mx, hout, cap, hlens)
    same = got == [hout[i * cap:i * cap + hlens[i]].tobytes() for i in range(N)]
    assert same, "encode_dev_progressive and encode_progressive_batch wrote different files"
    r = {"frames": N, "width": W, "height": H, "options": "4:2:0 q80, optimised tables, trellis (max preset)",
         "encode_dev_progressive_device_ms": events_ms(lambda: d.call(ctx, px, each, mx), stream),
         "encode_progressive_batch_pinned_ms": host_ms(lambda: host_batch(ctx, pinned, N, each, mx, hout, cap, hlens)),
         "files_identical": same, "file_bytes": int(sum(hlens))}
    rec["configs"]["max_420_q80_32x4k"] = r
    print("4k", json.dumps(r), flush=True)

    # ---- the scan stage alone -----------------------------------------------------------------------------
    plain = JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420, None, False, True, False)
    ny, nc = jpeg.block_counts(W, H, 2, 1)
    _, _, lq, cq = jpeg.quant_tables(80)
    dy = torch.empty(N * ny * 64, dtype=torch.int16, device=dev)
    dcb = torch.empty(N * nc * 64, dtype=torch.int16, device=dev)
    dcr = torch.empty(N * nc * 64, dtype=torch.int16, device=dev)

    def transform():
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
            ctx.handle, px.data_ptr(), each, N, W, H, 2, 1, lq.ctypes.data_as(fp), cq.ctypes.data_as(fp),
            dy.data_ptr(), ny * 64, dcb.data_ptr(), dcr.data_ptr(), nc * 64, 0, None))

    def scans_dev():
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_progressive_scans_dev(
            ctx.handle, dy.data_ptr(), ny * 64, dcb.data_ptr(), dcr.data_ptr(), nc * 64, N, W, H, 2, 1, None,
            d.out.data_ptr(), cap, d.lens.data_ptr(), d.ovf.data_ptr()))

    transform()
    whole = events_ms(lambda: d.call(ctx, px, each, plain), stream)
    r = {"options": "4:2:0 q80, standard tables, no trellis",
         "encode_dev_progressive_device_ms": whole,
         "transform_device_ms": events_ms(transform, stream),
         "progressive_scans_dev_host_ms": host_ms(lambda: (scans_dev(), ctx.sync())),
         "note": "the queued stage is encode_dev_progressive minus the transform and k_huff_tables (see kernels_ms); "
                 "progressive_scans_dev waits for the device, so it is timed by the host clock to its end"}
    rec["configs"]["scan_stage_420_q80_32x4k"] = r
    print("stage", json.dumps(r), flush=True)
    rec["kernels_ms"] = {"max_420_q80_32x4k": kernel_ms(lambda: d.call(ctx, px, each, mx), ctx),
                         "plain_420_q80_32x4k": kernel_ms(lambda: d.call(ctx, px, each, plain), ctx),
                         "progressive_scans_dev_32x4k": kernel_ms(scans_dev, ctx)}
    print("kernels", json.dumps(rec["kernels_ms"]), flush=True)
    del px, pinned, hout, dy, dcb, dcr, d
    torch.cuda.empty_cache()

    # ---- small batches: CALLS calls of FEW 1080p frames -------------------------------------------------------
    so = JpegOptions(SW, SH, ColorType.Rgb, 80, Subsampling.S420, None, True, True, True)
    seach = SW * SH * 3
    scap = (seach + 65536) // 256 * 256
    spx = [frames(dev, FEW, SW, SH, 20 + k) for k in range(CALLS)]
    spin = [p.cpu().pin_memory() for p in spx]
    sd = [Dev(dev, FEW, scap) for _ in range(CALLS)]
    shout = [np.empty(FEW * scap, np.uint8) for _ in range(CALLS)]
    slens = [(C.c_size_t * FEW)() for _ in range(CALLS)]

    def queued():
        for k in range(CALLS):
            sd[k].call(ctx, spx[k], seach, so)
        ctx.sync()

    def waiting():
        for k in range(CALLS):
            host_batch(ctx, spin[k], FEW, seach, so, shout[k], scap, slens[k])

    queued()
    waiting()
    same = all(sd[k].files(so) == [shout[k][i * scap:i * scap + slens[k][i]].tobytes() for i in range(FEW)]
               for k in range(CALLS))
    assert same, "the queued pipeline and the host batch calls wrote different files"
    r = {"calls": CALLS, "frames_per_call": FEW, "width": SW, "height": SH,
         "options": "4:2:0 q80, optimised tables, trellis (max preset)",
         "queued_one_sync_ms": host_ms(queued),
         "encode_progressive_batch_pinned_ms": host_ms(waiting),
         "note": "queued: the calls back to back and one ctx.sync(), files stay in device memory; "
                 "waiting: one encode_progressive_batch per call from pinned memory, files in host memory",
         "files_identical": same}
    rec["configs"]["pipeline_1080p"] = r
    print("pipeline", json.dumps(r), flush=True)

    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
