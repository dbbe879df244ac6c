"""Times pixo_b200_jpeg_encode_dev_opts (optimised tables built on the GPU, restart intervals) and writes
profiles/h100_jpeg_encode_dev_opts.json: the card's name and power limit, read in the same run, then
(CUDA events around REPS calls after one warm-up call; host clock around calls that end in a synchronise)
on 32 4K RGB frames
  - pixo's balanced preset (4:4:4 q75, optimised tables): encode_dev_opts, and encode_dev_opts plus the
    copies and host headers that make the 32 files, against the route that existed before it for the same
    files: pixo_b200_jpeg_coefficients_dev with d_hist, then one pixo_b200_jpeg_entropy_encode_dev per frame
    (both routes write the files into host memory allocated once);
  - 4:2:0 q80 with restart interval 8 (and optimised tables) against pixo_b200_jpeg_encode_dev (4:2:0 q80,
    standard tables, no restart interval) on the same frames;
  - per-kernel device time of k_huff_tables and the k_huff instantiations, from torch.profiler in a run
    of its own.
Content: bench.py's ring of frames (half gradients, half noise).  Every file of the balanced run is checked
against the old route's.

    python tools/jpeg_encode_dev_opts_time.py [out.json]
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
fp = C.POINTER(C.c_float)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frames(dev):
    """Even frames: a horizontal + vertical gradient with a per-frame offset; odd frames: uniform noise."""
    g = torch.Generator(device=dev).manual_seed(7)
    out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
    x = torch.arange(W, device=dev)[None, :, None]
    y = torch.arange(H, device=dev)[:, None, None]
    c = torch.arange(3, device=dev)[None, None, :]
    for i in range(N):
        if i % 2:
            out[i] = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, device=dev, generator=g)
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
        if "k_huff" in e.key or "k_jpeg" in e.key:
            name = e.key.replace("void ", "").replace("pixo::(anonymous namespace)::", "").split("(")[0]
            kt[name] = kt.get(name, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
    return {k: round(v, 3) for k, v in sorted(kt.items())}


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_jpeg_encode_dev_opts.json")
    lib = _lib.load()
    ctx = pixo_b200.Context(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)
    rec = {"card": gpu_info(), "frames": N, "width": W, "height": H,
           "note": f"ms per call of {N} frames; CUDA events (device) or host clock around calls ending in a "
                   f"synchronise (files), mean of {REPS} after one warm-up call; kernels from torch.profiler, "
                   "one call, in a run of its own",
           "configs": {}}
    px = frames(dev)
    each = W * H * 3
    cap = (each + 65536) // 256 * 256   # room for the noise frames at 4:4:4
    d_scan = torch.empty(N * cap, dtype=torch.uint8, device=dev)
    d_len = torch.empty(N, dtype=torch.int64, device=dev)
    d_ovf = torch.empty(N, dtype=torch.int32, device=dev)
    d_dht = torch.empty((N, jpeg.DHT_BYTES), dtype=torch.uint8, device=dev)

    # ---- the balanced preset --------------------------------------------------------------------------
    bal = JpegOptions.balanced(W, H, 75)

    def new():
        jpeg.encode_dev(px, each, N, bal, d_scan, cap, d_len, d_ovf, d_dht, ctx=ctx)

    # both routes write file i at files[i * fcap] (host memory allocated once), its length to flen[i]
    fcap = cap + 4096
    files = np.empty(N * fcap, np.uint8)
    flen = np.zeros(N, np.int64)
    lens = np.zeros(N, np.int64)
    tabs = np.zeros((N, jpeg.DHT_BYTES), np.uint8)

    def new_files():
        new()   # then the lengths, the tables, and each frame's scan bytes straight after its headers
        _lib.check(ctx.handle, lib.pixo_b200_download(ctx.handle, lens.ctypes.data, d_len.data_ptr(), lens.nbytes))
        _lib.check(ctx.handle, lib.pixo_b200_download(ctx.handle, tabs.ctypes.data, d_dht.data_ptr(), tabs.nbytes))
        for i in range(N):
            n = C.c_size_t()
            o = i * fcap
            _lib.check(None, lib.pixo_b200_jpeg_write_headers_dht(W, H, 2, 75, 0, 0, tabs[i].ctypes.data,
                                                                  files[o:].ctypes.data, 4096, C.byref(n)))
            k = n.value
            _lib.check(ctx.handle, lib.pixo_b200_download(ctx.handle, files[o + k:].ctypes.data,
                                                          d_scan.data_ptr() + i * cap, int(lens[i])))
            files[o + k + lens[i]:o + k + lens[i] + 2] = (0xFF, 0xD9)
            flen[i] = k + lens[i] + 2

    ny, nc = jpeg.block_counts(W, H, 2, 0)
    _, _, lq, cq = jpeg.quant_tables(75)
    dy = torch.empty(N * ny * 64, dtype=torch.int16, device=dev)
    dcb = torch.empty(N * nc * 64, dtype=torch.int16, device=dev)
    dcr = torch.empty(N * nc * 64, dtype=torch.int16, device=dev)
    dh = torch.empty(N * 536, dtype=torch.int64, device=dev)

    def old_files():
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
            ctx.handle, px.data_ptr(), each, N, W, H, 2, 0, lq.ctypes.data_as(fp), cq.ctypes.data_as(fp),
            dy.data_ptr(), ny * 64, dcb.data_ptr(), dcr.data_ptr(), nc * 64, 0, dh.data_ptr()))
        for i in range(N):
            n = C.c_size_t()
            _lib.check(ctx.handle, lib.pixo_b200_jpeg_entropy_encode_dev(
                ctx.handle, dy.data_ptr() + i * ny * 128, dcb.data_ptr() + i * nc * 128, dcr.data_ptr() + i * nc * 128,
                W, H, 2, 75, 0, 0, 1, files[i * fcap:].ctypes.data, fcap, C.byref(n)))
            flen[i] = n.value

    def snapshot():
        return [files[i * fcap:i * fcap + flen[i]].tobytes() for i in range(N)]

    new_files()
    got = snapshot()
    old_files()
    same = got == snapshot()
    assert same, "encode_dev_opts and the old route wrote different files"
    r = {"options": "4:4:4 q75, optimised tables (JpegOptions.balanced)",
         "encode_dev_opts_device_ms": events_ms(new, stream),
         "encode_dev_opts_to_files_ms": host_ms(new_files),
         "old_route_to_files_ms": host_ms(old_files),
         "old_route": "pixo_b200_jpeg_coefficients_dev(d_hist) + one pixo_b200_jpeg_entropy_encode_dev per frame",
         "files_identical": same,
         "scan_bytes": int(d_len.sum().item())}
    rec["configs"]["balanced_444_q75"] = r
    print("balanced", json.dumps(r), flush=True)
    del dy, dcb, dcr, dh, files
    torch.cuda.empty_cache()

    # ---- 4:2:0 q80 with restart 8 against encode_dev ----------------------------------------------------------
    rst = JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420, 8, True)

    def rst8():
        jpeg.encode_dev(px, each, N, rst, d_scan, cap, d_len, d_ovf, d_dht, ctx=ctx)

    def plain():
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_encode_dev(ctx.handle, px.data_ptr(), each, N, W, H, 2, 80, 1,
                                                             d_scan.data_ptr(), cap, d_len.data_ptr(),
                                                             d_ovf.data_ptr()))
    r = {"encode_dev_opts_420_q80_rst8_opt_ms": events_ms(rst8, stream),
         "encode_dev_420_q80_ms": events_ms(plain, stream)}
    rec["configs"]["420_q80"] = r
    print("420", json.dumps(r), flush=True)

    # ---- kernels -------------------------------------------------------------------------------------------
    rec["kernels_ms"] = {"balanced_444_q75": kernel_ms(new, ctx), "420_q80_rst8_opt": kernel_ms(rst8, ctx),
                         "encode_dev_420_q80": kernel_ms(plain, ctx)}
    print("kernels", json.dumps(rec["kernels_ms"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
