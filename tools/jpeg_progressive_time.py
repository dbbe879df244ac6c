"""Times the progressive scan stage (csrc/jpeg_progressive.cu) and pixo's max preset on the GPU, and writes
profiles/h100_jpeg_progressive.json: the card's name and power limit, then (CUDA events, mean of REPS after
one warm-up call; per-kernel times from torch.profiler in a run of their own)
  - 32 4K frames at the max preset (q80 4:2:0), device-resident: COEF_TRELLIS coefficients, then
    pixo_b200_jpeg_progressive_scans_dev on them;
  - the scan stage alone against k_huff (pixo_b200_jpeg_encode_dev) on the same frames;
  - the scan stage on plain coefficients (progressive without trellis);
  - one 16 384 x 16 384 4:2:0 frame, plain coefficients;
  - the host entry point end to end (pixo_b200_jpeg_encode_progressive_batch, pinned input and output);
  - the C oracle (oracle/jpeg_progressive.c, one thread; a restatement, not pixo) on one 4K frame.
Content: 8x8 blocks of random colour with light noise on every third row (as tools/jpeg_trellis_time.py).

    python tools/jpeg_progressive_time.py [out.json]
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
from pixo_b200 import _lib, jpeg  # noqa: E402

REPS = 3
fp = C.POINTER(C.c_float)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frames(n, w, h, dev, seed=3):
    g = torch.Generator(device=dev).manual_seed(seed)
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
    for i in range(n):
        base = torch.randint(0, 256, ((h + 7) // 8, (w + 7) // 8, 3), dtype=torch.uint8, device=dev, generator=g)
        f = base.repeat_interleave(8, 0).repeat_interleave(8, 1)[:h, :w]
        f[::3] ^= torch.randint(0, 8, f[::3].shape, dtype=torch.uint8, device=dev, generator=g)
        out[i] = f
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
    return a.elapsed_time(b) / REPS


def kernel_ms(fn, ctx, names):
    from torch.profiler import ProfilerActivity, profile
    ctx.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        ctx.sync()
    kt = {}
    for e in prof.key_averages():
        k = next((k for k in names if k in e.key), None)
        if k:
            kt[k] = kt.get(k, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
    return {k: round(v, 3) for k, v in sorted(kt.items())}


# (a kernel's time goes to the first name it contains: k_prog_emit_at before k_prog_emit)
PROG_KERNELS = ("k_prog_measure", "k_prog_carry", "k_prog_count", "k_prog_offsets", "k_prog_place", "k_prog_emit_at",
                "k_prog_emit", "k_seg_prefix", "k_seg_count", "k_seg_scan", "k_seg_fit", "k_seg_emit")


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_jpeg_progressive.json")
    lib = _lib.load()
    ctx = pixo_b200.Context(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)
    rec = {"card": gpu_info(),
           "note": f"ms per call; CUDA events, mean of {REPS} after one warm-up call; kernel times from torch.profiler",
           "configs": {}}
    for name, w, h, n in (("32x4K_q80_420", 3840, 2160, 32), ("1x16384sq_q80_420", 16384, 16384, 1)):
        px = frames(n, w, h, dev)
        ny, nc = jpeg.block_counts(w, h, 2, 1)
        dy = torch.empty(n * ny * 64, dtype=torch.int16, device=dev)
        dcb = torch.empty(n * nc * 64, dtype=torch.int16, device=dev)
        dcr = torch.empty(n * nc * 64, dtype=torch.int16, device=dev)
        _, _, lq, cq = jpeg.quant_tables(80)
        cap = (w * h * 3 // 2 + 65536) // 16 * 16
        d_out = torch.empty(n * cap, dtype=torch.uint8, device=dev)
        d_len = torch.empty((n, 7), dtype=torch.int64, device=dev)
        d_ovf = torch.empty(n, dtype=torch.int32, device=dev)

        def coef(flags):
            _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
                ctx.handle, px.data_ptr(), w * h * 3, n, w, h, 2, 1, lq.ctypes.data_as(fp), cq.ctypes.data_as(fp),
                dy.data_ptr(), ny * 64, dcb.data_ptr(), dcr.data_ptr(), nc * 64, flags, None))

        def scans():
            jpeg.progressive_scans_dev(dy, dcb, dcr, w, h, 2, 1, None, n, ny * 64, nc * 64, d_out, cap, d_len, d_ovf,
                                       ctx=ctx)

        r = {"frames": n, "width": w, "height": h, "quality": 80, "subsampling": "4:2:0", "blocks": n * (ny + 2 * nc)}
        coef(0)
        r["scans_plain_ms"] = round(events_ms(scans, stream), 3)
        r["scans_plain_kernel_ms"] = kernel_ms(scans, ctx, PROG_KERNELS)
        r["scan_bytes_plain"] = int(d_len.sum().item())
        if n > 1:
            r["coef_trellis_ms"] = round(events_ms(lambda: coef(jpeg.COEF_TRELLIS), stream), 3)
            r["scans_trellis_ms"] = round(events_ms(scans, stream), 3)
            r["scans_trellis_kernel_ms"] = kernel_ms(scans, ctx, PROG_KERNELS)
            r["max_preset_device_ms"] = round(r["coef_trellis_ms"] + r["scans_trellis_ms"], 3)
            # k_huff on the same frames: the baseline device entry (transform + k_huff), kernels from the profiler
            scan_cap = (w * h * 3 // 2 + 65536) // 256 * 256
            d_scan = torch.empty(n * scan_cap, dtype=torch.uint8, device=dev)
            d_sl = torch.empty(n, dtype=torch.int64, device=dev)
            d_so = torch.empty(n, dtype=torch.int32, device=dev)

            def base():
                _lib.check(ctx.handle, lib.pixo_b200_jpeg_encode_dev(ctx.handle, px.data_ptr(), w * h * 3, n, w, h, 2,
                                                                     80, 1, d_scan.data_ptr(), scan_cap,
                                                                     d_sl.data_ptr(), d_so.data_ptr()))
            r["baseline_encode_dev_ms"] = round(events_ms(base, stream), 3)
            r["baseline_kernel_ms"] = kernel_ms(base, ctx, ("k_huff", "k_jpeg_420"))
            del d_scan
            # host end to end: pinned input and output, the max preset
            hp = px.reshape(n, -1).cpu().pin_memory()
            out_cap = w * h * 3 + 65536
            ho = torch.empty(n * out_cap, dtype=torch.uint8).pin_memory()
            lens = (C.c_size_t * n)()

            def host():
                _lib.check(ctx.handle, lib.pixo_b200_jpeg_encode_progressive_batch(
                    ctx.handle, hp.data_ptr(), w * h * 3, n, w, h, 2, 80, 1, 0, 1, 1, ho.data_ptr(), out_cap, lens))
            host()
            t = time.perf_counter()
            for _ in range(REPS):
                host()
            r["host_e2e_pinned_ms"] = round((time.perf_counter() - t) * 1e3 / REPS, 3)
            r["host_e2e_bytes"] = int(sum(lens))
            from oracle import jpeg_progressive as jp
            jp.build()
            img = px[0].cpu().numpy().reshape(-1)
            t = time.perf_counter()
            jp.encode(img, w, h, 2, 1, 80)
            rec["cpu_oracle_4k_max_s"] = round(time.perf_counter() - t, 2)
            rec["cpu_note"] = ("oracle/jpeg_progressive.c (the test suite's C restatement, gcc -O2, one thread: "
                               "transform, plain + trellis coefficients, baseline tables, scans), not pixo itself")
        rec["configs"][name] = r
        print(name, json.dumps(r), flush=True)
        del px, dy, dcb, dcr, d_out
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
