"""Times device-resident pixo_b200_jpeg_coefficients_dev with PIXO_B200_COEF_TRELLIS against plain
coefficients (CUDA events, after warm-up), with per-kernel times (transform f32 mode, k_trellis) from
torch.profiler in a run of their own, the card's name and power limit read in the same run, and the C
oracle's single-thread trellis time on one 4K frame as the CPU figure (a restatement, not pixo).

    python tools/jpeg_trellis_time.py [out.json]        (needs a GPU; writes profiles/h100_jpeg_trellis.json)
    python tools/jpeg_trellis_time.py --plain-only OUT  (plain K1 / K2 only: run once per library for an A/B,
                                                         PIXO_B200_SO picks the library)

Configurations: 32 4K frames q80 4:2:0, 32 4K frames q75 4:4:4, one 16 384 x 16 384 frame q80 4:2:0.
Content: 8x8 blocks of random colour with light noise on every third row (a mix of flat and busy blocks).
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

REPS = 5
KERNELS = ("k_jpeg_420", "k_jpeg_444", "k_trellis")
CONFIGS = [("32x4K_q80_420", 3840, 2160, 32, 80, 1), ("32x4K_q75_444", 3840, 2160, 32, 75, 0),
           ("1x16384sq_q80_420", 16384, 16384, 1, 80, 1)]


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


def main():
    plain_only = "--plain-only" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--plain-only"]
    out_path = args[0] if args else os.path.join(ROOT, "profiles", "h100_jpeg_trellis.json")
    if plain_only:   # a library from before the trellis entry point may be the A side
        _lib.SYMBOLS.pop("pixo_b200_jpeg_trellis_quantize_dev")
    lib = _lib.load()
    ctx = pixo_b200.Context(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)   # the library's work and the events share one stream
    rec = {"card": gpu_info(), "library": _lib.SO_PATH if plain_only else "tree",
           "note": "ms per pixo_b200_jpeg_coefficients_dev call (device-resident, natural order); CUDA events, "
                   f"mean of {REPS} after one warm-up call", "configs": {}}
    for name, w, h, n, qual, ss in (CONFIGS[:2] if plain_only else CONFIGS):
        px = frames(n, w, h, dev)
        ny, nc = jpeg.block_counts(w, h, 2, ss)
        dy = torch.empty(n * ny * 64, dtype=torch.int16, device=dev)
        dcb = torch.empty(n * nc * 64, dtype=torch.int16, device=dev)
        dcr = torch.empty(n * nc * 64, dtype=torch.int16, device=dev)
        _, _, lq, cq = jpeg.quant_tables(qual)
        fp = C.POINTER(C.c_float)

        def call(flags):
            _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
                ctx.handle, px.data_ptr(), w * h * 3, n, w, h, 2, ss, lq.ctypes.data_as(fp), cq.ctypes.data_as(fp),
                dy.data_ptr(), ny * 64, dcb.data_ptr(), dcr.data_ptr(), nc * 64, flags, None))
        r = {"frames": n, "width": w, "height": h, "quality": qual, "subsampling": "4:2:0" if ss else "4:4:4",
             "blocks": n * (ny + 2 * nc)}
        r["plain_ms"] = round(events_ms(lambda: call(0), stream), 3)
        if not plain_only:
            r["trellis_ms"] = round(events_ms(lambda: call(jpeg.COEF_TRELLIS), stream), 3)
            r["trellis_mblocks_per_s"] = round(r["blocks"] / r["trellis_ms"] / 1e3, 1)
            from torch.profiler import ProfilerActivity, profile
            ctx.sync()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call(jpeg.COEF_TRELLIS)
                ctx.sync()
            kt = {}
            for e in prof.key_averages():
                k = next((k for k in KERNELS if k in e.key), None)
                if k:
                    k = k + ("<kDct>" if k != "k_trellis" else "")
                    kt[k] = kt.get(k, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
            r["trellis_kernel_ms"] = {k: round(v, 3) for k, v in sorted(kt.items())}
        rec["configs"][name] = r
        print(name, json.dumps(r), flush=True)
        del px, dy, dcb, dcr
        torch.cuda.empty_cache()
    if not plain_only:
        from oracle import jpeg_trellis as jt
        img = frames(1, 3840, 2160, dev)[0].cpu().numpy().reshape(-1)
        t = time.perf_counter()
        jt.jpeg_coefficients(img, 3840, 2160, 2, 1, 80)
        rec["cpu_oracle_4k_420_q80_s"] = round(time.perf_counter() - t, 2)
        rec["cpu_note"] = ("oracle/jpeg_trellis.c (the test suite's C restatement, gcc -O2, one thread, transform "
                           "included), not pixo itself")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
