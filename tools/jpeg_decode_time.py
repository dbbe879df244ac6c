"""Times the GPU baseline JPEG decoder (pixo_b200_jpeg_decode_to_device) and writes profiles/h100_jpeg_decode.json
(or --out).  Workloads: 256 1080p and 32 4K files, 4:2:0 q80, from the GPU encoder with pixo's fast preset (standard
tables) and balanced preset (optimised tables), half noise and half gradient; one dense (noise) 4K file, one dense
1080p file and 32 dense 4K files alone; one 16 384^2 gradient file.  Per
workload: the call's CUDA-event time (median of --reps, frames already sized, files in host memory), per-kernel
times from torch.profiler in a separate run, and for scale the C oracle on one host thread and PIL's decode of the
same files.  The card's name and power limit are recorded beside the numbers."""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

import pixo_b200
from pixo_b200 import ColorType, decode, jpeg
from pixo_b200.jpeg import JpegOptions, Subsampling
from oracle import jpeg_decode as jd
from oracle import pyoracle as po


def files_for(ctx, w, h, n, optimize, noise_only=False):
    """n files alternating noise and gradient (noise only: every file dense); above 2^24 pixels gradient only"""
    big = w * h > 1 << 24
    frames = [po.gen_noise(w, h, 3, 1)] if not big else []
    if not (noise_only and frames):
        frames.append(np.asarray(po.gen_gradient_rgb(w, h)).reshape(-1))
    enc = jpeg.encode_batch(np.stack(frames), JpegOptions(w, h, ColorType.Rgb, 80, Subsampling.S420, None, optimize),
                            ctx=ctx)
    return [enc[i % len(enc)] for i in range(n)]


def time_call(ctx, files, reps):
    """CUDA events around the call on a stream of its own, which the context is switched to (a null handle would
    mean the context's own stream, not torch's default one)"""
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            decode.decode_jpeg_batch_dev(files, ctx=ctx)   # warm-up: scratch, modules
            s.synchronize()
            ts = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                decode.decode_jpeg_batch_dev(files, ctx=ctx)
                b.record(s)
                b.synchronize()
                ts.append(a.elapsed_time(b))
    finally:
        ctx.set_stream(None)
    return statistics.median(ts), ts


def kernel_times(ctx, files):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decode.decode_jpeg_batch_dev(files, ctx=ctx)
        ctx.sync()
    out = {}
    for e in prof.key_averages():
        for k in ("k_jdec_scan", "k_jdec_idct", "k_jdec_color"):
            if k in e.key:
                out[k] = round(e.device_time_total / 1000.0, 3)
    return out


def cpu_times(files, n_cpu):
    sub = files[:n_cpu]
    t = time.perf_counter()
    for f in sub:
        jd.decode(f, coefs=False)
    oracle = (time.perf_counter() - t) / len(sub) * len(files) * 1000
    pil = None
    try:
        from PIL import Image
        Image.MAX_IMAGE_PIXELS = None   # the 16 384^2 frame is not a decompression bomb
        t = time.perf_counter()
        for f in sub:
            Image.open(io.BytesIO(f)).convert("RGB").tobytes()
        pil = (time.perf_counter() - t) / len(sub) * len(files) * 1000
    except ImportError:
        pass
    return oracle, pil


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_jpeg_decode.json"))
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctx = pixo_b200.Context(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "note": "call time: CUDA events around pixo_b200_jpeg_decode_to_device with the files in "
           "host memory (header parsing and upload included); kernels: torch.profiler in a separate run; CPU "
           "figures: one host thread, extrapolated from up to 8 files; noise and gradient files alternate unless the "
           "workload says dense (noise only)", "workloads": []}
    workloads = [("1080p x256", 1920, 1080, 256, False), ("4K x32", 3840, 2160, 32, False)]
    one = [("one dense 4K file", 3840, 2160, 1, True), ("one dense 1080p file", 1920, 1080, 1, True),
           ("32 dense 4K files", 3840, 2160, 32, True), ("16384^2 x1 (gradient)", 16384, 16384, 1, False)]
    runs = [(wl, p, o) for wl in workloads for p, o in (("fast", False), ("balanced", True))] + [(wl, "fast", False) for wl in one]
    for (name, w, h, n, noise_only), preset, opt in runs:
        files = files_for(ctx, w, h, n, opt, noise_only)
        med, best = time_call(ctx, files, a.reps)
        ker = kernel_times(ctx, files)
        oracle, pil = cpu_times(files, min(n, 8))
        mpx = w * h * n / 1e6
        row = {"workload": name, "preset": preset, "compressed_MB": round(sum(map(len, files)) / 1e6, 2),
               "call_ms_median": round(med, 3), "call_ms_each": [round(t, 3) for t in best], "Mpix_per_s": round(mpx / med * 1e3, 1),
               "scan_MB_per_s": round(sum(map(len, files)) / 1e6 / (ker.get("k_jdec_scan", med) / 1e3), 1),
               "kernels_ms": ker, "oracle_1thread_ms": round(oracle, 1),
               "pil_1thread_ms": None if pil is None else round(pil, 1)}
        print(json.dumps(row), flush=True)
        res["workloads"].append(row)
        # written after every workload, so that a run cut short still leaves what it measured
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)

if __name__ == "__main__":
    main()
