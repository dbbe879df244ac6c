"""Times the GPU PNG decoder (pixo_b200_png_decode_to_device) and writes profiles/h100_png_decode.json (or --out).
Workloads: 256 1080p RGB and 32 4K RGBA noise files (zlib level 1, filter None rows), one 4K RGBA file alone, one
16 384^2 RGB file (Up / None rows, each row periodic: mostly long matches), and the 126 palette-heavy reduce goldens.  Per workload:
the call's CUDA-event time (median of --reps, files in host memory, the call waits for the device once per pass), per-kernel
times from torch.profiler in a separate run, the inflated MB/s of one stream (inflated bytes of the longest stream over
k_png_inflate's time), and for scale the C oracle and PIL (zlib + its C unfilter) on one host thread.  The card's name
and power limit are recorded beside the numbers."""
import argparse
import glob
import io
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch

import pixo_b200
from pixo_b200 import decode
from oracle import png_decode as pd
from oracle import pyoracle as po
from png_decode_corpus import png

KERNELS = ("k_png_crc", "k_png_inflate", "k_png_unfilter", "k_png_expand")


def noise_files(w, h, ch, n):
    ct = {3: 2, 4: 6}[ch]
    enc = []
    for s in range(min(n, 4)):
        img = po.gen_noise(w, h, ch, s).reshape(h, w * ch)
        rows = np.concatenate([np.zeros((h, 1), np.uint8), img], axis=1)
        enc.append(png(w, h, 8, ct, zlib.compress(rows.tobytes(), 1)))
    return [enc[i % len(enc)] for i in range(n)]


def big_file():
    from test_png_decode_gpu import periodic_16k
    return [periodic_16k()[0]]


def time_call(ctx, files, reps):
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    try:
        with torch.cuda.stream(s):
            decode.decode_png_batch_dev(files, ctx=ctx)
            s.synchronize()
            ts = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                decode.decode_png_batch_dev(files, ctx=ctx)
                b.record(s)
                b.synchronize()
                ts.append(a.elapsed_time(b))
    finally:
        ctx.set_stream(None)
    return statistics.median(ts), ts


def kernel_times(ctx, files):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decode.decode_png_batch_dev(files, ctx=ctx)
        ctx.sync()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                out[k] = round(e.device_time_total / 1000.0, 3)
    return out


def cpu_times(files, n_cpu):
    sub = files[:n_cpu]
    t = time.perf_counter()
    for f in sub:
        pd.decode(f)
    oracle = (time.perf_counter() - t) / len(sub) * len(files) * 1000
    t = time.perf_counter()
    for f in sub:
        from PIL import Image
        Image.MAX_IMAGE_PIXELS = None
        Image.open(io.BytesIO(f)).tobytes()
    pil = (time.perf_counter() - t) / len(sub) * len(files) * 1000
    return oracle, pil


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_png_decode.json"))
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctx = pixo_b200.Context(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "note": "call time: CUDA events around pixo_b200_png_decode_to_device with the files in host "
           "memory (chunk walk, upload and the one wait per pass included); kernels: torch.profiler in a separate run; "
           "inflate_MB_per_s_per_stream: the longest stream's inflated bytes over k_png_inflate's time; CPU figures: "
           "one host thread (the C oracle, and PIL's decode, which is zlib + C unfilter), extrapolated from up to 8 "
           "files", "workloads": []}
    reduce = [open(p, "rb").read() for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "reduce", "*.png")))]
    workloads = [("1080p RGB x256", lambda: noise_files(1920, 1080, 3, 256)),
                 ("4K RGBA x32", lambda: noise_files(3840, 2160, 4, 32)),
                 ("one 4K RGBA file", lambda: noise_files(3840, 2160, 4, 1)),
                 ("16384^2 RGB x1", big_file),
                 ("reduce goldens x126 (palette-heavy)", lambda: reduce)]
    for name, make in workloads:
        files = make()
        med, each = time_call(ctx, files, a.reps)
        ker = kernel_times(ctx, files)
        oracle, pil = cpu_times(files, min(len(files), 8))
        longest = max(files, key=len)
        dec = pd.decode(longest)
        # inflated bytes of the longest stream: rows plus one filter byte each
        ch = {0: 1, 1: 2, 2: 3, 3: 4}[dec.color_type]
        inflated = dec.height * (1 + dec.width * ch) if longest[24] == 8 and longest[25] != 3 else None
        row = {"workload": name, "files": len(files), "compressed_MB": round(sum(map(len, files)) / 1e6, 2),
               "call_ms_median": round(med, 3), "call_ms_each": [round(t, 3) for t in each],
               "Mpix_per_s": round(sum(g.width * g.height for g in map(lambda f: pd.decode(f, pixels=False), files))
                                   / 1e6 / med * 1e3, 1),
               "kernels_ms": ker,
               "inflate_MB_per_s_per_stream": None if inflated is None or "k_png_inflate" not in ker
               else round(inflated / 1e6 / (ker["k_png_inflate"] / 1e3), 1),
               "oracle_1thread_ms": round(oracle, 1), "pil_1thread_ms": round(pil, 1)}
        print(json.dumps(row), flush=True)
        res["workloads"].append(row)
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
