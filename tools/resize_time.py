"""Times pixo_b200_resize_dev (CUDA events, after warm-up) on the workloads below, with per-kernel times from
torch.profiler in a run of their own, the card's name and power limit read in the same run, and
oracle/resize.c on one host thread for scale (that is the restatement used by the tests, not pixo).

    python tools/resize_time.py [out.json]      (needs a GPU; writes profiles/h100_resize.json)

Workloads: 32 4K RGBA frames -> 1080p and -> 8K under each algorithm, and 256 1080p RGB frames -> 640x360
Lanczos3.  Bytes moved: the destination written once, plus the source bytes the algorithm reads: Nearest
the sampled pixels only (at most one per destination pixel), Bilinear at most four per destination pixel,
Lanczos3 the whole source and the u8 intermediate (source rows x destination columns) written and read
once, since it goes through HBM.
Fraction of peak: those bytes over the time, against the H100 SXM data sheet's 3.35 TB/s.
"""
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
from pixo_b200 import ColorType  # noqa: E402
from pixo_b200 import resize as rs  # noqa: E402
from oracle import resize as rz  # noqa: E402

REPS = 5
PEAK = 3.35e12
KERNELS = ("k_resize_nearest", "k_resize_bilinear", "k_resize_lanczos_h", "k_resize_lanczos_v")
NAMES = ("Nearest", "Bilinear", "Lanczos3")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_resize.json")
    ctx = pixo_b200.Context(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)   # the library's work and the events share one stream
    work = [(32, 3840, 2160, 1920, 1080, 3, a) for a in range(3)] + [(32, 3840, 2160, 7680, 4320, 3, a) for a in range(3)]
    work.append((256, 1920, 1080, 640, 360, 2, 2))
    rec = {"card": gpu_info(), "peak_bytes_per_s": PEAK,
           "note": "ms per pixo_b200_resize_dev call on the whole batch, CUDA events after warm-up; kernel_ms from "
                   "torch.profiler in a separate run; oracle_ms_per_frame: oracle/resize.c, one host thread, one "
                   "frame (the tests' restatement, not pixo)", "workloads": []}
    rng = np.random.default_rng(1)
    for n, sw, sh, dw, dh, ct, alg in work:
        bpp = ct + 1
        base = rng.integers(0, 256, sw * sh * bpp, dtype=np.uint8)
        d_frame = torch.from_numpy(base).to(dev)
        src = torch.empty((n, sw * sh * bpp), dtype=torch.uint8, device=dev)
        for i in range(n):
            src[i] = torch.roll(d_frame, 13 * i)
        dst = torch.empty((n, dw * dh * bpp), dtype=torch.uint8, device=dev)
        o = rs.ResizeOptions.builder(sw, sh).dst(dw, dh).color_type(ColorType(ct)).algorithm(rs.ResizeAlgorithm(alg)).build()
        torch.cuda.synchronize()

        def call():
            rs.resize_dev(src, sw * sh * bpp, n, o, dst, dw * dh * bpp, ctx=ctx)
        call()
        ctx.sync()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(REPS):
            call()
        b.record(stream)
        b.synchronize()
        ms = a.elapsed_time(b) / REPS
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            ctx.sync()
        kt = {}
        for e in prof.key_averages():
            k = next((k for k in KERNELS if k in e.key), None)
            if k:
                kt[k] = kt.get(k, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
        src_px = (min(sw * sh, dw * dh), min(sw * sh, 4 * dw * dh), sw * sh + 2 * sh * dw)[alg]
        moved = n * (src_px + dw * dh) * bpp
        frame0 = src[0].cpu().numpy()
        t0 = time.perf_counter()
        want = rz.resize(frame0, sw, sh, dw, dh, ct, alg)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        assert np.array_equal(dst[0].cpu().numpy(), want), "device output differs from the oracle"
        r = {"frames": n, "src": [sw, sh], "dst": [dw, dh], "bytes_per_pixel": bpp, "algorithm": NAMES[alg],
             "call_ms": round(ms, 3), "bytes_moved": moved, "achieved_gb_per_s": round(moved / ms / 1e6, 1),
             "fraction_of_peak_bandwidth": round(moved / (ms / 1e3) / PEAK, 3),
             "kernel_ms": {k: round(v, 3) for k, v in sorted(kt.items())},
             "oracle_ms_per_frame": round(oracle_ms, 1)}
        rec["workloads"].append(r)
        print(json.dumps(r), flush=True)
        del src, dst
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
