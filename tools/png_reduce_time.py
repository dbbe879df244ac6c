"""Times pixo_b200_png_reduce_filter_dev on 16 4K RGBA frames per content class (CUDA events, after
warm-up) next to pixo_b200_png_filter_dev on the same frames, and the analysis kernel's share of HBM
bandwidth; the CPU figure is oracle/png_reduce.py (the numpy restatement, not pixo) on one frame.

    python tools/png_reduce_time.py [out.json]        (needs a GPU; writes profiles/h100_png_reduce.json)
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pixo_b200  # noqa: E402
from pixo_b200 import ColorType, _lib, png  # noqa: E402
from pixo_b200.png import PngOptions  # noqa: E402
from oracle import png_reduce as pr  # noqa: E402
from reduce_inputs import make_reduce_input  # noqa: E402

W, H, N, REPS = 3840, 2160, 16, 10
HBM = 3.35e12   # H100 SXM data sheet
KERNELS = ("k_reduce_analyze", "k_reduce_index", "k_reduce_pack", "k_png_band", "k_png_filter")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


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
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_png_reduce.json")
    ctx = pixo_b200.Context(0)
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)   # the library's work and the events share one stream
    opts = PngOptions.from_preset(W, H, 1)
    opts.color_type = ColorType.Rgba
    in_stride, out_stride = W * H * 4, H * (W * 4 + 1)
    d_in = torch.empty(N * in_stride, dtype=torch.uint8, device=dev)
    d_out = torch.empty(N * out_stride, dtype=torch.uint8, device=dev)
    d_ad = torch.zeros(N, dtype=torch.int32, device=dev)
    classes = {"palette200": ("palblk", 200), "opaque": ("opaque", 0), "gray_alpha": ("grayalpha", 0),
               "noise": ("noise", 0)}
    rec = {"card": gpu_info(), "frames": N, "width": W, "height": H, "preset": 1, "classes": {}}
    for name, (kind, n) in classes.items():
        frame = make_reduce_input(kind, W, H, 4, 1, n)
        d_frame = torch.from_numpy(frame).to(dev)
        for i in range(N):
            d_in[i * in_stride:(i + 1) * in_stride] = torch.roll(d_frame.view(H, -1), i, 0).reshape(-1)
        torch.cuda.synchronize()

        def reduce_call():
            png.reduce_and_filter_dev(d_in, in_stride, N, opts, d_out, out_stride, d_ad, ctx=ctx)

        def filter_call():
            _lib.check(ctx.handle, lib.pixo_b200_png_filter_dev(ctx.handle, d_in.data_ptr(), in_stride, N, W, H,
                                                                W * 4, 4, int(opts.filter_strategy) | 0x100,
                                                                d_out.data_ptr(), out_stride, d_ad.data_ptr()))

        for _ in range(2):
            reduce_call(); filter_call()   # noqa: E702
        ctx.sync()
        t_red = events_ms(reduce_call, stream)
        t_flt = events_ms(filter_call, stream)
        info = png.reduce_and_filter_dev(d_in, in_stride, N, opts, d_out, out_stride, d_ad, ctx=ctx)[0]
        # the analysis kernel alone, from the profiler
        from torch.profiler import ProfilerActivity, profile
        ctx.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            reduce_call()
            ctx.sync()
        kt = {}
        for e in prof.key_averages():
            k = next((k for k in KERNELS if k in e.key), None)
            if k:
                kt[k] = kt.get(k, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
        t_an = next((v for k, v in kt.items() if "k_reduce_analyze" in k), None)
        an_bytes = N * in_stride   # upper bound: every pixel read once
        t0 = time.perf_counter()
        pr.reduce(frame, W, H, 3, True, True)
        host_s = time.perf_counter() - t0
        rec["classes"][name] = {
            "reduces_to": {"color_type": info.color_type_byte, "bit_depth": info.bit_depth,
                           "palette_len": 0 if info.palette is None else len(info.palette)},
            "reduce_filter_dev_ms": round(t_red, 3), "filter_dev_ms": round(t_flt, 3),
            "reduce_overhead_ms": round(t_red - t_flt, 3), "kernel_ms": {k: round(v, 3) for k, v in kt.items()},
            "analyze_algorithmic_bytes_upper": an_bytes,
            "analyze_fraction_of_3.35TBps": None if not t_an else round(an_bytes / (t_an * 1e-3) / HBM, 3),
            "oracle_restatement_host_s_one_frame": round(host_s, 3)}
        print(name, json.dumps(rec["classes"][name]))
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
