"""Times pixo_b200_png_quantize_filter_dev on 16 4K RGBA frames per content class, dithered and plain
(CUDA events, after warm-up), with per-kernel times from torch.profiler in a run of their own, and the
card's name and power limit read in the same run.

    python tools/png_quantize_time.py [out.json]      (needs a GPU; writes profiles/h100_png_quantize.json)

Classes: about 1 000 opaque colours in blocks (Auto quantises: median cut + k-means), an opaque gradient
with noise mapped to a given 256-entry palette (Force; the gradient has more than 8 192 histogram colours,
pixo's truncation case, so the palette comes from the caller), 4 000 colours of which two thirds are
translucent (Auto; every translucent pixel is a full nearest-entry search), and noise (Auto declines: the
lossless reduction path).
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pixo_b200  # noqa: E402
from pixo_b200 import ColorType, png  # noqa: E402
from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode  # noqa: E402
from oracle import png_quantize as pq  # noqa: E402
from quantize_inputs import make_quantize_input  # noqa: E402

W, H, N, REPS = 3840, 2160, 16, 5
KERNELS = ("k_quant_sample", "k_quant_kmeans", "k_quant_update", "k_quant_lut", "k_quant_map", "k_quant_dither",
           "k_png_band", "k_png_filter", "k_reduce_analyze", "k_reduce_index", "k_reduce_pack", "RadixSort",
           "RunLength", "Rle")


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


def given_palette(frame):
    """A 256-entry palette the way a caller keeping palette design would make one: median cut and k-means
    on the 8 192 most frequent histogram colours."""
    keys, counts = pq.histogram(frame, 3)
    keep = np.sort(np.argsort(-counts.astype(np.int64), kind="stable")[:8192])
    return pq.kmeans(pq.median_cut(keys[keep], counts[keep], 256), keys[keep], counts[keep])


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_png_quantize.json")
    ctx = pixo_b200.Context(0)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    ctx.set_stream(stream.cuda_stream)   # the library's work and the events share one stream
    in_stride, out_stride = W * H * 4, H * (W * 4 + 1)
    d_in = torch.empty(N * in_stride, dtype=torch.uint8, device=dev)
    d_out = torch.empty(N * out_stride, dtype=torch.uint8, device=dev)
    d_ad = torch.zeros(N, dtype=torch.int32, device=dev)
    classes = {"blocks1000_opaque_auto": ("palblk", 1000, QuantizationMode.Auto),
               "gradient_noise_opaque_force_given_palette": ("grad", 0, QuantizationMode.Force),
               "translucent4000_auto": ("pal", 4000, QuantizationMode.Auto),
               "noise_auto_declines": ("noise", 0, QuantizationMode.Auto)}
    rec = {"card": gpu_info(), "frames": N, "width": W, "height": H, "preset": 1,
           "note": "ms per call of pixo_b200_png_quantize_filter_dev on 16 frames; CUDA events", "classes": {}}
    for name, (kind, n, mode) in classes.items():
        frame = make_quantize_input(kind, W, H, 4, 1, n)
        if kind in ("palblk", "grad"):
            frame.reshape(-1, 4)[:, 3] = 255      # opaque: the 6-6-6 table maps every pixel
        pals = [given_palette(frame)] * N if kind == "grad" else None
        d_frame = torch.from_numpy(frame).to(dev)
        for i in range(N):
            d_in[i * in_stride:(i + 1) * in_stride] = torch.roll(d_frame.view(H, -1), i, 0).reshape(-1)
        torch.cuda.synchronize()
        r = {}
        for dither in (True, False):
            opts = PngOptions(W, H, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, mode, 256, dither)

            def call():
                return png.quantize_and_filter_dev(d_in, in_stride, N, opts, d_out, out_stride, d_ad, palettes=pals,
                                                   ctx=ctx)
            info = call()
            ctx.sync()
            t = events_ms(call, stream)
            from torch.profiler import ProfilerActivity, profile
            ctx.sync()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                call()
                ctx.sync()
            kt = {}
            for e in prof.key_averages():
                k = next((k for k in KERNELS if k in e.key), None)
                if k:
                    kt[k] = kt.get(k, 0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1000.0
            r["dither" if dither else "plain"] = {
                "call_ms": round(t, 3), "kernel_ms": {k: round(v, 3) for k, v in sorted(kt.items())},
                "color_type": info[0].color_type_byte,
                "palette_len": 0 if info[0].palette is None else len(info[0].palette)}
        rec["classes"][name] = r
        print(name, json.dumps(r), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    json.dump(rec, open(out_path, "w"), indent=1)
    print(json.dumps({"card": rec["card"]}))


if __name__ == "__main__":
    main()
