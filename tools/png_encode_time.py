"""Times pixo_b200_png_encode_on_device (whole PNG files) at presets 0 and 1 on 32 1080p RGBA frames of three kinds
and on one 4K frame: the call's time on the host clock (the call returns synchronised), the compression ratio, the
same files through the three-call route (quantize_and_filter -> deflate_zlib_packed -> png_file, one frame at a
time, on the first OLD frames, per frame), and per-kernel times from torch.profiler in a run of their own, with k_png_idat's bytes/s (the zlib bytes read
and written) against the 3.35 TB/s data sheet.  The card's name and power limit are read in the same run.

    python tools/png_encode_time.py [out.json]      (needs a GPU; writes profiles/h100_png_encode.json)

Kinds: palette-like blocks (few colours: the palette route), a gradient with noise (many colours, DEFLATE finds
short matches) and RGBA noise (stored blocks: the most bytes through the container kernels).
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
from pixo_b200 import ColorType, compress, png  # noqa: E402
from oracle import png_deflate as pd  # noqa: E402

REPS = 1
OLD = 4
KERNELS = ("k_png_idat_finish", "k_png_idat", "k_lz77", "k_deflate_emit", "k_png_band", "k_png_filter",
           "k_reduce_analyze", "k_reduce_index", "k_reduce_pack", "k_quant")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frames(kind, n, w, h, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        if kind == "blocks":
            pal = rng.integers(0, 256, (24, 4), dtype=np.uint8)
            pal[:, 3] = 255
            idx = rng.integers(0, 24, (h // 16 + 1, w // 16 + 1))
            img = pal[np.kron(idx, np.ones((16, 16), np.int64))[:h, :w]]
        elif kind == "gradient_noise":
            g = (np.arange(w)[None, :, None] * 3 + np.arange(h)[:, None, None] * 2 + np.arange(4) * 50 + i) % 256
            img = np.clip(g + rng.integers(-6, 7, (h, w, 4)), 0, 255).astype(np.uint8)
            img[..., 3] = 255
        else:
            img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        out.append(np.ascontiguousarray(img))
    return out


def old_route(imgs, o, ctx):
    """The three calls a caller made before: the filter stage, DEFLATE and the container on the host."""
    files = []
    for img in imgs:
        red, f, _ = png.quantize_and_filter(img, o, ctx=ctx)
        z = compress.deflate_zlib_packed(f, o.compression_level, ctx=ctx)
        files.append(pd.png_file(o.width, o.height, red.bit_depth, red.color_type_byte, z, red.palette, red.trns))
    return files


def main(out_path):
    ctx = pixo_b200.Context(0)
    info = gpu_info()
    loads = [(kind, preset, 32, 1920, 1080) for kind in ("blocks", "gradient_noise", "noise") for preset in (0, 1)]
    loads += [("gradient_noise", preset, 1, 3840, 2160) for preset in (0, 1)]
    rows = []
    for kind, preset, n, w, h in loads:
        imgs = frames(kind, n, w, h)
        o = png.PngOptions.from_preset(w, h, preset)
        d_in = torch.from_numpy(np.stack(imgs).reshape(-1)).cuda()
        cap = png.encode_capacity(w, h, ColorType.Rgba)
        d_out = torch.empty(n * cap, dtype=torch.uint8, device="cuda")
        run = lambda: png.encode_on_device(d_in, w * h * 4, n, o, d_out, cap, ctx=ctx)
        lens, status, _ = run()
        assert (status == 0).all()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(REPS):
            run()
        call_ms = (time.perf_counter() - t0) / REPS * 1e3
        host = d_out.cpu().numpy()
        files = [host[i * cap:i * cap + int(lens[i])].tobytes() for i in range(n)]
        t0 = time.perf_counter()
        old = old_route(imgs[:OLD], o, ctx)
        old_ms = (time.perf_counter() - t0) * 1e3 / len(old)
        assert old == files[:OLD], (kind, preset)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            name = next((k for k in KERNELS if k in e.key), None)
            if name:
                kern[name] = kern.get(name, 0.0) + e.device_time_total / 1e3
        zbytes = sum(len(f) for f in files)
        idat_ms = kern.get("k_png_idat", 0.0)
        row = {"kind": kind, "preset": preset, "frames": n, "width": w, "height": h,
               "encode_on_device_ms": round(call_ms, 2), "old_route_ms_per_frame": round(old_ms, 2),
               "compression_ratio": round(n * w * h * 4 / zbytes, 3), "file_bytes": zbytes,
               "kernel_ms": {k: round(v, 3) for k, v in kern.items()},
               "k_png_idat_GBps": round(2 * zbytes / (idat_ms * 1e-3) / 1e9, 1) if idat_ms else None,
               "k_png_idat_share_of_3_35_TBps": round(2 * zbytes / (idat_ms * 1e-3) / 3.35e12, 4) if idat_ms else None}
        print(json.dumps(row), flush=True)
        rows.append(row)
    rec = {"gpu": info, "what": "pixo_b200_png_encode_on_device, whole PNG files; host clock around a call that ends "
                                "synchronised, mean of %d call(s) after one warm-up call" % REPS, "rows": rows}
    with open(out_path, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", out_path, "on", info)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_png_encode.json"))
