"""Times the host-buffer entry points on 4K frames in ordinary (pageable) numpy buffers, as a pixo caller hands
them over: each call stages its frames to the device, runs its kernels and copies the results back, so a call's
wall time is what the caller waits for.  One frame per call, except the JPEG batch calls: 8 baseline frames
(two groups of 4) and 4 progressive frames (two groups of 2).  jpeg_entropy_encode_dev takes the frame's
coefficients already on the device and returns the file in host memory.

    python tools/host_calls_time.py [--reps N]                      (the library PIXO_B200_SO selects)
    python tools/host_calls_time.py --ab A.so B.so [--rounds R] [--out out.json]

--ab runs the two libraries in alternating fresh processes, R rounds each, and reports per call the median
of each round (milliseconds), the median over the rounds, B / A, and whether both computed the same bytes.
The card's name, power limit and maximum SM clock are read in the same run.  profiles/h100_host_calls.json,
profiles/h100_host_encode_calls.json and profiles/h100_host_encode_tables.json hold such comparisons.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

W, H = 3840, 2160


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frame(bpp, seed):
    """A gradient with noise: every call does its full work (no reduction, many colours)."""
    rng = np.random.default_rng(seed)
    x = np.arange(W)[None, :, None] + 2 * np.arange(H)[:, None, None] + 60 * np.arange(bpp)[None, None, :]
    return ((x + rng.integers(0, 24, (H, W, bpp))) & 255).astype(np.uint8).reshape(-1)


def few_colours(n, seed):
    """RGBA pixels of n colours: quantisation designs its palette from at most 8192 of them."""
    rng = np.random.default_rng(seed)
    colours = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    return colours[rng.integers(0, n, W * H)].reshape(-1)


def calls(ctx):
    """name -> a call returning the bytes it produced"""
    from pixo_b200 import ColorType, jpeg, png
    from pixo_b200 import resize as rs
    from pixo_b200.jpeg import Subsampling
    from pixo_b200.png import FilterStrategy, PngOptions, QuantizationMode
    import torch
    rgb, rgba, indexed = frame(3, 1), frame(4, 2), few_colours(4000, 3)
    batch = np.stack([rgb] + [frame(3, 10 + k) for k in range(7)])
    q80 = jpeg.JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420)
    pmax = jpeg.JpegOptions.max(W, H, 80)
    balanced = jpeg.JpegOptions.balanced(W, H, 75)
    d_coef = [torch.from_numpy(a).cuda() for a in jpeg.compute_all_coefficients(rgb, W, H, ColorType.Rgb,
                                                                                 Subsampling.S444, 75, ctx=ctx)]
    torch.cuda.synchronize()
    quant = PngOptions(W, H, ColorType.Rgba, FilterStrategy.Adaptive, True, True, True, QuantizationMode.Force, 256, True)
    lanczos = rs.ResizeOptions.builder(W, H).dst(1920, 1080).color_type(ColorType.Rgba).algorithm(
        rs.ResizeAlgorithm.Lanczos3).build()
    return {
        "jpeg_coefficients_420_histograms": lambda: b"".join(
            a.tobytes() for a in jpeg.compute_all_coefficients(rgb, W, H, ColorType.Rgb, Subsampling.S420, 80,
                                                               histograms=True, ctx=ctx)),
        "png_filter_adaptive": lambda: b"".join(
            np.asarray(a).tobytes() for a in png.apply_filters(rgba, W, H, 4, PngOptions(W, H, ColorType.Rgba),
                                                               with_adler=True, ctx=ctx)),
        "png_reduce_filter_balanced": lambda: png.reduce_and_filter(rgba, PngOptions.from_preset(W, H, 1),
                                                                    ctx=ctx)[1].tobytes(),
        "png_quantize_filter_256_dither": lambda: png.quantize_and_filter(indexed, quant, ctx=ctx)[1].tobytes(),
        "adler32": lambda: png.adler32(rgba, ctx=ctx).to_bytes(4, "little"),
        "resize_lanczos3_to_1080p": lambda: rs.resize(rgba, lanczos, ctx=ctx).tobytes(),
        "jpeg_encode_420_q80": lambda: jpeg.encode(rgb, q80, ctx=ctx),
        "jpeg_encode_batch_8x_420_q80": lambda: b"".join(jpeg.encode_batch(batch, q80, ctx=ctx)),
        "jpeg_encode_progressive_max_q80": lambda: jpeg.encode_progressive(rgb, pmax, ctx=ctx),
        "jpeg_encode_progressive_batch_4x_max_q80": lambda: b"".join(
            jpeg.encode_progressive_batch(batch[:4], pmax, ctx=ctx)),
        "jpeg_encode_balanced_q75": lambda: jpeg.encode(rgb, balanced, ctx=ctx),
        "jpeg_encode_batch_8x_balanced_q75": lambda: b"".join(jpeg.encode_batch(batch, balanced, ctx=ctx)),
        "jpeg_entropy_encode_dev_444_q75_optimized": lambda: jpeg.entropy_encode_dev(*d_coef, balanced, ctx=ctx),
    }


def measure(reps):
    """One process, one library: per call the median and minimum wall time (ms) after two warm-up calls, and
    the CRC-32 of what the call produced."""
    import pixo_b200
    ctx = pixo_b200.Context(0)
    out = {}
    for name, fn in calls(ctx).items():
        crc = zlib.crc32(fn())
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()   # synchronous: returns with the results in the caller's memory
            ts.append((time.perf_counter() - t0) * 1e3)
        out[name] = {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3), "crc32": crc}
    return out


def run_child(so, reps):
    env = dict(os.environ, PIXO_B200_SO=os.path.abspath(so))
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--reps", str(reps)], env=env, capture_output=True,
                       text=True)
    if p.returncode != 0:
        raise RuntimeError(f"{so}: {p.stderr[-2000:]}")
    return json.loads(p.stdout.strip().splitlines()[-1])["calls"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--ab", nargs=2, metavar=("A_SO", "B_SO"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not args.ab:
        print(json.dumps({"card": gpu_info(), "calls": measure(args.reps)}))
        return
    runs = {"A": [], "B": []}
    for _ in range(args.rounds):
        for key, so in zip("AB", args.ab):
            runs[key].append(run_child(so, args.reps))
    rec = {"card (name, power limit, max SM clock)": gpu_info(), "A": args.ab[0], "B": args.ab[1],
           "note": f"ms per call on {W}x{H} frames in pageable numpy memory: median of {args.reps} calls after "
                   f"two warm-up calls, per round; {args.rounds} rounds per library, alternating A and B",
           "calls": {}}
    for name in runs["A"][0]:
        a = [r[name]["median_ms"] for r in runs["A"]]
        b = [r[name]["median_ms"] for r in runs["B"]]
        rec["calls"][name] = {"A_rounds_ms": a, "B_rounds_ms": b,
                              "A_ms": statistics.median(a), "B_ms": statistics.median(b),
                              "B_over_A": round(statistics.median(b) / statistics.median(a), 3),
                              "same_bytes": all(r[name]["crc32"] == runs["A"][0][name]["crc32"]
                                                for r in runs["A"] + runs["B"])}
        print(name, json.dumps(rec["calls"][name]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(rec, open(args.out, "w"), indent=1)
    print(json.dumps({"card": rec["card (name, power limit, max SM clock)"]}))


if __name__ == "__main__":
    main()
