"""Per-kernel device time of bench.py's encode step (pixo_b200_jpeg_encode_dev, 32 4K frames, q80
4:2:0, gradient / LCG noise alternating) from torch.profiler, in a run of its own.  --width / --height /
--frames / --quality / --s444 give the other configurations' shapes on the same frame mix.

    python tools/prof_encode_kernels.py [--root TREE] [--steps N] [--out FILE]

--root picks the tree whose pixo_b200 is imported (default: this one), so two builds can be compared
in one session.  Prints one JSON line: mean ms per step of every kernel the step launches."""
import argparse
import json
import os
import re
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--frames", type=int, default=32)
ap.add_argument("--width", type=int, default=3840)
ap.add_argument("--height", type=int, default=2160)
ap.add_argument("--quality", type=int, default=80)
ap.add_argument("--s444", action="store_true")
ap.add_argument("--out", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import pixo_b200  # noqa: E402
from pixo_b200 import _lib, synthetic  # noqa: E402

W, H, F = args.width, args.height, args.frames
SS = 0 if args.s444 else 1
lib = _lib.load()
ctx = pixo_b200.Context(0)
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)
ctx.set_stream(stream.cuda_stream)
g = synthetic.gradient_rgb(W, H).reshape(H, W * 3)
frames = np.stack([np.roll(g, k, axis=0).reshape(-1) if k % 2 == 0 else synthetic.noise(W, H, 3, 42 + k).reshape(-1)
                   for k in range(F)])
px = torch.from_numpy(frames).cuda()
cap = H * W * 3 // 256 * 256   # room for q=100 noise too: no frame overflows
scan = torch.empty((F, cap), dtype=torch.uint8, device="cuda")
slen = torch.zeros(F, dtype=torch.int64, device="cuda")
sovf = torch.zeros(F, dtype=torch.int32, device="cuda")


def step():
    _lib.check(ctx.handle, lib.pixo_b200_jpeg_encode_dev(ctx.handle, px.data_ptr(), H * W * 3, F, W, H, 2, args.quality, SS,
                                                         scan.data_ptr(), cap, slen.data_ptr(), sovf.data_ptr()))


for _ in range(3):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
per = {}
for e in prof.key_averages():
    if e.device_type == torch.autograd.DeviceType.CUDA and e.count:
        m = re.search(r"(k_\w+)(<[^>]*>)?", e.key)
        name = m.group(0) if m else e.key.strip()
        per[name] = per.get(name, 0.0) + e.device_time_total / 1e3 / args.steps   # us -> ms per step
res = {"root": os.path.abspath(args.root), "device": torch.cuda.get_device_name(0), "shape": f"{F}x{W}x{H} q{args.quality} "
       f"{'4:4:4' if args.s444 else '4:2:0'}", "steps": args.steps,
       "overflow": int(sovf.sum()), "ms_per_step": {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}}
print(json.dumps(res))
if args.out:
    with open(args.out, "a") as f:
        f.write(json.dumps(res) + "\n")
