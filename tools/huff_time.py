"""Entropy-stage time = encode_dev - coefficients_dev, CUDA events (dev aid; PIXO_B200_SO picks the library)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import pixo_b200
from pixo_b200 import _lib, jpeg, synthetic

lib = _lib.load()
ctx = pixo_b200.Context(0)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); ctx.set_stream(stream.cuda_stream)
W, H = 3840, 2160
g = synthetic.gradient_rgb(W, H).reshape(H, W * 3)
_, _, lq, cq = jpeg.quant_tables(80)
ny, nc = jpeg.block_counts(W, H, 2, 1)
res = []
for n, kind in [(1, "noise"), (1, "grad"), (8, "mix"), (32, "mix"), (32, "grad"), (32, "noise")]:
    fr = np.stack([np.roll(g, k, axis=0).reshape(-1) if (kind == "grad" or (kind == "mix" and k % 2 == 0))
                   else synthetic.noise(W, H, 3, 42 + k).reshape(-1) for k in range(n)])
    px = torch.from_numpy(fr).cuda()
    cap = (H * W * 3 // 2 + 65536 + 8192) // 256 * 256
    scan = torch.empty((n, cap), dtype=torch.uint8, device="cuda")
    sl = torch.zeros(n, dtype=torch.int64, device="cuda"); so = torch.zeros(n, dtype=torch.int32, device="cuda")
    y = torch.empty((n, ny * 64), dtype=torch.int16, device="cuda")
    cb = torch.empty((n, nc * 64), dtype=torch.int16, device="cuda"); cr = torch.empty_like(cb)
    def enc():
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_encode_dev(ctx.handle, px.data_ptr(), H * W * 3, n, W, H, 2, 80, 1,
                                                             scan.data_ptr(), cap, sl.data_ptr(), so.data_ptr()))
    def k1():
        _lib.check(ctx.handle, lib.pixo_b200_jpeg_coefficients_dev(
            ctx.handle, px.data_ptr(), H * W * 3, n, W, H, 2, 1, lq.ctypes.data_as(_lib.f32p),
            cq.ctypes.data_as(_lib.f32p), y.data_ptr(), ny * 64, cb.data_ptr(), cr.data_ptr(), nc * 64, 0, None))
    def t(fn, reps):
        for _ in range(3): fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps): fn()
        e1.record(stream); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps * 1e3
    reps = 20 if n < 32 else 8
    te, tk = t(enc, reps), t(k1, reps)
    res.append(f"n={n}/{kind}: enc {te:.0f} k1 {tk:.0f} huff {te - tk:.0f} us")
print(os.path.basename(os.environ.get("PIXO_B200_SO", "default")), "|", " | ".join(res))
