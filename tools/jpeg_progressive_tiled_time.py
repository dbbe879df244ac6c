"""Times one 16 384 x 16 384 frame at pixo's max preset (4:2:0, q80, optimised tables, trellis) whole and in MCU-row
bands (pixo_b200.parallel's progressive tiled flow), and writes profiles/h100_jpeg_progressive_tiled.json with the
card's name and power limit:
  - whole: pixo_b200_jpeg_encode_dev_progressive on one GPU (CUDA events, mean of REPS after one warm-up call);
  - 8 bands on one GPU, each band on its own: its transform, trellis, summary, statistics, band stage and splices,
    host clock around work that ends in a device synchronise (the band calls wait for the device), mean of REPS;
    the sum over the bands is what one GPU spends, the slowest band a bound on an 8-GPU wall time without the
    collectives;
  - the same 8 bands over NCCL, one process per GPU (wall time of rank 0 from a barrier to the file), only on a
    machine with >= 8 GPUs (or as many as it has, >= 2); "not measured" otherwise.
Every tiled file is checked against the whole frame's (sha256).  Content: 8x8 blocks of random colour with light
noise on every third row (as tools/jpeg_progressive_time.py).

    python tools/jpeg_progressive_tiled_time.py [out.json]
"""
import hashlib
import json
import os
import socket
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pixo_b200  # noqa: E402
from pixo_b200 import ColorType, jpeg, parallel  # noqa: E402
from pixo_b200.jpeg import JpegOptions, Subsampling  # noqa: E402

REPS = 3
W = H = 16384
WORLD = 8


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def frame(dev, seed=3):
    g = torch.Generator(device=dev).manual_seed(seed)
    base = torch.randint(0, 256, ((H + 7) // 8, (W + 7) // 8, 3), dtype=torch.uint8, device=dev, generator=g)
    f = base.repeat_interleave(8, 0).repeat_interleave(8, 1)[:H, :W].contiguous()
    f[::3] ^= torch.randint(0, 8, f[::3].shape, dtype=torch.uint8, device=dev, generator=g)
    return f


def options():
    return JpegOptions(W, H, ColorType.Rgb, 80, Subsampling.S420, None, True, True, True)


def whole(ctx, d_px, o):
    cap = (W * H * 3 // 2 + 65536) // 16 * 16
    out = torch.empty(cap, dtype=torch.uint8, device=d_px.device)
    lens = torch.empty((1, 7), dtype=torch.int64, device=d_px.device)
    ovf = torch.empty(1, dtype=torch.int32, device=d_px.device)
    dht = torch.empty((1, jpeg.DHT_BYTES), dtype=torch.uint8, device=d_px.device)
    stream = torch.cuda.Stream(d_px.device)
    torch.cuda.synchronize()
    ctx.set_stream(stream.cuda_stream)
    run = lambda: jpeg.encode_progressive_dev(d_px, d_px.numel(), 1, o, out, cap, lens, ovf, dht, ctx=ctx)
    run()
    stream.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(REPS):
        run()
    b.record(stream)
    b.synchronize()
    ctx.set_stream(None)
    assert not ovf.cpu().numpy().any()
    f = jpeg.progressive_file(o, dht.cpu().numpy()[0], out.cpu().numpy(), lens.cpu().numpy()[0])
    return a.elapsed_time(b) / REPS, f


def band_steps(ctx, rows, o, bands, r, seed, carry, hist):
    """Band r on its own: transform + trellis, summary, statistics, band stage, 7 splices (seeds, carries and the
    summed statistics are the frame's, taken from an untimed run)."""
    c = parallel.progressive_band_coder(ctx, rows, W, H, 2, 1, o.quality, True, bands, r)
    c.summary()
    c.histogram(seed[0])
    nbits, tails = c.code(seed[1], carry, hist)
    for k in range(7):
        c.splice(k, nbits[k], 0, 0, True)
    ctx.sync()


def bands_on_one_gpu(ctx, d_px, o):
    bands = parallel.plan_bands(W, H, WORLD)
    rows = [d_px[b.px_row0:b.px_row1].reshape(-1) for b in bands]
    coders = [parallel.progressive_band_coder(ctx, rows[r], W, H, 2, 1, o.quality, True, bands, r) for r in range(WORLD)]
    t0 = time.perf_counter()
    f = parallel.encode_progressive_tiled_local(coders, o)
    torch.cuda.synchronize()
    local_ms = (time.perf_counter() - t0) * 1e3   # (band stages and splices only: the coders are built)
    s = np.array([c.summary() for c in coders], np.int64)
    counts = s[:, [10, 11, 11]]
    hist = sum(c.histogram(parallel.prog_dc_seeds(s[:, 0:3], counts, r)) for r, c in enumerate(coders))
    args = [((parallel.prog_dc_seeds(s[:, 0:3], counts, r), parallel.prog_dc_seeds(s[:, 3:6], counts, r)),
             parallel.ac_carries(s[:, 6:10], r)) for r in range(WORLD)]
    del coders
    per_band = []
    for r in range(WORLD):
        band_steps(ctx, rows[r], o, bands, r, args[r][0], args[r][1], hist)   # warm-up
        t0 = time.perf_counter()
        for _ in range(REPS):
            band_steps(ctx, rows[r], o, bands, r, args[r][0], args[r][1], hist)
        per_band.append((time.perf_counter() - t0) * 1e3 / REPS)
    return per_band, local_ms, f


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _nccl_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    ctx = pixo_b200.Context(rank)
    o = options()
    d_px = frame(torch.device("cuda", rank)).reshape(H, W * 3)
    bands = parallel.plan_bands(W, H, world)
    b = bands[rank]
    rows = d_px[b.px_row0:b.px_row1].reshape(-1).contiguous()
    times, f = [], None
    for _ in range(REPS + 1):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        coder = parallel.progressive_band_coder(ctx, rows, W, H, 2, 1, o.quality, True, bands, rank)
        f = parallel.encode_progressive_tiled(coder, o, rank, world)
        dist.barrier()
        times.append((time.perf_counter() - t0) * 1e3)
    if rank == 0:
        json.dump({"ms": float(np.mean(times[1:])), "sha256": hashlib.sha256(f).hexdigest()}, open(out_path, "w"))
    dist.destroy_process_group()


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "h100_jpeg_progressive_tiled.json")
    dev = torch.device("cuda", 0)
    ctx = pixo_b200.Context(0)
    o = options()
    d_px = frame(dev).reshape(H, W * 3)
    whole_ms, f_whole = whole(ctx, d_px.reshape(-1), o)
    sha = hashlib.sha256(f_whole).hexdigest()
    per_band, local_ms, f_local = bands_on_one_gpu(ctx, d_px, o)
    assert hashlib.sha256(f_local).hexdigest() == sha, "the tiled file differs from the whole frame's"
    ndev = torch.cuda.device_count()
    nccl = "not measured (needs >= 2 GPUs; this machine has %d)" % ndev
    if ndev >= 2:
        import tempfile
        import torch.multiprocessing as mp
        world = min(ndev, WORLD)
        tmp = os.path.join(tempfile.mkdtemp(), "nccl.json")
        mp.spawn(_nccl_worker, args=(world, _free_port(), tmp), nprocs=world, join=True)
        r = json.load(open(tmp))
        assert r["sha256"] == sha
        nccl = {"gpus": world, "wall_ms": round(r["ms"], 3)}
    rec = {
        "card": gpu_info(),
        "note": "ms; one 16 384 x 16 384 RGB frame, pixo's max preset (4:2:0 q80, optimised tables, trellis); whole: "
                "CUDA events, mean of %d after one warm-up call; bands: host clock around each band's calls (they wait "
                "for the device), mean of %d after one warm-up" % (REPS, REPS),
        "frame": {"width": W, "height": H, "file_bytes": len(f_whole), "sha256": sha},
        "whole_encode_dev_progressive_ms": round(whole_ms, 3),
        "bands_on_one_gpu": {
            "bands": WORLD,
            "per_band_ms": [round(t, 3) for t in per_band],
            "sum_ms": round(sum(per_band), 3),
            "slowest_band_ms": round(max(per_band), 3),
            "what": "each band's transform + trellis, summary, statistics, band stage and 7 splices on its own",
            "local_flow_ms": round(local_ms, 3),
            "local_flow_what": "encode_progressive_tiled_local over the 8 built coders: summaries, statistics, band "
                               "stages, splices and the file, one after the other",
            "file_identical": True,
        },
        "nccl": nccl,
    }
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as fo:
        json.dump(rec, fo, indent=1)
    print(json.dumps(rec, indent=1))


if __name__ == "__main__":
    main()
