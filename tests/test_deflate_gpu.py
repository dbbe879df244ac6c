"""The GPU DEFLATE (png_deflate.cu: k_lz77, k_deflate_emit) against the oracle and real pixo output."""
import zlib

import numpy as np
import pytest
import torch

from deflate_inputs import constructed, golden_pngs, idat
from oracle import png_deflate as pd

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _build():
    pd.build()


def _batch(streams, level, ctx, cap=None, guard=64):
    """Every stream in one call, in back-to-back slots of exactly `cap` bytes between a leading and a trailing guard;
    returns (outputs, lens, status).  Checks that nothing was written to the guards, past a stream's length in its
    slot, or into a slot that was too small."""
    from pixo_b200 import compress
    stride = max(max((len(s) for s in streams), default=0), 1)
    src = np.zeros((len(streams), stride), np.uint8)
    for i, s in enumerate(streams):
        src[i, :len(s)] = np.frombuffer(s, np.uint8)
    cap = cap or 2 + stride + (stride // 65535 + 1) * 5 + 4
    d_src = torch.from_numpy(src).cuda()
    d_out = torch.full((guard + len(streams) * cap + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    lens, status = compress.deflate_zlib_packed_dev(d_src, stride, [len(s) for s in streams], level, d_out[guard:],
                                                    cap, ctx=ctx)
    host = d_out.cpu().numpy()
    assert (host[:guard] == 0xA5).all() and (host[guard + len(streams) * cap:] == 0xA5).all()
    outs = []
    for i in range(len(streams)):
        slot = host[guard + i * cap:guard + (i + 1) * cap]
        n = int(lens[i]) if status[i] == 0 else 0
        assert (slot[n:] == 0xA5).all(), i
        outs.append(slot[:n].tobytes())
    return outs, lens, status


def test_host_entry_point_reproduces_golden_idat(gpu_ctx):
    from pixo_b200 import compress
    for path, level in golden_pngs()[::9]:
        z = idat(open(path, "rb").read())
        assert compress.deflate_zlib_packed(zlib.decompress(z), level, ctx=gpu_ctx) == z, path


@pytest.mark.parametrize("level", [2, 6])
def test_dev_batch_reproduces_every_golden_idat(gpu_ctx, level):
    files = [(p, lv) for p, lv in golden_pngs() if lv == level]
    zs = [idat(open(p, "rb").read()) for p, _ in files]
    outs, _, status = _batch([zlib.decompress(z) for z in zs], level, gpu_ctx)
    assert (status == 0).all()
    for (p, _), z, o in zip(files, zs, outs):
        assert o == z, p


@pytest.mark.parametrize("level", range(1, 10))
def test_constructed_streams_equal_the_oracle(gpu_ctx, level):
    items = list(constructed().items())
    outs, lens, status = _batch([d for _, d in items], level, gpu_ctx)
    assert (status == 0).all()
    for (name, d), o in zip(items, outs):
        assert o == pd.deflate_zlib(d, level), (name, level)
        assert zlib.decompress(o) == d


def test_small_slots_are_refused_and_left_untouched(gpu_ctx):
    from pixo_b200 import _lib
    c = constructed()
    streams = [c["text"], c["tiny_fixed"], c["noise_12k"], c["empty"], c["tiny_fixed"]]
    want = [pd.deflate_zlib(s, 6) for s in streams]
    cap = len(want[1])   # the fixed stream fits exactly; text and noise do not
    outs, lens, status = _batch(streams, 6, gpu_ctx, cap=cap)
    assert [int(x) for x in lens] == [len(w) for w in want]
    assert [int(x) for x in status] == [0 if len(w) <= cap else _lib.ERR_OUTPUT_TOO_SMALL for w in want]
    assert status[0] == _lib.ERR_OUTPUT_TOO_SMALL and status[1] == 0
    for w, o, st in zip(want, outs, status):
        if st == 0:
            assert o == w


def test_batch_across_passes(gpu_ctx):
    """65 537 streams: a pass holds at most 65 536, so the last stream goes in a second pass, after the first pass's
    coding and with the scratch bound again."""
    rng = np.random.default_rng(4)
    streams = [bytes([i & 0xFF]) * int(rng.integers(0, 40)) + bytes([i >> 8 & 0xFF, i & 0xFF]) for i in range(65537)]
    before = gpu_ctx.launch_count
    outs, _, status = _batch(streams, 6, gpu_ctx, guard=16)
    assert gpu_ctx.launch_count - before == 4   # k_lz77 and k_deflate_emit per pass
    assert (status == 0).all()
    for i in list(range(0, 65537, 997)) + [65535, 65536]:
        assert outs[i] == pd.deflate_zlib(streams[i], 6), i
    assert all(zlib.decompress(o) == s for o, s in zip(outs, streams))


def test_overlapping_streams_are_refused(gpu_ctx):
    import pixo_b200
    from pixo_b200 import _lib, compress
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    with pytest.raises(pixo_b200.PixoError) as e:
        compress.deflate_zlib_packed_dev(d, 16, [16, 17], 6, d, 64, ctx=gpu_ctx)
    assert e.value.code == _lib.ERR_INVALID_DATA_LENGTH


def test_level_and_launches(gpu_ctx):
    import pixo_b200
    from pixo_b200 import _lib, compress
    with pytest.raises(pixo_b200.PixoError) as e:
        compress.deflate_zlib_packed(b"abc", 10, ctx=gpu_ctx)
    assert e.value.code == _lib.ERR_INVALID_COMPRESSION_LEVEL and "Invalid compression level 10: must be 1-9" in str(e.value)
    before = gpu_ctx.launch_count
    compress.deflate_zlib_packed(constructed()["text"], 6, ctx=gpu_ctx)
    assert gpu_ctx.launch_count - before == 2   # k_lz77, k_deflate_emit: one pass
    assert gpu_ctx.host_fallbacks == 0


def test_full_size_frames(gpu_ctx):
    """Filtered 4K RGBA frames (smooth and noisy rows) at levels 2 and 6, equal to the oracle."""
    rng = np.random.default_rng(11)
    w, h = 3840, 2160
    rows = (np.arange(w * 4, dtype=np.uint32)[None, :] // 9 + np.arange(h, dtype=np.uint32)[:, None] // 5) & 0xFF
    smooth = np.concatenate([np.ones((h, 1), np.uint32), rows], axis=1).astype(np.uint8).tobytes()
    noisy = bytearray(smooth)
    noisy[1000000:1400000] = rng.integers(0, 256, 400000, dtype=np.uint8).tobytes()
    for level in (2, 6):
        outs, _, status = _batch([smooth, bytes(noisy)], level, gpu_ctx)
        assert (status == 0).all()
        assert outs[0] == pd.deflate_zlib(smooth, level)
        assert outs[1] == pd.deflate_zlib(bytes(noisy), level)
        assert zlib.decompress(outs[1]) == bytes(noisy)
