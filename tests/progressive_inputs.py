"""Inputs of the progressive fixtures (oracle/wasm_ref/gen_golden_progressive.py) and of the tests that
re-encode them: mostly flat frames whose few busy 8x8 blocks sit where the EOB runs of the Y AC scans
between them are exactly 32 766, 32 767 and 32 768 empty blocks, and one run long enough to reach 0x7FFF
twice.  busy: Y block indices (compute_all_coefficients order: MCU order for 4:2:0) that hold noise."""
import numpy as np

CASES = [
    dict(w=2048, h=1024, ct=0, s420=0, q=80, seed=1, busy=[0, 32767]),           # 32 766 empties
    dict(w=2048, h=1032, ct=2, s420=0, q=80, seed=2, busy=[0, 32768, 33023]),    # 32 767
    dict(w=2048, h=1056, ct=2, s420=1, q=80, seed=3, busy=[5, 32774]),           # 32 768
    dict(w=4096, h=2048, ct=0, s420=0, q=80, seed=4, busy=[1, 70001]),           # 69 999: 0x7FFF twice
]


def block_origin(k: int, w: int, ct: int, s420: int):
    """Pixel (x, y) of Y block k in compute_all_coefficients order."""
    if ct == 0 or s420 == 0:
        bw = (w + 7) // 8
        return (k % bw) * 8, (k // bw) * 8
    mx = (w + 15) // 16
    mcu, sub = divmod(k, 4)
    return (mcu % mx) * 16 + (sub & 1) * 8, (mcu // mx) * 16 + (sub >> 1) * 8


def make_progressive_input(c) -> np.ndarray:
    ch = 1 if c["ct"] == 0 else 3
    img = np.full((c["h"], c["w"], ch), 120, np.uint8)
    rng = np.random.default_rng(c["seed"])
    for k in c["busy"]:
        x, y = block_origin(k, c["w"], c["ct"], c["s420"])
        img[y:y + 8, x:x + 8] = rng.choice(np.array([0, 255], np.uint8), (8, 8, ch))
    return np.ascontiguousarray(img).reshape(-1)
