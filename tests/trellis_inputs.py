"""Inputs of the trellis fixtures (oracle/wasm_ref/gen_golden_trellis.py) and of the tests that re-encode
them: tests/golden_inputs.py kinds, plus "hifreq", whose 8x8 blocks each hold one high-frequency cosine
product, so a block's quantised coefficients have a long zero run before one non-zero (ZRL states)."""
import numpy as np

from golden_inputs import make_input


def make_trellis_input(kind: str, w: int, h: int, ch: int, seed: int) -> np.ndarray:
    if kind == "gradient" and ch == 1:
        kind = "vgrad"   # the RGB gradient has no gray form
    if kind != "hifreq":
        return make_input(kind, w, h, ch, seed)
    rng = np.random.default_rng(seed)
    bw, bh = (w + 7) // 8, (h + 7) // 8
    u = rng.integers(3, 8, (bh, bw)); v = rng.integers(3, 8, (bh, bw))
    a = rng.uniform(20.0, 110.0, (bh, bw)) * rng.choice([-1, 1], (bh, bw))
    x = np.arange(w); y = np.arange(h)
    bu, bv, ba = (np.repeat(np.repeat(t, 8, 0), 8, 1)[:h, :w] for t in (u, v, a))
    cx = np.cos((2 * (x % 8) + 1)[None, :] * bu * np.pi / 16)
    cy = np.cos((2 * (y % 8) + 1)[:, None] * bv * np.pi / 16)
    img = np.clip(np.round(128 + ba * cx * cy), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(np.repeat(img[..., None], ch, -1)).reshape(-1)
