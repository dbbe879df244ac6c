"""Writes the libjpeg-turbo fixtures next to this file (through PIL) and their manifest.json: baseline files over
4:4:4, 4:2:2, 4:2:0 and gray at qualities 5-100, optimised tables, restart markers per block and per MCU row, custom
quantisation tables, sizes from 1x1 up; a CMYK and a progressive file the decoder refuses.  Seeded: the same PIL
writes the same bytes.  Run it from anywhere: python tests/golden/libjpeg/generate.py"""
import io
import json
import os

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))


def picture(w, h, seed, mode="RGB"):
    """a smooth field with edges and some noise, so every quality keeps a spread of coefficients"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    chans = 4 if mode == "CMYK" else 3
    base = np.stack([(x * (3 + c) + y * (5 - c) + 40 * ((x // 13 + y // 11 + c) % 2)) % 256 for c in range(chans)], -1)
    img = np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)
    if mode == "L":
        return Image.fromarray(img[..., 0], "L")
    return Image.fromarray(img, mode)


def cases():
    out = []
    for sub in ("4:4:4", "4:2:2", "4:2:0", "gray"):
        for q in (5, 50, 90, 100):
            out.append((f"q{q}_{sub.replace(':', '')}", 129, 67, sub, dict(quality=q)))
        for (w, h) in ((1, 1), (1, 37), (37, 1), (17, 9), (257, 131)):
            out.append((f"{w}x{h}_{sub.replace(':', '')}", w, h, sub, dict(quality=75)))
    for sub in ("4:2:2", "4:2:0", "gray"):
        out.append((f"optimize_{sub.replace(':', '')}", 129, 67, sub, dict(quality=80, optimize=True)))
    out.append(("restart_blocks1_420", 129, 67, "4:2:0", dict(quality=85, restart_marker_blocks=1)))
    out.append(("restart_blocks3_422", 97, 45, "4:2:2", dict(quality=85, restart_marker_blocks=3)))
    out.append(("restart_rows1_444", 129, 67, "4:4:4", dict(quality=85, restart_marker_rows=1)))
    out.append(("restart_rows2_gray", 131, 77, "gray", dict(quality=85, restart_marker_rows=2)))
    ramp = [1 + (i * 7) % 97 for i in range(64)]
    out.append(("qtables_420", 129, 67, "4:2:0", dict(qtables=[ramp, [2 + i for i in range(64)]])))
    out.append(("qtables_gray", 129, 67, "gray", dict(qtables=[[255 - i for i in range(64)]])))
    out.append(("optimize_restart_420", 129, 67, "4:2:0", dict(quality=60, optimize=True, restart_marker_rows=1)))
    out.append(("refused_cmyk", 33, 17, "cmyk", dict(quality=80)))
    out.append(("refused_progressive", 33, 17, "4:2:0", dict(quality=80, progressive=True)))
    return out


def main():
    manifest = []
    for k, (name, w, h, sub, kw) in enumerate(cases()):
        mode = {"gray": "L", "cmyk": "CMYK"}.get(sub, "RGB")
        im = picture(w, h, k, mode)
        if mode == "RGB":
            kw = dict(kw, subsampling=sub)
        b = io.BytesIO()
        im.save(b, "JPEG", **kw)
        with open(os.path.join(HERE, name + ".jpg"), "wb") as f:
            f.write(b.getvalue())
        manifest.append({"file": name + ".jpg", "w": w, "h": h, "sub": sub,
                         "refused": name.startswith("refused"),
                         "restart": any(k.startswith("restart") for k in kw)})
    with open(os.path.join(HERE, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=0)


if __name__ == "__main__":
    main()
