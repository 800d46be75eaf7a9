"""Writes tests/golden/anypng/: PNGs of seeded imagegen images written by libpng (through OpenCV: every zlib strategy, levels 0, 1
and 9) and by PIL (L, LA, RGB, RGBA, optimize=True), and manifest.json, which names each file's source image, so that the GPU tests
regenerate the expected pixels without PIL or OpenCV.  Run from the repository root: python tests/golden/make_anypng.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import pngwrite  # noqa: E402

OUT = os.path.join(HERE, "anypng")


def main():
    import cv2
    from PIL import Image

    os.makedirs(OUT, exist_ok=True)
    manifest = []

    def add(name, data, kind, w, h, c, index, writer):
        with open(os.path.join(OUT, name), "wb") as f:
            f.write(data)
        manifest.append({"file": name, "kind": kind, "w": w, "h": h, "chans": c, "index": index, "writer": writer})

    strategies = {"default": cv2.IMWRITE_PNG_STRATEGY_DEFAULT, "filtered": cv2.IMWRITE_PNG_STRATEGY_FILTERED,
                  "huffman": cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY, "rle": cv2.IMWRITE_PNG_STRATEGY_RLE,
                  "fixed": cv2.IMWRITE_PNG_STRATEGY_FIXED}
    k = 0
    for sname, strat in strategies.items():
        for level in (0, 1, 9):
            for c in (1, 3, 4):
                kind = ("g1", "g0", "runs")[k % 3]
                w, h = 37 + 11 * (k % 5), 23 + 7 * (k % 4)
                img = pngwrite.source(kind, w, h, c, k)
                bgr = img[..., 0] if c == 1 else img[..., [2, 1, 0] + ([3] if c == 4 else [])]
                ok, buf = cv2.imencode(".png", bgr, [cv2.IMWRITE_PNG_COMPRESSION, level, cv2.IMWRITE_PNG_STRATEGY, strat])
                assert ok
                add(f"cv2_{sname}_l{level}_c{c}.png", buf.tobytes(), kind, w, h, c, k, f"opencv {cv2.__version__}")
                k += 1
    for mode, c in (("L", 1), ("LA", 2), ("RGB", 3), ("RGBA", 4)):
        for kind in ("g1", "g0"):
            w, h = 61 + 3 * k % 17, 29 + k % 13
            img = pngwrite.source(kind, w, h, c, k)
            import io
            b = io.BytesIO()
            Image.fromarray(img[..., 0] if c == 1 else img, mode).save(b, format="PNG", optimize=True)
            add(f"pil_{mode}_{kind}.png", b.getvalue(), kind, w, h, c, k, f"PIL {Image.__version__ if hasattr(Image, '__version__') else ''}")
            k += 1
    with open(os.path.join(OUT, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
