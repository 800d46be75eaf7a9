"""The size table of the LZ77 mode, computed on the CPU from the exact oracles (the GPU files equal them byte for byte): for the
first `count` images of each workload, the total file bytes of encode_png_device / encode_labels_device with lz77 = 8, 32 and
128, of the same call without lz77 (run-only PNG files; for C2, the fpng files the default call writes), and of PIL and cv2 at
zlib levels 6 and 1.  Workloads: E1-E4 (tests/pngenc_workloads.py), V1-V3 (tools/bench_label_encode.py) and C2 (bench.py's
1920x1080 RGB gradient-plus-noise images).  PIL writes V1 / V2 as palette files and V3 as a mode "1" file, and cannot write E4
(16-bit RGBA: None); cv2 writes label maps as 8-bit gray ids (it has no palette or 1-bit output)."""
from __future__ import annotations

import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "tools"))

KS = (8, 32, 128)


def _pil(img, level, mode=None, palette=None):
    from PIL import Image
    a = img[..., 0] if img.ndim == 3 and img.shape[2] == 1 else img
    if mode == "1":
        im = Image.fromarray(a.astype(bool))
    elif palette is not None:
        im = Image.fromarray(a.astype(np.uint8), "P")
        im.putpalette(np.asarray(palette, np.uint8)[:, :3].reshape(-1).tolist())
    elif a.dtype == np.uint16:
        if a.ndim != 2:
            return None
        im = Image.fromarray(a, "I;16")
    else:
        im = Image.fromarray(a)
    b = io.BytesIO()
    im.save(b, format="PNG", compress_level=level)
    return len(b.getvalue())


def _cv2(img, level):
    import cv2
    a = img
    if a.ndim == 3 and a.shape[2] >= 3:
        a = a[:, :, [2, 1, 0, 3][:a.shape[2]]]
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(a), [cv2.IMWRITE_PNG_COMPRESSION, level])
    assert ok
    return len(buf)


def workload(name, count):
    """(kind, images, depth, palette): kind "png" ([h, w, c] arrays), "label" ([h, w] ids) or "fpng" (C2)"""
    import pngenc_workloads as pw
    if name.startswith("E"):
        return "png", pw.workload(name, count), None, None
    if name == "C2":
        import imagegen
        out = []
        for i in range(count):
            base = imagegen.gradient(1920, 1080, 3, i).astype(np.int16)
            rs = np.random.RandomState(1234 + i % 16)
            out.append(((base + rs.randint(-3, 4, size=base.shape).astype(np.int16)) & 255).astype(np.uint8))
        return "fpng", out, None, None
    from bench_label_encode import workload as vw
    ids, _, depth, pal = vw(name) if name != "V1" else _v1(count)
    return "label", ids[:count], depth, pal


def _v1(count):
    from bench_label_encode import voc_like
    from label_encode_cases import voc_palette
    return [voc_like(375, 500, 1000 + k) for k in range(count)], "int64", 8, voc_palette()


def table(names=("E1", "E2", "E3", "E4", "V1", "V2", "V3", "C2"), count=2):
    """{workload: {arm: total bytes}}"""
    import lz77_oracle as lo
    from label_oracle import LabelOracle
    from oracle.pngenc_oracle import PngEncodeOracle
    from oracle.pyoracle import Oracle
    png, lab = PngEncodeOracle(), LabelOracle()
    res = {}
    for name in names:
        kind, imgs, depth, pal = workload(name, count)
        row = {f"lz77_{k}": 0 for k in KS}
        row.update(run_only=0, pil_6=0, pil_1=0, cv2_6=0, cv2_1=0)
        for img in imgs:
            for k in KS:
                row[f"lz77_{k}"] += len(lo.label_encode(img, depth, k, pal) if kind == "label" else lo.png_encode(img, k))
            if kind == "label":
                row["run_only"] += len(lab.label_encode(img, depth, pal))
            elif kind == "fpng":
                row["run_only"] += len(Oracle().encode(img, img.shape[1], img.shape[0], 3, 0))
            else:
                row["run_only"] += len(png.png_encode(img))
            for lvl in (6, 1):
                p = _pil(img, lvl, "1" if kind == "label" and depth == 1 else None, pal if kind == "label" else None)
                row[f"pil_{lvl}"] = None if p is None or row[f"pil_{lvl}"] is None else row[f"pil_{lvl}"] + p
                row[f"cv2_{lvl}"] += _cv2(img.astype(np.uint8) if kind == "label" else img, lvl)
        res[name] = row
    return res


if __name__ == "__main__":
    import json
    import time
    t = time.time()
    print(json.dumps(table(count=int(sys.argv[1]) if len(sys.argv) > 1 else 2)), time.time() - t)
