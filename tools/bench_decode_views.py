"""Decode of packed files into many output images per call: fpngb_decode_packed_views_device against the torch chain a caller runs
without it.

V1 (eval): the 256 mixed M1 files of bench_ragged_decode.py to torchvision's Resize(256) + CenterCrop(224), bf16 NCHW with
    ImageNet scale and bias.  (b): decode_packed_ragged_device, ragged_views (a read-back), then per file torchvision's resize
    (antialias), center_crop and the affine map, cast into a preallocated batch.
V2 (ten-crop): 64 M1 files to 640 views of 224 x 224 uint8 (ten-crop of the shorter-side-256 resize).  (b): the ragged decode,
    ragged_views, then per file F.resize and F.ten_crop into the batch.
V3 (letterbox): bench.py's 256 x 1920x1080 RGB C2 files to 640 x 640 uint8 with fill 114 (letterbox_views).  (b): the ragged
    decode, ragged_views, then per file F.interpolate (bilinear, antialias) and a paste onto a 114 canvas.
Times are host wall time per call ending in a device synchronise, medians over alternating rounds; (a) is given every bound and
pixel_cap (no host synchronisation; its view table is built once).  The largest difference between (a) and (b) is reported on
the 0-255 scale.  Card name and power limit are read in the same run; one JSON line per configuration.

    python tools/bench_decode_views.py [--config v1 v2 v3] [--rounds 5] [--iters 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_decode_resized import c2_files, m1_files, packed  # noqa: E402
from bench_device_decode import card  # noqa: E402


def timed(arm_a, arm_b, rounds, iters):
    for fn in (arm_a, arm_b):
        fn()
    ta, tb = [], []
    for _ in range(rounds):
        for fn, acc in ((arm_a, ta), (arm_b, tb)):
            t0 = time.perf_counter()
            for _ in range(iters):
                fn()
            acc.append((time.perf_counter() - t0) * 1e3 / iters)
    return ta, tb


def run(name, files, rounds, iters):
    import torch
    import torch.nn.functional as Fn
    import torchvision.transforms.v2.functional as F

    import fpng_b200

    dev = torch.device("cuda", 0)
    data, offsets, sizes = packed(files, dev)
    info = fpng_b200.get_info_batch_device(data, offsets, sizes)
    dims = [(int(r[1]), int(r[2])) for r in info.cpu().numpy()]
    n, d = len(files), 3
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims),
                  pixel_cap=sum((w * h * d + 15) // 16 * 16 for w, h in dims))
    raw = torch.empty(bounds["pixel_cap"], dtype=torch.uint8, device=dev)
    rb = {k: v for k, v in bounds.items() if k != "pixel_cap"}
    if name == "V1":
        H = W = 224
        views = fpng_b200.resize_crop_views(info, 256, 224)
        s, b = fpng_b200.normalize_scale_bias((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
        st_, bt_ = torch.from_numpy(s).to(dev).view(3, 1, 1), torch.from_numpy(b).to(dev).view(3, 1, 1)
        out_a = torch.empty((n, d, H, W), dtype=torch.bfloat16, device=dev).permute(0, 2, 3, 1)
        out_b = torch.empty((n, d, H, W), dtype=torch.bfloat16, device=dev)
        kw = dict(dtype=torch.bfloat16, scale=s, bias=b)

        def per_file(i, v):
            x = F.center_crop(F.resize(v.permute(2, 0, 1).float(), 256, antialias=True), [224, 224])
            out_b[i] = (x * st_ + bt_).to(torch.bfloat16)

        def to_255(t_nchw):
            return (t_nchw.double() - bt_.double()) / st_.double()
        fill = None
    elif name == "V2":
        H = W = 224
        base = fpng_b200.resize_crop_views(info, 256, 224).cpu().numpy()
        rows = []
        for i in range(n):
            rh, rw, h, w = int(base[i, 5]), int(base[i, 6]), int(base[i, 3]), int(base[i, 4])
            c = (int(round((rh - 224) / 2)), int(round((rw - 224) / 2)))
            for flip in (0, fpng_b200.FPNGB_VIEW_HFLIP):
                rows += [(i, 0, 0, h, w, rh, rw, -t, -l, flip) for (t, l) in ((0, 0), (0, rw - 224), (rh - 224, 0), (rh - 224, rw - 224), c)]
        views = torch.tensor(rows, dtype=torch.int32, device=dev)
        out_a = torch.empty((10 * n, H, W, d), dtype=torch.uint8, device=dev)
        out_b = torch.empty((10 * n, d, H, W), dtype=torch.uint8, device=dev)
        kw = {}

        def per_file(i, v):
            x = F.resize(v.permute(2, 0, 1), 256, antialias=True)
            out_b[10 * i:10 * i + 10] = torch.stack(F.ten_crop(x, [224, 224]))

        def to_255(t_nchw):
            return t_nchw.double()
        fill = None
    else:
        H = W = 640
        views = fpng_b200.letterbox_views(info, (H, W))
        vt = views.cpu().numpy()
        out_a = torch.empty((n, H, W, d), dtype=torch.uint8, device=dev)
        out_b = torch.empty((n, d, H, W), dtype=torch.uint8, device=dev)
        kw = {}

        def per_file(i, v):
            rh, rw, oy, ox = (int(x) for x in vt[i, 5:9])
            x = Fn.interpolate(v.permute(2, 0, 1)[None].float(), size=(rh, rw), mode="bilinear", align_corners=False, antialias=True)
            out_b[i].fill_(114)
            out_b[i, :, oy:oy + rh, ox:ox + rw] = x[0].round().clamp(0, 255).to(torch.uint8)

        def to_255(t_nchw):
            return t_nchw.double()
        fill = 114

    def arm_a():
        fpng_b200.decode_packed_views_device(data, offsets, sizes, views, (H, W), d, fill=fill, out=out_a, **kw, **bounds)
        torch.cuda.synchronize()

    def arm_b():
        px, oo, inf, st = fpng_b200.decode_packed_ragged_device(data, offsets, sizes, d, out=raw, **rb)
        for i, v in enumerate(fpng_b200.ragged_views(px, oo, inf, st, d)):
            per_file(i, v)
        torch.cuda.synchronize()

    ta, tb = timed(arm_a, arm_b, rounds, iters)
    diff = float((to_255(out_a.permute(0, 3, 1, 2)) - to_255(out_b)).abs().max())
    gpu, power = card()
    return {"config": name, "files": n, "views": int(views.shape[0]), "canvas": [H, W], "dtype": str(out_a.dtype).replace("torch.", ""),
            "a_views_ms": statistics.median(ta), "a_min_max": [min(ta), max(ta)],
            "b_torch_chain_ms": statistics.median(tb), "b_min_max": [min(tb), max(tb)],
            "speedup_b_over_a": statistics.median(tb) / statistics.median(ta),
            "max_abs_diff_a_b_0_255": diff, "gpu": gpu, "power_limit": power}


def main():
    import torch

    import fpng_b200
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--config", nargs="+", default=["v1", "v2", "v3"], choices=["v1", "v2", "v3"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    fpng_b200.fpng_init(0)
    dev = torch.device("cuda", 0)
    m1 = None
    for cfg in a.config:
        if cfg in ("v1", "v2") and m1 is None:
            m1 = m1_files(dev)
        files = m1 if cfg == "v1" else m1[:64] if cfg == "v2" else c2_files(dev)
        print(json.dumps(run(cfg.upper(), files, a.rounds, a.iters)), flush=True)


if __name__ == "__main__":
    main()
