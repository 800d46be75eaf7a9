"""Label maps into a fixed-size batch: the index + nearest resized decode (one call) against today's GPU route.

L1: 256 VOC-like palette masks of about 500x375 (21 blob-shaped classes and the 255 border id, VOC's colour map), each cropped to
a random-resized-crop box and resized nearest to 512x512 uint8 ids.  L2: 64 16-bit gray 2048x1024 instance maps (Cityscapes-style
ids class * 1000 + instance), whole images nearest to 1024x512 uint16.  Files are generated from a seed by tests/pngwrite_formats.
Two arms, timed alternately (host wall time per call ending in a device synchronise, median over rounds):
  (a) decode_packed_resized_device(indices=True, interpolation="nearest") with every bound and pixel_cap given;
  (b) the GPU route without it: the all_formats (L1, RGB) or native (L2, uint16) ragged decode, ragged_views (a read-back), then
      per file in torch a crop, a palette-colour -> id lookup (L1) and F.interpolate(mode="nearest") into a preallocated batch
      (L2 through float32, which holds every 16-bit id exactly, as torch's CUDA nearest kernel has no uint16).
Also reported: the nearest kernel's time (profile slot 8 of fpngb_decode_profile_read) and its bytes (gathered source elements plus
written output) as a share of 3.35 TB/s; the device time of png_unfilter_ext_kernel and decode_nearest_kernel per call from
torch.profiler in a separate pass; whether the two arms' outputs are byte-identical; the card name and power limit, read in the
same run.  One JSON line per workload.

    python tools/bench_decode_labels.py [--workload l1 l2] [--rounds 7] [--iters 3]
"""
from __future__ import annotations

import argparse
import ctypes as C
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

from bench_decode_resized import packed  # noqa: E402
from bench_device_decode import card  # noqa: E402

HBM = 3.35e12


def voc_palette():
    """PASCAL VOC's colour map: bits of the index spread over the high bits of R, G and B"""
    pal = np.zeros((256, 3), np.uint8)
    for i in range(256):
        c, r, g, b = i, 0, 0, 0
        for j in range(8):
            r |= ((c >> 0) & 1) << (7 - j)
            g |= ((c >> 1) & 1) << (7 - j)
            b |= ((c >> 2) & 1) << (7 - j)
            c >>= 3
        pal[i] = (r, g, b)
    return pal


def blobs(rs, h, w, ids, n_blobs, border=None):
    """[h, w] labels: background 0 and n_blobs filled ellipses of ids drawn from `ids`, outlined with `border` when given"""
    y, x = np.mgrid[0:h, 0:w]
    lab = np.zeros((h, w), np.uint32)
    for _ in range(n_blobs):
        cy, cx = rs.randint(0, h), rs.randint(0, w)
        ry, rx = rs.randint(h // 16 + 1, h // 3 + 2), rs.randint(w // 16 + 1, w // 3 + 2)
        d = ((y - cy) / ry) ** 2 + ((x - cx) / rx) ** 2
        lab[d <= 1] = ids[rs.randint(len(ids))]
        if border is not None:
            lab[(d > 1) & (d <= 1.15)] = border
    return lab


def l1_files(rs):
    import pngwrite_formats as pf
    pal = voc_palette()
    files, labels = [], []
    for k in range(256):
        h, w = int(rs.randint(330, 420)), int(rs.randint(450, 501))
        lab = blobs(rs, h, w, np.arange(1, 21), int(rs.randint(1, 5)), 255)
        files.append(pf.make_png(lab[..., None], 3, 8, plte=pal, filters=0, seed=k))
        labels.append(lab)
    return files, labels, pal


def l2_files(rs):
    import pngwrite_formats as pf
    files = []
    for k in range(64):
        ids = np.concatenate([np.arange(7, 24), 1000 * rs.randint(24, 34, 40) + rs.randint(0, 60, 40)])
        lab = blobs(rs, 1024, 2048, ids, 12)
        files.append(pf.make_png(lab[..., None], 0, 16, filters=2, seed=k))
    return files


def random_resized_crop(rs, w, h):
    """torchvision's RandomResizedCrop box (scale 0.08..1, ratio 3/4..4/3, 10 tries, then the whole image)"""
    for _ in range(10):
        area = w * h * rs.uniform(0.08, 1.0)
        ratio = np.exp(rs.uniform(np.log(3 / 4), np.log(4 / 3)))
        bw, bh = int(round(np.sqrt(area * ratio))), int(round(np.sqrt(area / ratio)))
        if 0 < bw <= w and 0 < bh <= h:
            return int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1)), bh, bw
    return 0, 0, h, w


def kernel_times(fn, iters):
    """device ms per call of the two kernels, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
    out = {"png_unfilter_ext_kernel": 0.0, "decode_nearest_kernel": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        for k in out:
            if k in e.key:
                out[k] += t / 1e3 / iters
    torch.cuda.synchronize()
    return out


def run(name, files, size, dtype, boxes_np, lut, rounds, iters):
    import torch
    import torch.nn.functional as F

    import fpng_b200
    from fpng_b200._lib import lib

    dev = torch.device("cuda", 0)
    data, offsets, sizes = packed(files, dev)
    n, (H, W) = len(files), size
    infos = [fpng_b200.get_png_info(f, all_formats=True) for f in files]
    dims = [(i[1], i[2]) for i in infos]
    es = dtype.itemsize
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims))
    cap = sum((w * h * es + 15) // 16 * 16 for w, h in dims)
    boxes = None if boxes_np is None else torch.from_numpy(boxes_np).to(dev)
    full = dict(any_png=True, all_formats=True, native=True)
    out_a = torch.empty((n, H, W, 1), dtype=dtype, device=dev)
    out_b = torch.empty((n, H, W, 1), dtype=dtype, device=dev)
    if lut is not None:                                   # L1: RGB decode, colour -> id through a dense 2^24 table on the device
        d_b, raw = 3, torch.empty(sum((w * h * 3 + 15) // 16 * 16 for w, h in dims), dtype=torch.uint8, device=dev)
        table = torch.zeros(1 << 24, dtype=torch.uint8, device=dev)
        key = torch.from_numpy((lut[:, 0].astype(np.int64) << 16) | (lut[:, 1].astype(np.int64) << 8) | lut[:, 2]).to(dev)
        table[key] = torch.arange(256, dtype=torch.int64, device=dev).to(torch.uint8)
    else:
        d_b, raw = 1, torch.empty(cap // es, dtype=dtype, device=dev)

    def arm_a():
        fpng_b200.decode_packed_resized_device(data, offsets, sizes, size, 1, boxes=boxes, out=out_a, pixel_cap=cap,
                                               interpolation="nearest", indices=True, **full, **bounds)
        torch.cuda.synchronize()

    def arm_b():
        if lut is not None:
            px, oo, inf, st = fpng_b200.decode_packed_ragged_device(data, offsets, sizes, 3, out=raw, any_png=True, all_formats=True,
                                                                    **bounds)
        else:
            px, oo, inf, st = fpng_b200.decode_packed_ragged_device(data, offsets, sizes, 1, out=raw, dtype=dtype, **full, **bounds)
        views = fpng_b200.ragged_views(px, oo, inf, st, d_b)
        for i, v in enumerate(views):
            t, l, bh, bw = (0, 0, v.shape[0], v.shape[1]) if boxes_np is None else (int(x) for x in boxes_np[i])
            c = v[t:t + bh, l:l + bw]
            if lut is not None:
                c = c.to(torch.int32)
                ids = table[(c[..., 0] << 16) | (c[..., 1] << 8) | c[..., 2]]
                out_b[i, ..., 0] = F.interpolate(ids[None, None], size=size, mode="nearest")[0, 0]
            else:
                out_b[i, ..., 0] = F.interpolate(c[..., 0].float()[None, None], size=size, mode="nearest")[0, 0].to(dtype)
        torch.cuda.synchronize()

    for fn in (arm_a, arm_b):
        fn()
    ta, tb = [], []
    for _ in range(rounds):
        for fn, acc in ((arm_a, ta), (arm_b, tb)):
            t0 = time.perf_counter()
            for _ in range(iters):
                fn()
            acc.append((time.perf_counter() - t0) * 1e3 / iters)
    identical = bool(torch.equal(out_a.view(torch.uint8) if es == 1 else out_a.view(torch.int16),
                                 out_b.view(torch.uint8) if es == 1 else out_b.view(torch.int16)))
    L = lib()
    L.fpngb_decode_profile_enable(1)
    ks = []
    ms = (C.c_float * 9)()
    for _ in range(iters):
        arm_a()
        assert L.fpngb_decode_profile_read(ms, 9) == 1
        ks.append(ms[8])
    L.fpngb_decode_profile_enable(0)
    k_ms = statistics.median(ks)
    kt = kernel_times(arm_a, iters)
    nbytes = 2 * n * H * W * es                           # one gathered source element and one stored element per output pixel
    gpu, power = card()
    return {"workload": name, "files": n, "size": [H, W], "dtype": str(dtype).replace("torch.", ""),
            "boxes": "random resized crop" if boxes_np is not None else "whole image",
            "a_index_nearest_ms": statistics.median(ta), "a_min_max": [min(ta), max(ta)],
            "b_ragged_torch_ms": statistics.median(tb), "b_min_max": [min(tb), max(tb)],
            "speedup_b_over_a": statistics.median(tb) / statistics.median(ta),
            "nearest_kernel_slot8_ms": k_ms, "nearest_kernel_bytes": nbytes,
            "nearest_kernel_hbm_share": nbytes / (k_ms * 1e-3) / HBM if k_ms > 0 else None,
            "profiler_nearest_kernel_ms": kt["decode_nearest_kernel"], "profiler_unfilter_ext_kernel_ms": kt["png_unfilter_ext_kernel"],
            "outputs_byte_identical": identical, "gpu": gpu, "power_limit": power}


def main():
    import torch

    import fpng_b200
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["l1", "l2"], choices=["l1", "l2"])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    fpng_b200.fpng_init(0)
    for wl in a.workload:
        rs = np.random.RandomState(2024 if wl == "l1" else 2025)
        if wl == "l1":
            files, labels, pal = l1_files(rs)
            boxes = np.array([random_resized_crop(rs, lab.shape[1], lab.shape[0]) for lab in labels], np.int32)
            res = run("L1", files, (512, 512), torch.uint8, boxes, pal, a.rounds, a.iters)
        else:
            res = run("L2", l2_files(rs), (512, 1024), torch.uint16, None, None, a.rounds, a.iters)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
