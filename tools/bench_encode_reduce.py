"""Benchmark of encode_png_device(reduce=True) (colour-type reduction on the GPU) against the same call without reduce and against
what a user does without it: a D2H copy, np.unique per image and a PIL save in the reduced mode on 16 threads.

Workloads (seeded, on the device):
  S1  64 colour-coded segmentation masks, 1024x1024 RGB, 20 colours as blobs (tests/pngenc_workloads.py label_mask);
  S2  64 binary masks stored as RGB 0 / 255, 1024x1024;
  S3  64 grey scans stored as RGB, 1024x1024 (gradient plus noise, R = G = B);
  S4  64 opaque RGBA renders, 1024x1024 (C2-like content plus alpha 255);
  C2  256 1920x1080 RGB photos of bench.py's C2 (gradient plus noise): nothing reduces, the analysis cost shows.
Arms: (a) reduce=True; (b) the same call without reduce; (c) pinned D2H copy, then per image on 16 threads np.unique and a PIL save
in the mode the rule picks (P with a palette, 1/L, LA, RGB, RGBA).  Times are host wall times ending in a device synchronise (GPU
arms) or in the last file (PIL), over alternating rounds; medians are reported, with the analysis kernels' time (profile slot 10)
and the conversion's (slot 9).  One JSON line per workload, with the card and its power limit."""
from __future__ import annotations

import argparse
import ctypes as C
import io
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_device_decode import card  # noqa: E402
import pngenc_workloads as pw  # noqa: E402
from reduce_model import choose  # noqa: E402


def workload(name, device):
    """list of [h, w, c] uint8 CUDA tensors"""
    import torch
    import bench
    if name == "C2":
        b = bench.make_device_batch(bench.WORKLOADS["c2"], "g1", 256, device)
        return [b[i] for i in range(b.shape[0])]
    rng = np.random.default_rng(11)
    out = []
    for k in range(64):
        if name == "S1":
            cols = torch.from_numpy(rng.integers(0, 256, (20, 3), dtype=np.uint8)).to(device)
            m = torch.from_numpy(pw.label_mask(1024, 1024, 3000 + k, labels=20, blobs=12)[..., 0].astype(np.int64)).to(device)
            out.append(cols[m])
        elif name == "S2":
            m = torch.from_numpy((pw.label_mask(1024, 1024, 4000 + k, labels=2)[..., 0] > 0).astype(np.uint8) * 255).to(device)
            out.append(m[..., None].expand(-1, -1, 3).contiguous())
        elif name == "S3":
            g = bench.make_device_batch(dict(w=1024, h=1024, chans=3, images=1, flags=0), "g1", 1, device, k)[0]
            out.append(g[..., :1].expand(-1, -1, 3).contiguous())
        elif name == "S4":
            g = bench.make_device_batch(dict(w=1024, h=1024, chans=4, images=1, flags=0), "g1", 1, device, k)[0]
            g[..., 3] = 255
            out.append(g)
        else:
            raise ValueError(name)
    return out


def pil_save(a):
    """np.unique and a PIL save in the mode the reduction rule picks for a, an [h, w, c] uint8 array"""
    from PIL import Image
    c = a.shape[2]
    flat = a.reshape(-1, c)
    keys = flat[:, 0].astype(np.uint32) << 16 | flat[:, 1].astype(np.uint32) << 8 | flat[:, 2] if c >= 3 else flat[:, 0].astype(np.uint32)
    if c == 4:
        keys = keys.astype(np.uint64) << 8 | flat[:, 3]
    uniq, inv = np.unique(keys, return_inverse=True)
    fmt, bits, depth = choose(a) if len(uniq) <= 256 else (("rgba" if c == 4 and (a[..., 3] != 255).any() else "rgb"), 0, 8)
    b = io.BytesIO()
    if fmt == "palette":
        im = Image.fromarray(inv.reshape(a.shape[:2]).astype(np.uint8), mode="P")
        pal = np.zeros((len(uniq), 3), np.uint8)
        for j in range(3):
            pal[:, j] = (uniq >> (8 * (2 - j) + (8 if c == 4 else 0))) & 255 if c >= 3 else uniq
        im.putpalette(pal.reshape(-1).tolist())
        im.save(b, format="PNG", bits=depth)
    elif fmt == "gray":
        g = a[..., 0]
        im = Image.fromarray(g > 0, mode="1") if depth == 1 else Image.fromarray(g, mode="L")
        im.save(b, format="PNG")
    else:
        chans = {"ga": [0, c - 1], "rgb": [0, 1, 2], "rgba": [0, 1, 2, 3]}[fmt]
        Image.fromarray(np.ascontiguousarray(a[..., chans]), mode={"ga": "LA", "rgb": "RGB", "rgba": "RGBA"}[fmt]).save(b, format="PNG")
    return b.tell()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="S1,S2,S3,S4,C2")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--pil", type=int, default=1, help="0: skip the PIL arm")
    ap.add_argument("--out", default=None, help="also write the result rows to this JSON file")
    args = ap.parse_args()
    import torch

    import fpng_b200
    from fpng_b200._lib import lib
    fpng_b200.fpng_init(0)
    name, power = card()
    pool = ThreadPoolExecutor(args.threads)
    L = lib()
    L.fpngb_profile_enable.argtypes = [C.c_int]
    L.fpngb_profile_read.argtypes = [C.POINTER(C.c_float), C.c_int]
    results = []
    for wl in args.workloads.split(","):
        imgs = workload(wl, torch.device("cuda", 0))
        pinned = [torch.empty(t.shape, dtype=torch.uint8, pin_memory=True) for t in imgs]
        mp = sum(t.shape[0] * t.shape[1] for t in imgs) / 1e6

        def arm_a():
            r = fpng_b200.encode_png_device(imgs, reduce=True)
            torch.cuda.synchronize()
            return r

        def arm_b():
            r = fpng_b200.encode_png_device(imgs)
            torch.cuda.synchronize()
            return r

        def arm_c():
            for p, t in zip(pinned, imgs):
                p.copy_(t, non_blocking=True)
            torch.cuda.synchronize()
            return list(pool.map(lambda p: pil_save(p.numpy()), pinned))

        arm_a(); arm_b()
        if args.pil:
            arm_c()
        ta, tb, tc, pil_sizes = [], [], [], []
        for _ in range(args.rounds):
            t0 = time.perf_counter(); _, _, sizes_a = arm_a(); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); _, _, sizes_b = arm_b(); tb.append(time.perf_counter() - t0)
            if args.pil:
                t0 = time.perf_counter(); pil_sizes = arm_c(); tc.append(time.perf_counter() - t0)
        L.fpngb_profile_enable(1)
        ms = (C.c_float * 11)()
        L.fpngb_profile_read(ms, 11)
        for _ in range(args.rounds):
            arm_a()
        assert L.fpngb_profile_read(ms, 11) >= 1
        L.fpngb_profile_enable(0)
        a, b = statistics.median(ta), statistics.median(tb)
        row = {"workload": wl, "images": len(imgs), "megapixels": round(mp, 2), "format": "/".join(map(str, choose(pinned[0].numpy())[::2])),
               "a_reduce_ms": round(1e3 * a, 2), "b_plain_ms": round(1e3 * b, 2),
               "c_pil_ms": round(1e3 * statistics.median(tc), 2) if tc else None,
               "a_bytes": int(sizes_a.long().sum().item()), "b_bytes": int(sizes_b.long().sum().item()),
               "c_bytes": int(sum(pil_sizes)) if pil_sizes else None,
               "analysis_ms": round(float(ms[10]), 3), "conversion_ms": round(float(ms[9]), 3),
               "pil_threads": args.threads, "card": name, "power_limit": power}
        print(json.dumps(row), flush=True)
        results.append(row)
        del imgs, pinned
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
