"""Benchmark of encode_png_device (gray, gray+alpha and 16-bit PNGs on the GPU) against what a user does today: a pinned
device-to-host copy and cv2.imencode at IMWRITE_PNG_COMPRESSION=1 on every host thread.

Workloads (tests/pngenc_workloads.py, generated from seeds): E1 256 gray8 1024x1024 label masks, E2 256 gray16 640x480 depth
maps, E3 128 gray8 1920x1080 gradient+noise, E4 64 RGBA16 1920x1080.  Each arm's time is host wall time ending in a device
synchronise (GPU) or in the last file (CPU), over alternating rounds; medians are reported.  A separate torch.profiler run gives
the kernel split of the GPU arm.  Prints one JSON line per workload, with the card and its power limit; --out also writes the
rows to a JSON file."""
from __future__ import annotations

import argparse
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="E1,E2,E3,E4")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result rows to this JSON file")
    args = ap.parse_args()
    import cv2
    import torch

    import fpng_b200
    fpng_b200.fpng_init(0)
    name, power = card()
    threads = os.cpu_count() or 1
    pool = ThreadPoolExecutor(threads)
    results = []
    for wl in args.workloads.split(","):
        imgs = pw.workload(wl)
        dev = [torch.from_numpy(i).cuda() for i in imgs]
        pinned = [torch.empty(i.shape, dtype=t.dtype, pin_memory=True) for i, t in zip(imgs, dev)]
        mp = sum(i.shape[0] * i.shape[1] for i in imgs) / 1e6

        def gpu():
            r = fpng_b200.encode_png_device(dev)
            torch.cuda.synchronize()
            return r

        def cpu():
            for p, t in zip(pinned, dev):
                p.copy_(t, non_blocking=True)
            torch.cuda.synchronize()

            def one(p):
                a = p.numpy()
                a = a[..., 0] if a.shape[2] == 1 else a[..., [2, 1, 0, 3][:a.shape[2]]]
                return len(cv2.imencode(".png", a, [cv2.IMWRITE_PNG_COMPRESSION, 1])[1])
            return list(pool.map(one, pinned))

        gpu(); cpu()                                                   # warm-up: module loads, workspace growth, thread pool
        tg, tc = [], []
        for _ in range(args.rounds):
            t0 = time.perf_counter(); out, offsets, sizes = gpu(); tg.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); cv_sizes = cpu(); tc.append(time.perf_counter() - t0)
        gpu_bytes = int(sizes.long().sum().item())
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            gpu()
        split = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.key and "Memset" not in e.key:
                k = e.key.split("<")[0].split("(")[0].replace("void ", "").replace("fpngb::", "")
                split[k] = round(split.get(k, 0.0) + e.self_device_time_total / 1e3, 3)
        g, c = statistics.median(tg), statistics.median(tc)
        row = {"workload": wl, "images": len(imgs), "megapixels": round(mp, 2), "gpu_ms": round(1e3 * g, 2), "cv2_ms": round(1e3 * c, 2),
               "gpu_MPps": round(mp / g, 1), "cv2_MPps": round(mp / c, 1), "gpu_bytes": gpu_bytes, "cv2_bytes": int(sum(cv_sizes)),
               "kernel_ms": split, "cv2_threads": threads, "card": name, "power_limit": power}
        print(json.dumps(row), flush=True)
        results.append(row)
        del dev, pinned
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
