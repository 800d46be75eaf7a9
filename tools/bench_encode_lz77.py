"""Benchmark of the LZ77 mode of the PNG encode (encode_png_device / encode_labels_device with lz77=K) against the call without it
and against what a user does on the host: a pinned D2H copy, then a PIL and a cv2 PNG save at zlib level 6 per image on 16
threads.

Workloads (tests/lz77_sizes.py): E1-E4 of tests/pngenc_workloads.py, the label maps V1-V3 of tools/bench_label_encode.py and C2
(bench.py's 1920x1080 RGB images, whose default files are fpng files), the first --count images of each, on the device.  Arms:
lz77 = 8, 32 and 128; the call without lz77; the PIL and cv2 arms (PIL: palette / 1-bit files for label maps, none for 16-bit
RGBA; cv2: 8-bit gray ids for label maps).  Times are host wall times ending in a device synchronise (GPU arms) or in the last file
(host arms), medians over --rounds alternating rounds; bytes are the total file size.  The GPU arms report the kernel split from
the profile slots (0 filter pass, 11 match, 1 Huffman, 2 segment bits, 3 offsets, 6 pack, 7 Adler-32, 8 CRC).  One JSON line per
workload, with the card and its power limit."""
from __future__ import annotations

import argparse
import ctypes as C
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
import lz77_sizes as ls  # noqa: E402

SLOTS = {"filter": 0, "match": 11, "huffman": 1, "seg_bits": 2, "offsets": 3, "pack": 6, "adler": 7, "crc": 8}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="E1,E2,E3,E4,V1,V2,V3,C2")
    ap.add_argument("--count", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    import fpng_b200 as fp
    from fpng_b200._lib import lib
    fp.fpng_init(0)
    name_, power = card()
    info = {"card": name_, "power_limit": power}
    pool = ThreadPoolExecutor(16)
    for name in args.workloads.split(","):
        kind, host_imgs, depth, pal = ls.workload(name, args.count)
        imgs = [torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in host_imgs]
        arms = {f"lz77_{k}": k for k in ls.KS}
        arms["default"] = 0

        def gpu(k):
            if kind == "label":
                r = fp.encode_labels_device(imgs, palette=pal, depth=depth, lz77=k)
            else:
                r = fp.encode_png_device(imgs, lz77=k)
            torch.cuda.synchronize()
            return r

        def host(which):
            pinned = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in imgs]
            for p, t in zip(pinned, imgs):
                p.copy_(t, non_blocking=True)
            torch.cuda.synchronize()

            def save(a):
                a = a.numpy()
                if which == "pil":
                    return ls._pil(a, 6, "1" if kind == "label" and depth == 1 else None, pal if kind == "label" else None)
                return ls._cv2(a.astype(np.uint8) if kind == "label" else a, 6)
            sizes = list(pool.map(save, pinned))
            return None if None in sizes else sum(sizes)

        res = {"workload": name, "images": len(imgs), **info}
        for k in arms.values():
            gpu(k)
        times = {a: [] for a in list(arms) + ["pil_6", "cv2_6"]}
        host_bytes = {}
        for _ in range(args.rounds):
            for a, k in arms.items():
                t0 = time.perf_counter(); gpu(k); times[a].append(time.perf_counter() - t0)
            for which in ("pil", "cv2"):
                t0 = time.perf_counter(); host_bytes[which] = host(which); times[f"{which}_6"].append(time.perf_counter() - t0)
        for a, k in arms.items():
            out, offsets, sizes = gpu(k)
            lib().fpngb_profile_enable(1)
            gpu(k)
            ms = (C.c_float * 12)()
            lib().fpngb_profile_read(ms, 12)
            lib().fpngb_profile_enable(0)
            res[a] = {"ms": round(1e3 * statistics.median(times[a]), 3), "bytes": int(sizes.sum()),
                      "kernels_ms": {s: round(ms[i], 3) for s, i in SLOTS.items()}}
        for which in ("pil", "cv2"):
            res[f"{which}_6"] = {"ms": round(1e3 * statistics.median(times[f"{which}_6"]), 3), "bytes": host_bytes[which]}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
