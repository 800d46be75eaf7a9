"""Benchmark of encode_labels_device (label maps to palette / low-bit gray PNGs on the GPU) against what a user does without it.

Workloads (seeded):
  V1  256 VOC-like 500x375 maps: 21 classes as blobs plus void 255 on the class boundaries, the 256-entry VOC palette, int64 ids
      on the device (argmax output);
  V2  E1's 256 1024x1024 8-label masks (tests/pngenc_workloads.py) as a 4-bit palette from uint8;
  V3  256 1024x1024 binary masks at 1 bit from uint8.
Arms: (a) encode_labels_device; (b) ids.to(uint8) + encode_png_device gray8 (INTEGRATION's earlier recipe: wraps ids >= 256 and
writes no palette); (c) a pinned D2H copy, then PIL palette / mode-1 saves on 16 threads.  Each arm's time is host wall time ending
in a device synchronise (GPU arms) or in the last file (PIL), over alternating rounds; medians are reported.  Also: the pre-pass
kernel's time (profile slot 9 of fpngb_profile_read) and its bytes (ids read plus packed rows written) against 3.35 TB/s, and the
kernel split of arm (a) from a separate torch.profiler run.  One JSON line per workload, with the card and its power limit."""
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
from label_encode_cases import voc_palette  # noqa: E402
import pngenc_workloads as pw  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def voc_like(h, w, seed):
    """21 classes as ellipses over background 0, with void 255 on every class boundary"""
    m = pw.label_mask(h, w, seed, labels=21, blobs=12)[..., 0].astype(np.int64)
    edge = np.zeros_like(m, bool)
    edge[1:, :] |= m[1:, :] != m[:-1, :]
    edge[:, 1:] |= m[:, 1:] != m[:, :-1]
    m[edge] = 255
    return m


def workload(name):
    """(ids list as numpy, torch dtype name, depth, palette)"""
    if name == "V1":
        return [voc_like(375, 500, 1000 + k) for k in range(256)], "int64", 8, voc_palette()
    if name == "V2":
        rng = np.random.default_rng(7)
        return [m[..., 0] for m in pw.workload("E1")], "uint8", 4, rng.integers(0, 256, (8, 3)).astype(np.uint8)
    if name == "V3":
        return [(pw.label_mask(1024, 1024, 2000 + k, labels=2)[..., 0] > 0).astype(np.uint8) for k in range(256)], "uint8", 1, None
    raise ValueError(name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="V1,V2,V3")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the result rows to this JSON file")
    args = ap.parse_args()
    import torch
    from PIL import Image

    import fpng_b200
    from fpng_b200._lib import lib
    fpng_b200.fpng_init(0)
    name, power = card()
    pool = ThreadPoolExecutor(args.threads)
    L = lib()
    results = []
    for wl in args.workloads.split(","):
        maps, dt, depth, pal = workload(wl)
        T = getattr(torch, dt)
        dev = [torch.from_numpy(m.astype(dt)).cuda() for m in maps]
        pinned = [torch.empty(m.shape, dtype=T, pin_memory=True) for m in maps]
        mp = sum(m.size for m in maps) / 1e6
        flat_pal = None if pal is None else pal.reshape(-1).tolist()

        def arm_a():
            r = fpng_b200.encode_labels_device(dev, palette=pal, depth=depth)
            torch.cuda.synchronize()
            return r

        def arm_b():
            r = fpng_b200.encode_png_device([t.to(torch.uint8)[..., None] for t in dev])
            torch.cuda.synchronize()
            return r

        def arm_c():
            for p, t in zip(pinned, dev):
                p.copy_(t, non_blocking=True)
            torch.cuda.synchronize()

            def one(p):
                a = p.numpy().astype(np.uint8)
                if pal is None:
                    im = Image.fromarray(a.astype(bool), mode="1") if depth == 1 else Image.fromarray(a, mode="L")
                else:
                    im = Image.fromarray(a, mode="P")
                    im.putpalette(flat_pal)
                b = io.BytesIO()
                im.save(b, format="PNG", bits=depth) if pal is not None else im.save(b, format="PNG")
                return b.tell()
            return list(pool.map(one, pinned))

        arm_a(); arm_b(); arm_c()                                      # warm-up: module loads, workspace growth, thread pool
        ta, tb, tc = [], [], []
        for _ in range(args.rounds):
            t0 = time.perf_counter(); out, offsets, sizes = arm_a(); ta.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); _, _, sizes_b = arm_b(); tb.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); pil_sizes = arm_c(); tc.append(time.perf_counter() - t0)
        assert int((sizes == 0).sum()) == 0
        L.fpngb_profile_enable(1)
        ms = (C.c_float * 10)()
        L.fpngb_profile_read(ms, 10)                                    # drop anything recorded before
        for _ in range(args.rounds):
            arm_a()
        assert L.fpngb_profile_read(ms, 10) >= 1
        L.fpngb_profile_enable(0)
        prepass_ms = float(ms[9])
        words = sum(((m.shape[1] * depth + 31) // 32) * m.shape[0] for m in maps)
        prepass_bytes = sum(m.size * T.itemsize for m in maps) + 4 * words
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            arm_a()
        split = {}
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.key and "Memset" not in e.key:
                k = e.key.split("<")[0].split("(")[0].replace("void ", "").replace("fpngb::", "")
                split[k] = round(split.get(k, 0.0) + e.self_device_time_total / 1e3, 3)
        a, b, c = statistics.median(ta), statistics.median(tb), statistics.median(tc)
        row = {"workload": wl, "images": len(maps), "megapixels": round(mp, 2), "ids": dt, "depth": depth,
               "palette": 0 if pal is None else len(pal),
               "a_labels_ms": round(1e3 * a, 2), "b_gray8_ms": round(1e3 * b, 2), "c_pil_ms": round(1e3 * c, 2),
               "a_bytes": int(sizes.long().sum().item()), "b_bytes": int(sizes_b.long().sum().item()), "c_bytes": int(sum(pil_sizes)),
               "prepass_ms": round(prepass_ms, 3), "prepass_bytes": prepass_bytes,
               "prepass_share_of_hbm": round(prepass_bytes / HBM_BYTES_PER_S / (prepass_ms / 1e3), 3) if prepass_ms > 0 else None,
               "kernel_ms": split, "pil_threads": args.threads, "card": name, "power_limit": power}
        print(json.dumps(row), flush=True)
        results.append(row)
        del dev, pinned
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
