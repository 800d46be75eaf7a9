"""Decode of packed files of mixed shapes into one fixed-size batch: fpngb_decode_packed_resized_device against the torch chain.

M1: the 256 mixed files of bench_ragged_decode.py; C2: bench.py's 256 x 1920x1080 RGB batch packed by dist.compact.  Output
224x224 NCHW with ImageNet scale and bias, in bf16 and f32, antialias on and off, boxes the whole image or the centre square.
Two arms, timed alternately:
  (a) decode_packed_resized_device with every bound and pixel_cap given (no host synchronisation);
  (b) what a caller does without it: the uint8 decode_packed_ragged_device, ragged_views (a read-back), then per file in torch a
      crop, F.interpolate(mode="bilinear", antialias=...), multiply, add and cast into a preallocated NCHW batch.
Times are host wall time per call ending in a device synchronise (median over alternating rounds).  The resize kernel's time is
profile slot 8 of fpngb_decode_profile_read; its bytes are the crop bytes it reads plus the output bytes it writes, reported as
a share of 3.35 TB/s.  The largest difference between (a) and (b) is reported on the 0-255 scale.  Card name and power limit
are read in the same run; one JSON line per configuration.

    python tools/bench_decode_resized.py [--workload m1 c2] [--rounds 5] [--iters 3]
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

from bench_device_decode import card  # noqa: E402
from bench_ragged_decode import M1_SHAPES  # noqa: E402

HBM = 3.35e12
SIZE = (224, 224)


def m1_files(dev):
    import bench
    import fpng_b200
    n, files = 256, []
    for k, (w, h, c) in enumerate(M1_SHAPES):
        idx = list(range(k, n, len(M1_SHAPES)))
        batch = bench.make_device_batch(dict(w=w, h=h, chans=c), "g1", len(idx), dev)
        enc, sizes = fpng_b200.encode_batch_device(batch, 0)
        enc, sizes = enc.cpu().numpy(), sizes.cpu().numpy()
        files += [(i, enc[t, :sizes[t]].tobytes()) for t, i in enumerate(idx)]
        del batch, enc
    files.sort()
    files = [f for _, f in files]
    order = np.random.RandomState(1234).permutation(n)
    return [files[i] for i in order]


def c2_files(dev):
    import bench
    import fpng_b200
    wl = bench.WORKLOADS["c2"]
    batch = bench.make_device_batch(wl, "g1", wl["images"], dev)
    enc, sizes = fpng_b200.encode_batch_device(batch, 0)
    enc, sizes = enc.cpu().numpy(), sizes.cpu().numpy()
    return [enc[i, :sizes[i]].tobytes() for i in range(len(sizes))]


def packed(files, dev):
    import torch
    n = len(files)
    offs = np.zeros(n + 1, np.int64)
    offs[1:] = np.cumsum([(len(f) + 15) // 16 * 16 for f in files])
    buf = np.zeros(int(offs[-1]), np.uint8)
    for i, f in enumerate(files):
        buf[offs[i]: offs[i] + len(f)] = np.frombuffer(f, np.uint8)
    return (torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev),
            torch.from_numpy(np.array([len(f) for f in files], np.uint32).view(np.int32)).to(dev))


def run(name, files, dtype, aa, centre, rounds, iters):
    import torch
    import torch.nn.functional as F

    import fpng_b200
    from fpng_b200._lib import lib

    dev = torch.device("cuda", 0)
    data, offsets, sizes = packed(files, dev)
    info = [fpng_b200.get_info_ex(f) for f in files]
    n, d = len(files), 3
    dims = [(i[1], i[2]) for i in info]
    boxes_np = np.array([((h - min(w, h)) // 2, (w - min(w, h)) // 2, min(w, h), min(w, h)) if centre else (0, 0, h, w)
                         for (w, h) in dims], np.int32)
    boxes = torch.from_numpy(boxes_np).to(dev)
    s, b = fpng_b200.normalize_scale_bias((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims))
    cap = sum((w * h * d + 15) // 16 * 16 for w, h in dims)
    out_a = torch.empty((n, d) + SIZE, dtype=dtype, device=dev).permute(0, 2, 3, 1)
    out_b = torch.empty((n, d) + SIZE, dtype=dtype, device=dev)
    raw = torch.empty(cap, dtype=torch.uint8, device=dev)
    st_, bt_ = torch.from_numpy(s).to(dev).view(1, 3, 1, 1), torch.from_numpy(b).to(dev).view(1, 3, 1, 1)

    def arm_a():
        fpng_b200.decode_packed_resized_device(data, offsets, sizes, SIZE, d, boxes=boxes, antialias=aa, out=out_a, scale=s, bias=b,
                                               pixel_cap=cap, **bounds)
        torch.cuda.synchronize()

    def arm_b():
        px, oo, inf, st = fpng_b200.decode_packed_ragged_device(data, offsets, sizes, d, out=raw, **bounds)
        views = fpng_b200.ragged_views(px, oo, inf, st, d)
        for i, v in enumerate(views):
            t, l, bh, bw = (int(x) for x in boxes_np[i])
            x = v[t:t + bh, l:l + bw].permute(2, 0, 1)[None].float()
            y = F.interpolate(x, size=SIZE, mode="bilinear", align_corners=False, antialias=aa)
            out_b[i] = (y * st_ + bt_)[0].to(dtype)
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
    crop_bytes = int(sum(int(bh) * int(bw) * d for _, _, bh, bw in boxes_np))
    out_bytes = n * SIZE[0] * SIZE[1] * d * out_a.element_size()
    # difference of the two arms on the 0-255 scale (undo the affine map in float64)
    sa = (out_a.permute(0, 3, 1, 2).double() - bt_.double()) / st_.double()
    sb = (out_b.double() - bt_.double()) / st_.double()
    diff = float((sa - sb).abs().max())
    gpu, power = card()
    return {"workload": name, "dtype": str(dtype).replace("torch.", ""), "antialias": aa, "boxes": "centre square" if centre else "whole image",
            "files": n, "size": list(SIZE), "layout": "NCHW",
            "a_resized_ms": statistics.median(ta), "a_min_max": [min(ta), max(ta)],
            "b_torch_chain_ms": statistics.median(tb), "b_min_max": [min(tb), max(tb)],
            "speedup_b_over_a": statistics.median(tb) / statistics.median(ta),
            "resize_kernel_ms": k_ms, "resize_kernel_bytes": crop_bytes + out_bytes,
            "resize_kernel_hbm_share": (crop_bytes + out_bytes) / (k_ms * 1e-3) / HBM if k_ms > 0 else None,
            "max_abs_diff_a_b_0_255": diff, "tolerance": 1e-3 if aa else 0.05, "gpu": gpu, "power_limit": power}


def main():
    import torch

    import fpng_b200
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["m1", "c2"], choices=["m1", "c2"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    fpng_b200.fpng_init(0)
    dev = torch.device("cuda", 0)
    for wl in a.workload:
        files = m1_files(dev) if wl == "m1" else c2_files(dev)
        configs = ([(dt, aa, centre) for dt in (torch.bfloat16, torch.float32) for aa in (True, False) for centre in (False, True)]
                   if wl == "m1" else [(torch.bfloat16, True, False), (torch.float32, False, True)])
        for dt, aa, centre in configs:
            print(json.dumps(run(wl.upper(), files, dt, aa, centre, a.rounds, a.iters)), flush=True)


if __name__ == "__main__":
    main()
