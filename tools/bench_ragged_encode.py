"""Encode of device images of mixed shapes: fpngb_encode_ragged_device against one call per shape or per image.

M1, mixed: 256 bench.py-style g1 images cycling through 640x480 RGB, 1280x720 RGB, 1920x1080 RGB, 1920x1080 RGBA, 687x1012 RGB
and 3840x2160 RGB, one device tensor each.  Arms, timed alternately:
  (a) encode_ragged_device over the list (1-pass);
  (b) one encode_batch_device per shape on per-shape batches stacked outside the timed region (favours (b));
  (c) one encode_batch_device per image;
  (a) + compact_packed_device, with the compaction timed on its own.
M2, many small images: 4096 seeded images with sides drawn from 16-256, RGB and RGBA mixed; arms (a) and (c).  The
launch-bound case.
U, uniform: bench.py's C2 batch as a list of 256 views, encode_ragged_device against encode_batch_device.
Times are host wall time per call ending in a device synchronise, median over alternating rounds.  The files of all arms are
compared byte for byte.  Card name and power limit are read in the same run; one JSON line per workload.

    python tools/bench_ragged_encode.py [--workload m1 m2 u] [--rounds 5] [--iters 3]
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

from bench_device_decode import card  # noqa: E402

M1_SHAPES = [(640, 480, 3), (1280, 720, 3), (1920, 1080, 3), (1920, 1080, 4), (687, 1012, 3), (3840, 2160, 3)]


def timed(fn, iters):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def run_arms(arms, rounds, iters):
    for fn in list(arms.values()) * 2:                                   # warm-up: workspace, staging, first-launch costs
        fn()
    import torch
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(timed(fn, iters))
    return {k: stats(v) for k, v in ms.items()}


def ragged_files(res):
    out, offsets, sizes = res
    o = offsets.cpu().numpy()
    s = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return [(int(o[i]), int(s[i])) for i in range(len(s))], out


def equal_files(ragged_res, per_image):
    """per_image: list of (out 1-D uint8 tensor, size) per image"""
    import torch
    slots, out = ragged_files(ragged_res)
    ok = len(slots) == len(per_image)
    for (o, s), (f, fs) in zip(slots, per_image):
        ok &= s == fs and bool(torch.equal(out[o:o + s], f[:fs]))
    return ok


def uniform_files(out, sizes):
    s = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return [(out[i], int(s[i])) for i in range(len(s))]


def m1(rounds, iters):
    import torch

    import bench
    import fpng_b200

    dev = torch.device("cuda", 0)
    n = 256
    images = [None] * n
    for k, (w, h, c) in enumerate(M1_SHAPES):                           # image i has shape M1_SHAPES[i % 6]
        idx = list(range(k, n, len(M1_SHAPES)))
        batch = bench.make_device_batch(dict(w=w, h=h, chans=c), "g1", len(idx), dev)
        for t, i in enumerate(idx):
            images[i] = batch[t].clone()                                   # one tensor per image
        del batch
    groups = {}
    for i, im in enumerate(images):
        groups.setdefault(tuple(im.shape), []).append(i)
    stacked = {k: torch.stack([images[i] for i in idx]) for k, idx in groups.items()}   # (b): stacked outside the timed region
    shapes = [tuple(im.shape) for im in images]
    total = int(fpng_b200.ragged_slot_offsets(shapes)[-1])
    out_a = torch.empty(total, dtype=torch.uint8, device=dev)
    comp_out = torch.empty(total, dtype=torch.uint8, device=dev)
    res = {}

    def arm_a():
        res["a"] = fpng_b200.encode_ragged_device(images, 0, out=out_a)

    def arm_b():
        res["b"] = {k: fpng_b200.encode_batch_device(v, 0) for k, v in stacked.items()}

    def arm_c():
        res["c"] = [fpng_b200.encode_batch_device(im[None], 0) for im in images]

    def arm_compact():
        _, offsets, sizes = res["a"]
        res["compact"] = fpng_b200.compact_packed_device(out_a, offsets, sizes, out=comp_out)

    def arm_a_compact():
        arm_a()
        arm_compact()

    t = run_arms({"a": arm_a, "b": arm_b, "c": arm_c, "a_plus_compact": arm_a_compact, "compact_alone": arm_compact}, rounds, iters)
    per_b = [None] * n
    for k, (o, s) in res["b"].items():
        for t_, (f, fs) in enumerate(uniform_files(o, s)):
            per_b[groups[k][t_]] = (f, fs)
    per_c = [uniform_files(o, s)[0] for o, s in res["c"]]
    equal = equal_files(res["a"], per_b) and equal_files(res["a"], per_c)
    # the compacted buffer holds the same files back to back
    _, offsets, sizes = res["a"]
    co = res["compact"][1].cpu().numpy()
    slots, _ = ragged_files(res["a"])
    for i, (o, s) in enumerate(slots):
        equal &= bool(torch.equal(comp_out[int(co[i]):int(co[i]) + s], out_a[o:o + s]))
    return {"workload": "M1 256 mixed g1 1-pass, one tensor each: " + ", ".join(f"{w}x{h}x{c}" for w, h, c in M1_SHAPES),
            "slot_bytes": total, "compact_bytes": int(co[-1]),
            "a_ragged_ms": t["a"], "b_per_shape_ms": t["b"], "c_per_image_ms": t["c"],
            "a_plus_compact_ms": t["a_plus_compact"], "compact_alone_ms": t["compact_alone"], "outputs_equal": equal}


def m2(rounds, iters):
    import torch

    import fpng_b200
    import imagegen

    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(4096)
    n = 4096
    images = []
    for i in range(n):
        w, h, c = int(rs.randint(16, 257)), int(rs.randint(16, 257)), int(rs.choice([3, 4]))
        images.append(torch.from_numpy(imagegen.make("g1", w, h, c, i).reshape(h, w, c)).to(dev))
    total = int(fpng_b200.ragged_slot_offsets([tuple(im.shape) for im in images])[-1])
    out_a = torch.empty(total, dtype=torch.uint8, device=dev)
    res = {}

    def arm_a():
        res["a"] = fpng_b200.encode_ragged_device(images, 0, out=out_a)

    def arm_c():
        res["c"] = [fpng_b200.encode_batch_device(im[None], 0) for im in images]

    t = run_arms({"a": arm_a, "c": arm_c}, rounds, iters)
    equal = equal_files(res["a"], [uniform_files(o, s)[0] for o, s in res["c"]])
    return {"workload": "M2 4096 seeded g1 images, sides 16-256, RGB and RGBA mixed, 1-pass", "slot_bytes": total,
            "a_ragged_ms": t["a"], "c_per_image_ms": t["c"], "outputs_equal": equal}


def uniform(rounds, iters):
    import torch

    import bench
    import fpng_b200

    wl = bench.WORKLOADS["c2"]
    w, h, c, n = wl["w"], wl["h"], wl["chans"], wl["images"]
    dev = torch.device("cuda", 0)
    batch = bench.make_device_batch(wl, "g1", n, dev)
    views = list(batch.unbind(0))
    total = int(fpng_b200.ragged_slot_offsets([(h, w, c)] * n)[-1])
    out_r = torch.empty(total, dtype=torch.uint8, device=dev)
    stride = (fpng_b200.max_encoded_size(w, h, c) + 15) // 16 * 16
    out_u = torch.empty((n, stride), dtype=torch.uint8, device=dev)
    sizes_u = torch.empty((n,), dtype=torch.int32, device=dev)
    res = {}

    def arm_uniform():
        res["u"] = fpng_b200.encode_batch_device(batch, 0, out=out_u, sizes=sizes_u)

    def arm_ragged():
        res["r"] = fpng_b200.encode_ragged_device(views, 0, out=out_r)

    t = run_arms({"uniform": arm_uniform, "ragged": arm_ragged}, rounds, iters)
    equal = equal_files(res["r"], uniform_files(*res["u"]))
    return {"workload": "U " + wl["name"] + " as a list of 256 views", "encode_batch_device_ms": t["uniform"],
            "ragged_ms": t["ragged"], "outputs_equal": equal}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["m1", "m2", "u"], choices=["m1", "m2", "u"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_encode: no CUDA device")
    import fpng_b200
    fpng_b200.fpng_init(0)
    fns = {"m1": m1, "m2": m2, "u": uniform}
    for k in args.workload:
        r = fns[k](args.rounds, args.iters)
        name, power = card()
        r.update({"card": name, "power_limit": power, "rounds": args.rounds, "iters_per_round": args.iters,
                  "timing": "host wall time per call ending in a device synchronise, median of alternating rounds"})
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
