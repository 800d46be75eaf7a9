"""Decode of general PNG files (any writer) on the GPU against what users do today.

Workloads:
  P1  1024 PIL-written RGB PNGs (compress level 6, PIL's default) of seeded sizes, sides 256-512, imagegen g1 and g0 alternating;
  P2  64 PIL-written 1920 x 1080 RGB PNGs (g1 and g0): few large files.
Arms (host wall time ending in a device synchronise, median of alternating rounds):
  a  decode_packed_ragged_device(any_png=True) with all bounds given, files already in device memory;
  b  cv2.imdecode over a thread pool of all host cores, then pinned uploads into device tensors (PIL when OpenCV is missing;
     the line says which);
  c  the same images fpng-encoded, through the existing ragged decode (the fast path, for scale);
  d  the fpng batch of (c) through any_png=True against any_png=False (the cost of the opt-in when nobody needs it).
Also the split of walk, gather, inflate and unfilter kernels from a separate torch.profiler run, and arm (a) with the decode
verify switch on.  Card name and power limit are read in the same run; one JSON line per workload.

    python tools/bench_png_decode.py [--workload P1 P2] [--rounds 5]
"""
from __future__ import annotations

import argparse
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


def images(workload):
    import imagegen
    rs = np.random.RandomState(2024)
    if workload == "P1":
        dims = [(int(rs.randint(256, 513)), int(rs.randint(256, 513))) for _ in range(1024)]
    else:
        dims = [(1920, 1080)] * 64
    return [imagegen.make(("g1", "g0")[k % 2], w, h, 3, k) for k, (w, h) in enumerate(dims)]


def pil_png(img):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img, "RGB").save(b, format="PNG", compress_level=6)
    return b.getvalue()


def host_decoder():
    try:
        import cv2
        return f"opencv {cv2.__version__}", lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)
    except ImportError:
        from PIL import Image
        return "PIL", lambda b: np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))


def packed(files, dev):
    import torch
    offs, at = [], 0
    for f in files:
        at = (at + 15) // 16 * 16
        offs.append(at)
        at += len(f)
    buf = np.zeros(at, np.uint8)
    for o, f in zip(offs, files):
        buf[o:o + len(f)] = np.frombuffer(f, np.uint8)
    sizes = torch.tensor(np.array([len(f) for f in files], np.uint32).view(np.int32), device=dev)
    return torch.from_numpy(buf).to(dev), torch.tensor(offs, dtype=torch.int64, device=dev), sizes


def run(workload, rounds):
    import torch
    import fpng_b200
    dev = torch.device("cuda")
    imgs = images(workload)
    pngs = [pil_png(im) for im in imgs]
    fpngs = [fpng_b200.fpng_encode_image_to_memory(im, im.shape[1], im.shape[0], 3)[1] for im in imgs]
    raw_bytes = sum(im.size for im in imgs)
    mw, mh = max(im.shape[1] for im in imgs), max(im.shape[0] for im in imgs)
    cap = sum((im.size + 15) // 16 * 16 for im in imgs)
    out = torch.empty(cap, dtype=torch.uint8, device=dev)
    P, F = packed(pngs, dev), packed(fpngs, dev)

    def ragged(pk, files, any_png):
        return lambda: fpng_b200.decode_packed_ragged_device(*pk, 3, out=out, max_file_size=max(len(f) for f in files), max_w=mw,
                                                             max_h=mh, any_png=any_png)
    arm_a, arm_c = ragged(P, pngs, True), ragged(F, fpngs, False)
    arm_d = ragged(F, fpngs, True)
    name, dec = host_decoder()
    pool = ThreadPoolExecutor(os.cpu_count())

    def arm_b():
        px = list(pool.map(dec, pngs))
        pinned = [torch.from_numpy(p).pin_memory() for p in px]
        return [p.to(dev, non_blocking=True) for p in pinned]

    # correctness of the timed arms
    _, oo, info, st = arm_a()
    assert (st.cpu() == 0).all()
    views = fpng_b200.ragged_views(out, oo, info, st, 3)
    for k in range(0, len(imgs), max(1, len(imgs) // 16)):
        assert np.array_equal(views[k].cpu().numpy(), imgs[k])
    arms = {"a": arm_a, "b": arm_b, "c": arm_c, "d_any": arm_d, "d_off": arm_c}
    times = {k: [] for k in arms}
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    fpng_b200.set_decode_verify(True)
    tv = []
    arm_a()
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        arm_a()
        torch.cuda.synchronize()
        tv.append((time.perf_counter() - t0) * 1e3)
    fpng_b200.set_decode_verify(False)
    split = {}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm_a()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        for key in ("container_walk_kernel", "decode_place_kernel", "png_gather_kernel", "png_inflate_kernel", "png_unfilter_kernel"):
            if key in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                split[key] = round(split.get(key, 0.0) + t / 1e3, 3)
    gpu, power = card()
    med = {k: round(statistics.median(v), 3) for k, v in times.items()}
    return {"workload": workload, "files": len(imgs), "raw_mb": round(raw_bytes / 1e6, 1),
            "png_mb": round(sum(map(len, pngs)) / 1e6, 1), "compression_ratio": round(raw_bytes / sum(map(len, pngs)), 3),
            "a_any_png_ms": med["a"], "b_host_ms": med["b"], "b_decoder": name, "b_threads": os.cpu_count(),
            "c_fpng_ms": med["c"], "d_fpng_any_png_ms": med["d_any"], "d_fpng_off_ms": med["d_off"],
            "a_verify_ms": round(statistics.median(tv), 3), "a_over_b": round(med["a"] / med["b"], 3),
            "kernel_ms": split, "rounds": rounds, "gpu": gpu, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["P1", "P2"])
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import fpng_b200
    fpng_b200.fpng_init()
    for w in a.workload:
        print(json.dumps(run(w, a.rounds)), flush=True)


if __name__ == "__main__":
    main()
