"""Decode of palette and 16-bit PNGs on the GPU (all_formats=True) against what users do today.

Workloads:
  F1  1024 PIL 8-bit palette ("P", 256 colors, fast-octree quantised imagegen images) PNGs of seeded sizes, sides 256-512, decoded to RGB uint8;
  F2  256 cv2.imwrite 16-bit gray 640 x 480 depth maps (smooth ramps with noise), decoded to float32 (one channel replicated to 3);
  P1  bench_png_decode.py's P1 (1024 PIL RGB PNGs) through any_png=True with all_formats on and off in alternating rounds: the cost of
      the flag when a batch has no file that needs it.
Arms (host wall time ending in a device synchronise, median of alternating rounds): the GPU decode with every bound given, files
already in device memory; cv2.imdecode(IMREAD_UNCHANGED) over a thread pool of all host cores, then pinned uploads into device
tensors (F2 converts to float32 on the device).  Also the kernel split of the GPU arm from a separate torch.profiler run.  Card name
and power limit are read in the same run; one JSON line per workload.

    python tools/bench_png_formats.py [--workload F1 F2 P1] [--rounds 5]
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
from bench_png_decode import images as p1_images, packed, pil_png  # noqa: E402

KERNELS = ("container_walk_kernel", "decode_place_kernel", "png_gather_kernel", "png_inflate_kernel", "png_unfilter_kernel",
           "png_unfilter_ext_kernel")


def corpus(workload):
    import cv2
    import imagegen
    from PIL import Image
    rs = np.random.RandomState(2025)
    if workload == "F1":
        dims = [(int(rs.randint(256, 513)), int(rs.randint(256, 513))) for _ in range(1024)]

        def one(k):
            w, h = dims[k]
            im = Image.fromarray(imagegen.make(("g1", "g0")[k % 2], w, h, 3, k), "RGB").quantize(256, method=Image.Quantize.FASTOCTREE)
            b = io.BytesIO()
            im.save(b, format="PNG")
            return b.getvalue()
        with ThreadPoolExecutor(os.cpu_count()) as ex:
            return list(ex.map(one, range(1024))), 3, None
    yy, xx = np.mgrid[0:480, 0:640]
    files = []
    for k in range(256):
        depth = (1000 + 20 * xx + 35 * yy + 500 * np.sin((xx + 7 * k) / 40.0) + rs.randint(0, 64, (480, 640))).astype(np.uint16)
        ok, enc = cv2.imencode(".png", depth)
        assert ok
        files.append(enc.tobytes())
    return files, 3, "float32"


def run(workload, rounds):
    import cv2
    import torch
    import fpng_b200
    dev = torch.device("cuda")
    if workload == "P1":
        files, d, dt = [pil_png(im) for im in p1_images("P1")], 3, None
    else:
        files, d, dt = corpus(workload)
    infos = [fpng_b200.get_png_info(f, all_formats=True) for f in files]
    assert all(i[0] == 0 for i in infos)
    mw, mh = max(i[1] for i in infos), max(i[2] for i in infos)
    T = getattr(torch, dt) if dt else torch.uint8
    es = torch.empty((), dtype=T).element_size()
    cap = sum((i[1] * i[2] * d * es + 15) // 16 * 16 for i in infos)
    out = torch.empty(cap // es, dtype=T, device=dev)
    pk = packed(files, dev)
    mfs = max(len(f) for f in files)

    def gpu_arm(all_formats):
        return lambda: fpng_b200.decode_packed_ragged_device(*pk, d, out=out, max_file_size=mfs, max_w=mw, max_h=mh, any_png=True,
                                                             all_formats=all_formats)
    pool = ThreadPoolExecutor(os.cpu_count())

    def host_arm():
        px = list(pool.map(lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_UNCHANGED), files))
        up = [torch.from_numpy(np.ascontiguousarray(p)).pin_memory().to(dev, non_blocking=True) for p in px]
        return [u.float() for u in up] if dt else up

    # correctness of the GPU arm on a sample: against cv2 (high byte / palette lookup, BGR -> RGB)
    _, oo, info, st = gpu_arm(True)()
    assert (st.cpu() == 0).all()
    views = fpng_b200.ragged_views(out, oo, info, st, d)
    for k in range(0, len(files), max(1, len(files) // 16)):
        ref = cv2.imdecode(np.frombuffer(files[k], np.uint8), cv2.IMREAD_UNCHANGED)
        if ref.dtype == np.uint16:
            want = np.repeat((ref.astype(np.float32) / np.float32(257.0))[..., None], 3, 2)
        else:
            want = ref[..., ::-1] if ref.ndim == 3 else np.repeat(ref[..., None], 3, 2)
        assert np.array_equal(views[k].cpu().numpy(), want[..., :3]), k
    arms = {"gpu_on": gpu_arm(True), "gpu_off": gpu_arm(False)} if workload == "P1" else {"gpu": gpu_arm(True), "host": host_arm}
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
    split = {}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gpu_arm(True)()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        for key in KERNELS:
            if key + "<" in e.key or e.key.split("(")[0].endswith(key) or ("::" + key) in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                split[key] = round(split.get(key, 0.0) + t / 1e3, 3)
    gpu, power = card()
    res = {"workload": workload, "files": len(files), "file_mb": round(sum(map(len, files)) / 1e6, 1), "desired": d,
           "dtype": dt or "uint8", "rounds": rounds, "kernel_ms": split, "gpu": gpu, "power_limit": power}
    for k, v in times.items():
        res[k + "_ms"] = round(statistics.median(v), 3)
        res[k + "_all_ms"] = [round(x, 3) for x in v]
    if "host" in times:
        res["host_threads"] = os.cpu_count()
        res["gpu_over_host"] = round(res["gpu_ms"] / res["host_ms"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["F1", "F2", "P1"])
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import fpng_b200
    fpng_b200.fpng_init()
    for w in a.workload:
        print(json.dumps(run(w, a.rounds)), flush=True)


if __name__ == "__main__":
    main()
