"""Native-output any-PNG decode (native=True, FPNGB_PNG_NATIVE / FPNGB_RESIZE_NATIVE) against the routes users take without it.

Workloads:
  N1  256 cv2.imencode 16-bit gray 640 x 480 depth maps (pngenc_workloads.depth_map) decoded to [h, w, 1] uint16.  Arms: native
      uint16 at 1 channel; today's route (float32 RGB decode, x 257, round, channel 0 sliced out, to int32); cv2.imdecode
      (IMREAD_UNCHANGED) over 16 threads plus pinned uploads.
  N2  1024 gray8 512 x 512 label masks (pngenc_workloads.label_mask, written by encode_png_device) decoded to [h, w, 1] uint8.
      Arms: native desired 1; desired 3 plus a slice of channel 0.
  N3  N1 resized to 256 x 256 float32 (antialiased).  Arms: the native resize (16-bit samples) and today's resize (high bytes).  Also
      the largest error of each, in 16-bit units, against a float64 model of the resample on 8 of the files.
Output bytes per pixel of each arm's result are reported as arithmetic.  Times are host wall time ending in a device synchronise,
median of alternating rounds, files already in device memory (the cv2 arm starts from host bytes).  Card name and power limit are read
in the same run; one JSON line per workload.

    python tools/bench_png_native.py [--workload N1 N2 N3] [--rounds 5]
"""
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

HOST_THREADS = 16


def depth_files():
    import cv2
    import pngenc_workloads as pw
    imgs = [pw.depth_map(480, 640, 5000 + k) for k in range(256)]
    files = []
    for im in imgs:
        ok, enc = cv2.imencode(".png", im[..., 0] if im.ndim == 3 else im)
        assert ok
        files.append(enc.tobytes())
    return files, [im.reshape(480, 640) for im in imgs]


def mask_files(dev):
    import torch
    import fpng_b200
    import pngenc_workloads as pw
    imgs = [pw.label_mask(512, 512, 7000 + k) for k in range(1024)]
    imgs = [im if im.ndim == 3 else im[..., None] for im in imgs]
    data, offsets, sizes = fpng_b200.encode_png_device([torch.from_numpy(np.ascontiguousarray(i)).to(dev) for i in imgs])
    o, z, d = offsets.cpu().numpy(), sizes.cpu().numpy(), data.cpu().numpy()
    return [d[o[k]:o[k] + z[k]].tobytes() for k in range(len(imgs))], imgs


def packed(files, dev):
    import torch
    offs, at = [], 0
    for f in files:
        offs.append(at)
        at = (at + len(f) + 15) // 16 * 16
    buf = np.zeros(at, np.uint8)
    for o, f in zip(offs, files):
        buf[o:o + len(f)] = np.frombuffer(f, np.uint8)
    sz = np.array([len(f) for f in files], np.uint32).view(np.int32)
    return (torch.from_numpy(buf).to(dev), torch.tensor(offs, dtype=torch.int64, device=dev), torch.from_numpy(sz).to(dev))


def timed(arms, rounds):
    import torch
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    return {k: round(statistics.median(v), 3) for k, v in times.items()}, {k: [round(x, 3) for x in v] for k, v in times.items()}


def run(workload, rounds):
    import cv2
    import torch
    import fpng_b200
    dev = torch.device("cuda")
    res = {"workload": workload}
    if workload in ("N1", "N3"):
        files, srcs = depth_files()
    else:
        files, srcs = mask_files(dev)
    pk = packed(files, dev)
    n, (h, w) = len(files), srcs[0].shape[:2]
    bounds = dict(max_file_size=max(map(len, files)), max_w=w, max_h=h)
    kw = dict(any_png=True, all_formats=True)
    if workload == "N1":
        u16 = torch.empty(n * h * w, dtype=torch.uint16, device=dev)
        f32 = torch.empty(n * h * w * 3, dtype=torch.float32, device=dev)
        pool = ThreadPoolExecutor(HOST_THREADS)

        def native():
            return fpng_b200.decode_packed_ragged_device(*pk, 0, out=u16, native=True, **kw, **bounds)

        def today():
            fpng_b200.decode_packed_ragged_device(*pk, 3, out=f32, **kw, **bounds)
            return (f32.view(n, h, w, 3)[..., :1] * 257.0).round().to(torch.int32)

        def host():
            px = list(pool.map(lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_UNCHANGED), files))
            return [torch.from_numpy(p.view(np.int16)).pin_memory().to(dev, non_blocking=True) for p in px]
        native()
        torch.cuda.synchronize()
        got = u16.view(torch.int16).cpu().numpy().view(np.uint16).reshape(n, h, w)
        assert all(np.array_equal(got[k], srcs[k]) for k in range(n))
        assert np.array_equal(today().cpu().numpy()[..., 0], got.astype(np.int32))
        arms = {"native": native, "today_float_x257": today, "cv2_pinned": host}
        res["out_bytes_per_px"] = {"native": 2, "today_float_x257": 12, "cv2_pinned": 2}
        res["host_threads"] = HOST_THREADS
    elif workload == "N2":
        u1 = torch.empty(n * h * w, dtype=torch.uint8, device=dev)
        u3 = torch.empty(n * h * w * 3, dtype=torch.uint8, device=dev)

        def native():
            return fpng_b200.decode_packed_ragged_device(*pk, 1, out=u1, native=True, **kw, **bounds)

        def today():
            fpng_b200.decode_packed_ragged_device(*pk, 3, out=u3, **kw, **bounds)
            return u3.view(n, h, w, 3)[..., :1].contiguous()
        native()
        torch.cuda.synchronize()
        assert torch.equal(u1.view(n, h, w, 1).cpu(), torch.from_numpy(np.stack(srcs)))
        assert torch.equal(today().cpu(), u1.view(n, h, w, 1).cpu())
        arms = {"native": native, "today_desired3_slice": today}
        res["out_bytes_per_px"] = {"native": 1, "today_desired3_slice": 3}
    else:
        from test_decode_resized_cpu import resize_model
        H = W = 256
        out_n = torch.empty(n, H, W, 1, dtype=torch.float32, device=dev)
        out_t = torch.empty(n, H, W, 3, dtype=torch.float32, device=dev)

        def native():
            return fpng_b200.decode_packed_resized_device(*pk, (H, W), 1, out=out_n, native=True, pixel_cap=n * h * w * 2, **kw,
                                                          **bounds)

        def today():
            return fpng_b200.decode_packed_resized_device(*pk, (H, W), 3, out=out_t, pixel_cap=n * h * w * 3, **kw, **bounds)
        native()
        today()
        torch.cuda.synchronize()
        err_n = err_t = 0.0
        for k in range(0, n, n // 8):
            r = resize_model(srcs[k][..., None].astype(np.float64), H, W, True)[..., 0]
            err_n = max(err_n, float(np.abs(out_n[k, ..., 0].double().cpu().numpy() * 257.0 - r).max()))
            err_t = max(err_t, float(np.abs(out_t[k, ..., 0].double().cpu().numpy() * 257.0 - r).max()))
        res["max_err_16bit_units"] = {"native": round(err_n, 3), "today_high_byte": round(err_t, 3)}
        arms = {"native": native, "today_high_byte": today}
    med, allv = timed(arms, rounds)
    gpu, power = card()
    res.update({"files": n, "file_mb": round(sum(map(len, files)) / 1e6, 1), "shape": [h, w], "rounds": rounds, "gpu": gpu,
                "power_limit": power})
    res.update({k + "_ms": v for k, v in med.items()})
    res.update({k + "_all_ms": v for k, v in allv.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", nargs="+", default=["N1", "N2", "N3"])
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import fpng_b200
    fpng_b200.fpng_init()
    for wl in a.workload:
        print(json.dumps(run(wl, a.rounds)), flush=True)


if __name__ == "__main__":
    main()
