"""Decode of files that are already in device memory: what a caller had to do before fpngb_decode_packed_device, against it.

The files are bench.py's synthetic batch (same generator), encoded with encode_batch_device and packed with dist.compact, so
they sit on the GPU as one flat buffer with int64 offsets and int32 sizes.  Two arms, timed alternately in the same process:
  (a) host walk: copy the packed files to (pinned) host memory, container-walk every file on the host (get_info_ex), lay
      them out at a fixed stride, upload, decode_batch_device -- what the strided call needs;
  (b) decode_packed_device on the packed buffer (container walk on the device, no host synchronisation).
Each arm's time is host wall time from the start of its work to a device synchronise after it (arm (a) needs the host
anyway).  Also reported: the device time of the walk kernel alone (get_info_batch_device, CUDA events), the same with a 1 MiB
ancillary chunk in every file (its CRC runs serially on one thread per file), and whether (a) and (b) give identical pixels.
Prints one JSON line per workload; card name and power limit are read in the same run.

    python tools/bench_device_decode.py [--workload c2 c3] [--rounds 5] [--iters 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return name, power
    except Exception as e:                                            # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(), f"unknown ({e.__class__.__name__})"


def with_ancillary(f: bytes, nbytes: int) -> bytes:
    body = bytes(nbytes)
    ch = len(body).to_bytes(4, "big") + b"tEXt" + body + (zlib.crc32(b"tEXt" + body) & 0xFFFFFFFF).to_bytes(4, "big")
    return f[:33] + ch + f[33:]


def run(wl_key: str, rounds: int, iters: int) -> dict:
    import torch

    import bench
    import fpng_b200
    from fpng_b200 import dist

    wl = bench.WORKLOADS[wl_key]
    w, h, c, n, flags = wl["w"], wl["h"], wl["chans"], wl["images"], wl["flags"]
    dev = torch.device("cuda", 0)
    batch = bench.make_device_batch(wl, "g1", n, dev)
    enc, sizes = fpng_b200.encode_batch_device(batch, flags)
    flat, offsets = dist.compact(enc, sizes)
    del enc
    torch.cuda.synchronize()
    file_bytes = int(offsets[-1].item())

    # ---- arm (a): D2H, host walk, strided upload, decode_batch_device
    h_flat = torch.empty(file_bytes, dtype=torch.uint8, pin_memory=True)
    h_offs = torch.empty(n + 1, dtype=torch.int64, pin_memory=True)
    h_sizes = torch.empty(n, dtype=torch.int32, pin_memory=True)
    stride = (int(sizes.max().item()) + 16 + 15) // 16 * 16                # the tightest stride (the caller learns it from the sizes)
    h_strided = torch.zeros((n, stride), dtype=torch.uint8, pin_memory=True)
    d_strided = torch.empty((n, stride), dtype=torch.uint8, device=dev)
    px_a = torch.empty((n, h, w, c), dtype=torch.uint8, device=dev)
    st_a = torch.empty((n,), dtype=torch.int32, device=dev)

    def arm_a():
        h_flat.copy_(flat[:file_bytes], non_blocking=True); h_offs.copy_(offsets, non_blocking=True); h_sizes.copy_(sizes, non_blocking=True)
        torch.cuda.synchronize()
        buf, ofs, sz = h_flat.numpy(), h_offs.numpy(), h_sizes.numpy().view(np.uint32)
        hs = h_strided.numpy()
        io = np.empty(n, np.uint32); il = np.empty(n, np.uint32)
        for i in range(n):
            f = buf[ofs[i]: ofs[i] + sz[i]]
            st, ww, hh, cc, io[i], il[i] = fpng_b200.get_info_ex(f)
            if st or (ww, hh, cc) != (w, h, c):
                raise RuntimeError(f"file {i}: status {st}")
            hs[i, : sz[i]] = f
        d_strided.copy_(h_strided, non_blocking=True)
        fpng_b200.decode_batch_device(d_strided, sz, io, il, w, h, c, c, out=px_a, status=st_a)
        torch.cuda.synchronize()

    # ---- arm (b): decode_packed_device
    px_b = torch.empty((n, h, w, c), dtype=torch.uint8, device=dev)
    st_b = torch.empty((n,), dtype=torch.int32, device=dev)

    def arm_b():
        fpng_b200.decode_packed_device(flat, offsets, sizes, w, h, c, c, out=px_b, status=st_b)
        torch.cuda.synchronize()

    tight = int(sizes.max().item())

    def arm_b_tight():                                               # (b) with max_file_size = the largest file, known to the caller
        fpng_b200.decode_packed_device(flat, offsets, sizes, w, h, c, c, max_file_size=tight, out=px_b, status=st_b)
        torch.cuda.synchronize()

    def timed(fn):
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        return (time.perf_counter() - t0) * 1e3 / iters

    for _ in range(2):
        arm_a(); arm_b()
    arm_b_tight()
    a_ms, b_ms, bt_ms = [], [], []
    for _ in range(rounds):                                          # alternating arms
        a_ms.append(timed(arm_a))
        b_ms.append(timed(arm_b))
        bt_ms.append(timed(arm_b_tight))
    arm_b()
    identical = bool(torch.equal(px_a, px_b)) and bool(torch.equal(st_a, st_b))
    matches_input = bool(torch.equal(px_b, batch)) and bool((st_b == 0).all().item())

    def walk_ms(data, offs, szs):
        fpng_b200.get_info_batch_device(data, offs, szs)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            info = fpng_b200.get_info_batch_device(data, offs, szs)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters, info

    walk, info = walk_ms(flat, offsets, sizes)
    walk_ok = bool((info[:, 0] == 0).all().item())
    # every file with a 1 MiB ancillary chunk in front of fdEC (serial per-file CRC of 1 MiB)
    hb, ho, hsz = flat.cpu().numpy(), offsets.cpu().numpy(), sizes.cpu().numpy().view(np.uint32)
    big = [with_ancillary(bytes(hb[ho[i]: ho[i] + hsz[i]]), 1 << 20) for i in range(n)]
    bo = np.zeros(n + 1, np.int64)
    bo[1:] = np.cumsum([(len(f) + 15) // 16 * 16 for f in big])
    bbuf = np.zeros(int(bo[-1]), np.uint8)
    for i, f in enumerate(big):
        bbuf[bo[i]: bo[i] + len(f)] = np.frombuffer(f, np.uint8)
    bdata = torch.from_numpy(bbuf).to(dev)
    boffs = torch.from_numpy(bo).to(dev)
    bsz = torch.from_numpy(np.array([len(f) for f in big], np.uint32).view(np.int32)).to(dev)
    del big, bbuf
    walk_big, binfo = walk_ms(bdata, boffs, bsz)
    walk_big_ok = bool((binfo[:, 0] == 0).all().item())

    name, power = card()
    return {
        "workload": wl["name"], "kind": "g1", "images": n, "file_bytes": file_bytes, "card": name, "power_limit": power,
        "a_host_walk_ms": {"median": statistics.median(a_ms), "min": min(a_ms), "max": max(a_ms)},
        "b_decode_packed_device_ms": {"median": statistics.median(b_ms), "min": min(b_ms), "max": max(b_ms)},
        "b_max_file_size_tight_ms": {"median": statistics.median(bt_ms), "min": min(bt_ms), "max": max(bt_ms)},
        "speedup_median": statistics.median(a_ms) / statistics.median(b_ms),
        "walk_kernel_ms": walk, "walk_kernel_1MiB_ancillary_ms": walk_big, "walk_status_ok": walk_ok and walk_big_ok,
        "identical_pixels_and_status_a_b": identical, "b_equals_input": matches_input,
        "rounds": rounds, "iters_per_round": iters,
        "timing": "host wall time per call, each call ends in a device synchronise; walk kernels: CUDA events",
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["c2", "c3"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_decode: no CUDA device")
    import fpng_b200
    fpng_b200.fpng_init(0)
    for k in args.workload:
        print(json.dumps(run(k, args.rounds, args.iters)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
