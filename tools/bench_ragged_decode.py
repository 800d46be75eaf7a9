"""Decode of packed device files of mixed shapes: fpngb_decode_packed_ragged_device against grouping by shape on the host.

M1, mixed: 256 bench.py-style g1 images cycling through 640x480 RGB, 1280x720 RGB, 1920x1080 RGB, 1920x1080 RGBA, 687x1012 RGB
and 3840x2160 RGB, encoded 1-pass per shape group with encode_batch_device and packed interleaved in a seeded order (16-byte
aligned files, one flat device buffer).  Three arms, timed alternately:
  (a) decode_packed_ragged_device with every bound given (no host synchronisation);
  (b) what a caller did before: get_info_batch_device, read the info back, group by shape on the host, one
      decode_packed_device per shape with its own offsets / sizes tensors;
  (c) the decode_packed_device calls of (b) alone, shapes and groups known in advance (a floor).
U, uniform: bench.py's C2 batch packed by dist.compact, the ragged call against decode_packed_device (same max_file_size).
Times are host wall time per call ending in a device synchronise (median over alternating rounds); per-kernel device times come
from fpngb_decode_profile_read (prepare, scan, link, write, stored, unfilter + status), summed over the calls of an arm.  The
outputs of all arms are compared byte for byte.  Card name and power limit are read in the same run; one JSON line per workload.

    python tools/bench_ragged_decode.py [--workload m1 u] [--rounds 5] [--iters 3]
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

M1_SHAPES = [(640, 480, 3), (1280, 720, 3), (1920, 1080, 3), (1920, 1080, 4), (687, 1012, 3), (3840, 2160, 3)]
KERNELS = ["prepare", "scan", "link", "write", "stored", "unfilter_status"]


def profile(fn):
    """device times of the decode kernels of the calls fn makes, summed (one profile read after each call)"""
    from fpng_b200._lib import lib
    L = lib()
    L.fpngb_decode_profile_enable(1)
    total = np.zeros(6)
    ms = (C.c_float * 6)()
    for after_call in fn(each=True):
        if not after_call:
            continue
        assert L.fpngb_decode_profile_read(ms, 6) == 1
        total += np.array(ms[:])
    L.fpngb_decode_profile_enable(0)
    return dict(zip(KERNELS, [round(float(v), 4) for v in total]))


def timed(fn, iters):
    t0 = time.perf_counter()
    for _ in range(iters):
        for _ in fn():
            pass
    return (time.perf_counter() - t0) * 1e3 / iters


def stats(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def m1(rounds, iters):
    import torch

    import bench
    import fpng_b200

    dev = torch.device("cuda", 0)
    n = 256
    files = []
    for k, (w, h, c) in enumerate(M1_SHAPES):                           # image i has shape M1_SHAPES[i % 6]
        idx = list(range(k, n, len(M1_SHAPES)))
        batch = bench.make_device_batch(dict(w=w, h=h, chans=c), "g1", len(idx), dev)     # one encode call per shape group
        enc, sizes = fpng_b200.encode_batch_device(batch, 0)
        enc, sizes = enc.cpu().numpy(), sizes.cpu().numpy()
        files += [(i, enc[t, :sizes[t]].tobytes()) for t, i in enumerate(idx)]
        del batch, enc
    files.sort()
    files = [f for _, f in files]
    order = np.random.RandomState(1234).permutation(n)                   # interleaved, seeded
    files = [files[i] for i in order]
    offs = np.zeros(n + 1, np.int64)
    offs[1:] = np.cumsum([(len(f) + 15) // 16 * 16 for f in files])
    buf = np.zeros(int(offs[-1]), np.uint8)
    for i, f in enumerate(files):
        buf[offs[i]: offs[i] + len(f)] = np.frombuffer(f, np.uint8)
    data = torch.from_numpy(buf).to(dev)
    offsets = torch.from_numpy(offs).to(dev)
    sizes = torch.from_numpy(np.array([len(f) for f in files], np.uint32).view(np.int32)).to(dev)
    del buf
    info = [fpng_b200.get_info_ex(f) for f in files]
    max_file_size = max(len(f) for f in files)
    max_w, max_h = max(i[1] for i in info), max(i[2] for i in info)
    del files

    # (a) the ragged call
    d_out_total = sum((i[1] * i[2] * 3 + 15) // 16 * 16 for i in info)
    out_a = torch.empty(d_out_total, dtype=torch.uint8, device=dev)
    res_a = {}

    def arm_a(each=False):
        res_a["r"] = decode_ragged()
        if each:
            yield True
        torch.cuda.synchronize()
        yield False

    def decode_ragged():
        # desired = the file's own channel count is not one value for a mixed batch: decode to 3 channels (RGB), as (b) does
        return fpng_b200.decode_packed_ragged_device(data, offsets, sizes, 3, out=out_a, max_file_size=max_file_size,
                                                    max_w=max_w, max_h=max_h)

    # (b) walk, read back, group on the host, one decode_packed_device per shape
    outs_b = {}

    def arm_b(each=False):
        inf = fpng_b200.get_info_batch_device(data, offsets, sizes).cpu().numpy()
        groups = {}
        for i in range(n):
            groups.setdefault((int(inf[i, 1]), int(inf[i, 2]), int(inf[i, 3])), []).append(i)
        for (w, h, c), idx in groups.items():
            ix = torch.tensor(idx, dtype=torch.int64, device=dev)
            outs_b[(w, h, c)] = (idx,) + fpng_b200.decode_packed_device(data, offsets[ix], sizes[ix], w, h, c, 3,
                                                                        max_file_size=max_file_size)
            if each:
                yield True
        torch.cuda.synchronize()
        yield False

    # (c) the decode calls of (b) alone, groups prepared in advance
    groups_c = {}
    for i, inf in enumerate(info):
        groups_c.setdefault(inf[1:4], []).append(i)
    prep_c = {k: (torch.tensor(v, dtype=torch.int64, device=dev),) for k, v in groups_c.items()}
    prep_c = {k: (offsets[ix], sizes[ix], torch.empty((len(groups_c[k]), k[1], k[0], 3), dtype=torch.uint8, device=dev),
                  torch.empty((len(groups_c[k]),), dtype=torch.int32, device=dev)) for k, (ix,) in prep_c.items()}

    def arm_c(each=False):
        for (w, h, c), (o, s, px, st) in prep_c.items():
            fpng_b200.decode_packed_device(data, o, s, w, h, c, 3, max_file_size=max_file_size, out=px, status=st)
            if each:
                yield True
        torch.cuda.synchronize()
        yield False

    for fn in (arm_a, arm_b, arm_c, arm_a, arm_b, arm_c):
        for _ in fn():
            pass
    a_ms, b_ms, c_ms = [], [], []
    for _ in range(rounds):
        a_ms.append(timed(arm_a, iters)); b_ms.append(timed(arm_b, iters)); c_ms.append(timed(arm_c, iters))
    prof = {"a": profile(arm_a), "b": profile(arm_b), "c": profile(arm_c)}

    # equal outputs: every file's pixels and status in (a), (b) and (c)
    out, oo, inf_a, st_a = res_a["r"]
    views = fpng_b200.ragged_views(out, oo, inf_a, st_a, 3)
    equal = bool((st_a == 0).all().item())
    for key, (idx, px, st) in outs_b.items():
        o, s, pxc, stc = prep_c[key]
        equal &= bool(torch.equal(px, pxc)) and bool((st == 0).all().item()) and bool((stc == 0).all().item())
        for k, i in enumerate(idx):
            equal &= views[i] is not None and bool(torch.equal(views[i], px[k]))
    torch.cuda.synchronize()
    return {"workload": "M1 256 mixed g1 1-pass: " + ", ".join(f"{w}x{h}x{c}" for w, h, c in M1_SHAPES) + " -> RGB",
            "file_bytes": int(offs[-1]), "pixel_bytes": d_out_total,
            "a_ragged_ms": stats(a_ms), "b_walk_readback_group_ms": stats(b_ms), "c_group_decodes_alone_ms": stats(c_ms),
            "kernel_ms": prof, "outputs_equal_a_b_c": equal}


def uniform(rounds, iters):
    import torch

    import bench
    import fpng_b200
    from fpng_b200 import dist

    wl = bench.WORKLOADS["c2"]
    w, h, c, n = wl["w"], wl["h"], wl["chans"], wl["images"]
    dev = torch.device("cuda", 0)
    batch = bench.make_device_batch(wl, "g1", n, dev)
    enc, sizes = fpng_b200.encode_batch_device(batch, 0)
    flat, offsets = dist.compact(enc, sizes)
    del enc
    mfs = int(sizes.max().item())
    px_p = torch.empty((n, h, w, c), dtype=torch.uint8, device=dev)
    st_p = torch.empty((n,), dtype=torch.int32, device=dev)
    out_r = torch.empty(n * h * w * c, dtype=torch.uint8, device=dev)
    res = {}

    def arm_packed(each=False):
        fpng_b200.decode_packed_device(flat, offsets, sizes, w, h, c, c, max_file_size=mfs, out=px_p, status=st_p)
        if each:
            yield True
        torch.cuda.synchronize()
        yield False

    def arm_ragged(each=False):
        res["r"] = fpng_b200.decode_packed_ragged_device(flat, offsets, sizes, c, out=out_r, max_file_size=mfs, max_w=w, max_h=h)
        if each:
            yield True
        torch.cuda.synchronize()
        yield False

    for fn in (arm_packed, arm_ragged, arm_packed, arm_ragged):
        for _ in fn():
            pass
    p_ms, r_ms = [], []
    for _ in range(rounds):
        p_ms.append(timed(arm_packed, iters)); r_ms.append(timed(arm_ragged, iters))
    prof = {"packed": profile(arm_packed), "ragged": profile(arm_ragged)}
    _, oo, info, st = res["r"]
    equal = bool(torch.equal(out_r.view(n, h, w, c), px_p)) and bool(torch.equal(st, st_p)) and bool((st == 0).all().item())
    equal &= bool(torch.equal(px_p, batch))
    return {"workload": "U " + wl["name"] + " packed by dist.compact", "decode_packed_device_ms": stats(p_ms),
            "ragged_ms": stats(r_ms), "kernel_ms": prof, "outputs_equal_and_input": equal}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["m1", "u"], choices=["m1", "u"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_decode: no CUDA device")
    import fpng_b200
    fpng_b200.fpng_init(0)
    for k in args.workload:
        r = (m1 if k == "m1" else uniform)(args.rounds, args.iters)
        name, power = card()
        r.update({"card": name, "power_limit": power, "rounds": args.rounds, "iters_per_round": args.iters,
                  "timing": "host wall time per call ending in a device synchronise, median of alternating rounds; "
                            "kernel_ms: fpngb_decode_profile_read summed over an arm's decode calls"})
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
