"""Cost of the decoder's opt-in integrity check (fpngb_set_decode_verify): switch off against on, alternating in one process.

Workloads: C2 (256 x 1920x1080 RGB, G1 images) and C3 (128 x 3840x2160 RGBA) through decode_packed_device, and M1 (256 mixed
shapes up to 4K) through decode_packed_ragged_device.  Per round each arm runs `iters` calls timed with CUDA events; the median of
the rounds is reported, with the device times of the two verify kernels (decode profile slots 6 and 7) from one profiled call.
The outputs of the two arms are compared byte for byte.  Card name and power limit are read in the same run; one JSON line per
workload."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_device_decode import card  # noqa: E402
from bench_ragged_decode import M1_SHAPES  # noqa: E402


def packed(files, dev):
    import torch
    offs = np.zeros(len(files) + 1, np.int64)
    offs[1:] = np.cumsum([(len(f) + 15) // 16 * 16 for f in files])
    buf = np.zeros(int(offs[-1]) + 16, np.uint8)
    for i, f in enumerate(files):
        buf[offs[i]: offs[i] + len(f)] = np.frombuffer(f, np.uint8)
    return (torch.from_numpy(buf).to(dev), torch.from_numpy(offs[:-1].copy()).to(dev),
            torch.from_numpy(np.array([len(f) for f in files], np.uint32).view(np.int32)).to(dev))


def encode_files(shapes, dev):
    """shapes: [(w, h, c)] per image -> files (one encode call per shape group, G1 images)"""
    import bench
    import fpng_b200
    files = [None] * len(shapes)
    groups = {}
    for i, s in enumerate(shapes):
        groups.setdefault(s, []).append(i)
    for (w, h, c), idx in groups.items():
        batch = bench.make_device_batch(dict(w=w, h=h, chans=c), "g1", len(idx), dev)
        enc, sizes = fpng_b200.encode_batch_device(batch, 0)
        enc, sizes = enc.cpu().numpy(), sizes.cpu().numpy()
        for t, i in enumerate(idx):
            files[i] = enc[t, :sizes[t]].tobytes()
        del batch, enc
    return files


def workload(name, dev):
    import torch

    import fpng_b200
    if name == "m1":
        n = 256
        shapes = [M1_SHAPES[i % len(M1_SHAPES)] for i in range(n)]
        files = encode_files(shapes, dev)
        order = np.random.RandomState(1234).permutation(n)
        files = [files[i] for i in order]
        data, offsets, sizes = packed(files, dev)
        info = [fpng_b200.get_info_ex(f) for f in files]
        mfs, mw, mh = max(map(len, files)), max(i[1] for i in info), max(i[2] for i in info)
        out = torch.empty(sum((i[1] * i[2] * 3 + 15) // 16 * 16 for i in info), dtype=torch.uint8, device=dev)

        def call():
            return fpng_b200.decode_packed_ragged_device(data, offsets, sizes, 3, out=out, max_file_size=mfs, max_w=mw, max_h=mh)[3]
        return call, out, n
    w, h, c, n = (1920, 1080, 3, 256) if name == "c2" else (3840, 2160, 4, 128)
    files = encode_files([(w, h, c)] * n, dev)
    data, offsets, sizes = packed(files, dev)
    mfs = max(map(len, files))
    out = torch.empty((n, h, w, c), dtype=torch.uint8, device=dev)

    def call():
        return fpng_b200.decode_packed_device(data, offsets, sizes, w, h, c, c, max_file_size=mfs, out=out)[1]
    return call, out, n


def run(name, rounds, iters):
    import torch

    import fpng_b200
    from fpng_b200._lib import lib
    dev = torch.device("cuda", 0)
    call, out, n = workload(name, dev)
    L = lib()
    L.fpngb_decode_profile_enable.argtypes = [C.c_int]
    L.fpngb_decode_profile_read.argtypes = [C.POINTER(C.c_float), C.c_int]
    ref = {}
    for on in (False, True):                                 # warm-up, outputs and statuses of both arms
        fpng_b200.set_decode_verify(on)
        out.fill_(0)
        st = call()
        torch.cuda.synchronize()
        ref[on] = (out.cpu().numpy().copy(), st.cpu().numpy().copy())
    identical = bool(np.array_equal(ref[False][0], ref[True][0]) and np.array_equal(ref[False][1], ref[True][1]))
    assert int(np.count_nonzero(ref[True][1])) == 0
    times = {False: [], True: []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for on in (False, True):
            fpng_b200.set_decode_verify(on)
            ev0.record()
            for _ in range(iters):
                call()
            ev1.record()
            torch.cuda.synchronize()
            times[on].append(ev0.elapsed_time(ev1) / iters)
    fpng_b200.set_decode_verify(True)
    L.fpngb_decode_profile_enable(1)
    call()
    ms = (C.c_float * 8)()
    assert L.fpngb_decode_profile_read(ms, 8) == 1
    L.fpngb_decode_profile_enable(0)
    fpng_b200.set_decode_verify(False)
    off, on = statistics.median(times[False]), statistics.median(times[True])
    return {"workload": name, "files": n, "off_ms": round(off, 3), "on_ms": round(on, 3), "cost_ms": round(on - off, 3),
            "off_all": [round(t, 3) for t in times[False]], "on_all": [round(t, 3) for t in times[True]],
            "crc_kernel_ms": round(float(ms[6]), 4), "adler_kernel_ms": round(float(ms[7]), 4), "outputs_identical": identical}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["c2", "c3", "m1"], choices=["c2", "c3", "m1"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import fpng_b200
    fpng_b200.fpng_init(0)
    name, power = card()
    for w in args.workload:
        r = run(w, args.rounds, args.iters)
        r.update({"card": name, "power_limit": power, "rounds": args.rounds, "iters_per_round": args.iters})
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
