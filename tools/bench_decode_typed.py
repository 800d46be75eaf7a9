"""Typed decode (float32 / bfloat16 output with a per-channel scale and bias, converted in the unfilter pass) against the uint8
decode followed by the usual torch chain, alternating in one process.

Arms, per workload:
  (a) uint8 decode into NHWC, as the uint8 calls write it;
  (b) the uint8 decode, then x = out.permute(0, 3, 1, 2).float().mul_(scale).add_(bias) (and .to(torch.bfloat16) for bf16);
  (c) the typed decode into a contiguous NCHW tensor of the same values (for M1: each file's HWC slot of the ragged output).
Workloads: C2 (256 x 1920x1080 RGB) and C3 (128 x 3840x2160 RGBA, decoded to RGB) through decode_packed_device, M1 (256 mixed
shapes) through decode_packed_ragged_device, where (b) runs the chain per file.  Each arm's calls are timed with CUDA events,
rounds alternate the arms and the median is reported.  (b) and (c) are compared bit for bit.  One profiled typed call gives the
unfilter kernel's time (decode profile slot 5), its bytes (delta rows read + elements written) and its rate against the H100 SXM
data sheet's 3.35 TB/s.  Card name and power limit are read in the same run; one JSON line per workload and dtype."""
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

from bench_decode_verify import encode_files, packed  # noqa: E402
from bench_device_decode import card  # noqa: E402
from bench_ragged_decode import M1_SHAPES  # noqa: E402

HBM_TBS = 3.35


def workload(name, dev, dtype):
    """(uint8 call, chain, typed call, compare, unfilter bytes, files)"""
    import torch

    import fpng_b200
    s_np, b_np = fpng_b200.normalize_scale_bias((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
    s_t, b_t = torch.from_numpy(s_np).to(dev).view(1, 3, 1, 1), torch.from_numpy(b_np).to(dev).view(1, 3, 1, 1)
    es = torch.empty((), dtype=dtype).element_size()
    d = 3
    if name == "m1":
        n = 256
        shapes = [M1_SHAPES[i % len(M1_SHAPES)] for i in range(n)]
        files = encode_files(shapes, dev)
        files = [files[i] for i in np.random.RandomState(1234).permutation(n)]
        data, offsets, sizes = packed(files, dev)
        info = [fpng_b200.get_info_ex(f) for f in files]
        mfs, mw, mh = max(map(len, files)), max(i[1] for i in info), max(i[2] for i in info)
        u8 = torch.empty(sum((i[1] * i[2] * d + 15) // 16 * 16 for i in info), dtype=torch.uint8, device=dev)
        typed = torch.empty(sum((i[1] * i[2] * d * es + 15) // 16 * 16 for i in info) // es, dtype=dtype, device=dev)
        oo = [0]
        for i in info:
            oo.append(oo[-1] + (i[1] * i[2] * d * es + 15) // 16 * 16)
        oo8 = [0]
        for i in info:
            oo8.append(oo8[-1] + (i[1] * i[2] * d + 15) // 16 * 16)
        views8 = [u8[oo8[k]:oo8[k] + i[1] * i[2] * d].view(i[2], i[1], d) for k, i in enumerate(info)]
        viewsT = [typed[oo[k] // es:oo[k] // es + i[1] * i[2] * d].view(i[2], i[1], d) for k, i in enumerate(info)]

        def a():
            fpng_b200.decode_packed_ragged_device(data, offsets, sizes, d, out=u8, max_file_size=mfs, max_w=mw, max_h=mh)

        def b():
            a()
            return [(v.permute(2, 0, 1).float().mul_(s_t[0]).add_(b_t[0])).to(dtype) for v in views8]

        def c():
            fpng_b200.decode_packed_ragged_device(data, offsets, sizes, d, out=typed, max_file_size=mfs, max_w=mw, max_h=mh,
                                                  scale=s_np, bias=b_np)

        def same(xs):
            return all(torch.equal(x.contiguous().view(torch.int16 if es == 2 else torch.int32),
                                   v.permute(2, 0, 1).contiguous().view(torch.int16 if es == 2 else torch.int32)) for x, v in zip(xs, viewsT))
        px = sum(i[1] * i[2] for i in info)
        delta = sum(i[2] * ((i[1] * i[3] + 15) // 16 * 16) for i in info)
        return a, b, c, same, delta + px * d * es, n
    w, h, cf, n = (1920, 1080, 3, 256) if name == "c2" else (3840, 2160, 4, 128)
    files = encode_files([(w, h, cf)] * n, dev)
    data, offsets, sizes = packed(files, dev)
    mfs = max(map(len, files))
    u8 = torch.empty((n, h, w, d), dtype=torch.uint8, device=dev)
    nchw = torch.empty((n, d, h, w), dtype=dtype, device=dev)

    def a():
        fpng_b200.decode_packed_device(data, offsets, sizes, w, h, cf, d, max_file_size=mfs, out=u8)

    def b():
        a()
        x = u8.permute(0, 3, 1, 2).float().mul_(s_t).add_(b_t)
        return x if dtype == torch.float32 else x.to(dtype)

    def c():
        fpng_b200.decode_packed_device(data, offsets, sizes, w, h, cf, d, max_file_size=mfs, out=nchw.permute(0, 2, 3, 1),
                                       scale=s_np, bias=b_np)

    def same(x):
        it = torch.int16 if es == 2 else torch.int32
        return bool(torch.equal(x.contiguous().view(it), nchw.view(it)))
    return a, b, c, same, n * h * ((w * cf + 15) // 16 * 16) + n * h * w * d * es, n


def run(name, dtype, rounds, iters):
    import torch

    from fpng_b200._lib import lib
    dev = torch.device("cuda", 0)
    a, b, c, same, unfilter_bytes, n = workload(name, dev, dtype)
    L = lib()
    L.fpngb_decode_profile_enable.argtypes = [C.c_int]
    L.fpngb_decode_profile_read.argtypes = [C.POINTER(C.c_float), C.c_int]
    a(); c()
    x = b()
    torch.cuda.synchronize()
    identical = same(x)
    del x
    arms = {"a": a, "b": b, "c": c}
    times = {k: [] for k in arms}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, fn in arms.items():
            ev0.record()
            for _ in range(iters):
                fn()
            ev1.record()
            torch.cuda.synchronize()
            times[k].append(ev0.elapsed_time(ev1) / iters)
    L.fpngb_decode_profile_enable(1)
    ms = (C.c_float * 8)()
    unf = []
    for _ in range(3):
        c()
        assert L.fpngb_decode_profile_read(ms, 8) == 1
        unf.append(float(ms[5]))
    a()
    assert L.fpngb_decode_profile_read(ms, 8) == 1
    unf8 = float(ms[5])
    L.fpngb_decode_profile_enable(0)
    med = {k: statistics.median(v) for k, v in times.items()}
    u = statistics.median(unf)
    return {"workload": name, "dtype": str(dtype).replace("torch.", ""), "files": n,
            "a_uint8_ms": round(med["a"], 3), "b_uint8_torch_chain_ms": round(med["b"], 3), "c_typed_ms": round(med["c"], 3),
            "c_vs_b_speedup": round(med["b"] / med["c"], 3), "b_equals_c_bitwise": identical,
            "typed_unfilter_ms": round(u, 3), "uint8_unfilter_ms": round(unf8, 3), "typed_unfilter_bytes": unfilter_bytes,
            "typed_unfilter_GBps": round(unfilter_bytes / (u * 1e-3) / 1e9, 1),
            "typed_unfilter_share_of_3.35TBps": round(unfilter_bytes / (u * 1e-3) / (HBM_TBS * 1e12), 3),
            "all_ms": {k: [round(t, 3) for t in v] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["c2", "c3", "m1"], choices=["c2", "c3", "m1"])
    ap.add_argument("--dtype", nargs="+", default=["float32", "bfloat16"], choices=["float32", "float16", "bfloat16"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch

    import fpng_b200
    fpng_b200.fpng_init(0)
    name, power = card()
    for w in args.workload:
        for dt in args.dtype:
            r = run(w, getattr(torch, dt), args.rounds, args.iters)
            r.update({"card": name, "power_limit": power, "rounds": args.rounds, "iters_per_round": args.iters})
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
