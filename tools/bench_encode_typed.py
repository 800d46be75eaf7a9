"""Typed encode (float32 / bfloat16 input with a per-channel scale and bias, rounded to 8 bits by the conversion pre-pass) against
the torch chain followed by the uint8 encode, alternating in one process.

Arms, per workload:
  (a) encode_batch_device of the uint8 pixels (NHWC): the floor;
  (b) q = x.float().mul(s).add_(b).nan_to_num_(nan=0).round_().clamp_(0, 255).to(torch.uint8) in x's own layout, with the
      multiply in place after .float() for 16-bit input (one float32 temporary: the cheapest eager form of the chain), then the uint8
      encode of q's [n, h, w, c] view (planar for NCHW input);
  (c) encode_batch_device(x_view, scale=s, bias=b).
Workloads: C2 (256 x 1920x1080 RGB) and C3 (128 x 3840x2160 RGBA) of bench.py's g1 pixels, as float32 and bfloat16, NCHW and
NHWC, x = (v - 127.5) / 127.5 and s = b = 127.5; M1 (256 images of mixed shapes) as a list of bfloat16 CHW tensors through
encode_ragged_device, where (b) runs the chain per image.  1-pass.  Each round times 3 calls of every arm with CUDA events, rounds
alternate the arms, the median of 5 rounds is reported, and (b) and (c) are compared byte for byte in every round.  One profiled
typed call gives the conversion kernel's time (encode profile slot 9); its bytes are the elements read (x sizeof(T)) plus the
uint8 bytes written, against the H100 SXM data sheet's 3.35 TB/s.  Card name and power limit are read in the same run; one JSON
line per workload, dtype and layout.

    python tools/bench_encode_typed.py [--workload c2 c3 m1] [--dtype float32 bfloat16] [--layout nchw nhwc] [--rounds 5] [--iters 3]
"""
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

import bench  # noqa: E402
from bench_device_decode import card  # noqa: E402
from bench_ragged_encode import M1_SHAPES  # noqa: E402

HBM_TBS = 3.35
SCALE = BIAS = 127.5


def to_float(u8, dtype, nchw):
    """(v - 127.5) / 127.5 of a uint8 [.., h, w, c] tensor as dtype, stored NCHW (CHW) or NHWC; returns the stored tensor"""
    import torch
    x = u8.permute(0, 3, 1, 2) if (nchw and u8.dim() == 4) else (u8.permute(2, 0, 1) if nchw else u8)
    return x.float().sub_(127.5).div_(127.5).to(dtype).contiguous()


def chain(x, c, channel_dim):
    import torch
    shape = [1] * x.dim()
    shape[channel_dim] = c
    s = torch.full(shape, SCALE, dtype=torch.float32, device=x.device)
    b = torch.full(shape, BIAS, dtype=torch.float32, device=x.device)
    y = x.mul(s) if x.dtype == torch.float32 else x.float().mul_(s)      # one float32 temporary
    return y.add_(b).nan_to_num_(nan=0.0).round_().clamp_(0, 255).to(torch.uint8)


def same_batch(r1, r2):
    import torch
    (o1, s1), (o2, s2) = r1, r2
    if not torch.equal(s1, s2):
        return False
    sz = s1.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return all(torch.equal(o1[i, :sz[i]], o2[i, :sz[i]]) for i in range(len(sz)))


def same_ragged(r1, r2):
    import torch
    (o1, f1, s1), (o2, f2, s2) = r1, r2
    if not (torch.equal(f1, f2) and torch.equal(s1, s2)):
        return False
    offs, sz = f1.cpu().numpy(), s1.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    return all(torch.equal(o1[offs[i]:offs[i] + sz[i]], o2[offs[i]:offs[i] + sz[i]]) for i in range(len(sz)))


def workload(name, dtype, nchw, dev):
    """(arms a, b, c; compare(b_result, c_result); elements converted; sizeof(T))"""
    import torch

    import fpng_b200
    es = torch.empty((), dtype=dtype).element_size()
    if name == "m1":
        n = 256
        shapes = [M1_SHAPES[i % len(M1_SHAPES)] for i in range(n)]
        u8 = []
        for (w, h, c) in sorted(set(shapes)):
            k = shapes.count((w, h, c))
            batch = bench.make_device_batch(dict(w=w, h=h, chans=c), "g1", k, dev)
            u8 += [(shapes.index((w, h, c)), batch[j]) for j in range(k)]
        u8 = [t for _, t in sorted(u8, key=lambda p: p[0])]
        xs = [to_float(t, dtype, True) for t in u8]                         # CHW per image
        views = [x.permute(1, 2, 0) for x in xs]
        a = lambda: fpng_b200.encode_ragged_device(u8, 0)                   # noqa: E731
        b = lambda: fpng_b200.encode_ragged_device([chain(x, x.shape[0], 0).permute(1, 2, 0) for x in xs], 0)   # noqa: E731
        c = lambda: fpng_b200.encode_ragged_device(views, 0, scale=SCALE, bias=BIAS)   # noqa: E731
        return a, b, c, same_ragged, sum(t.numel() for t in u8), es
    wl = bench.WORKLOADS[name]
    n, h, w, ch = wl["images"], wl["h"], wl["w"], wl["chans"]
    u8 = bench.make_device_batch(wl, "g1", n, dev)
    x = to_float(u8, dtype, nchw)
    view = x.permute(0, 2, 3, 1) if nchw else x

    def b():
        q = chain(x, ch, 1 if nchw else 3)
        return fpng_b200.encode_batch_device(q.permute(0, 2, 3, 1) if nchw else q, 0)
    return (lambda: fpng_b200.encode_batch_device(u8, 0), b, lambda: fpng_b200.encode_batch_device(view, 0, scale=SCALE, bias=BIAS),
            same_batch, u8.numel(), es)


def run(name, dtype, nchw, rounds, iters):
    import torch

    from fpng_b200._lib import lib
    dev = torch.device("cuda", 0)
    a, b, c, same, elems, es = workload(name, dtype, nchw, dev)
    L = lib()
    L.fpngb_profile_enable.argtypes = [C.c_int]
    L.fpngb_profile_read.argtypes = [C.POINTER(C.c_float), C.c_int]
    for fn in (a, b, c, a, b, c):                                          # warm-up: workspace, conversion buffer, first launches
        fn()
    torch.cuda.synchronize()
    arms = {"a": a, "b": b, "c": c}
    times = {k: [] for k in arms}
    identical = []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        last = {}
        for k, fn in arms.items():
            ev0.record()
            for _ in range(iters):
                last[k] = fn()
            ev1.record()
            torch.cuda.synchronize()
            times[k].append(ev0.elapsed_time(ev1) / iters)
        identical.append(same(last["b"], last["c"]))
        del last
    ms = (C.c_float * 10)()
    L.fpngb_profile_read(ms, 10)
    L.fpngb_profile_enable(1)
    conv = []
    for _ in range(3):
        c()
        assert L.fpngb_profile_read(ms, 10) == 1
        conv.append(float(ms[9]))
    L.fpngb_profile_enable(0)
    med = {k: statistics.median(v) for k, v in times.items()}
    u = statistics.median(conv)
    conv_bytes = elems * es + elems
    return {"workload": name, "dtype": str(dtype).replace("torch.", ""), "layout": "chw list" if name == "m1" else ("nchw" if nchw else "nhwc"),
            "a_uint8_encode_ms": round(med["a"], 3), "b_torch_chain_then_uint8_encode_ms": round(med["b"], 3),
            "c_typed_encode_ms": round(med["c"], 3), "c_vs_b_speedup": round(med["b"] / med["c"], 3),
            "c_minus_a_ms": round(med["c"] - med["a"], 3), "b_equals_c_bytewise_every_round": all(identical),
            "conversion_kernel_ms": round(u, 3), "conversion_bytes": conv_bytes,
            "conversion_GBps": round(conv_bytes / (u * 1e-3) / 1e9, 1),
            "conversion_share_of_3.35TBps": round(conv_bytes / (u * 1e-3) / (HBM_TBS * 1e12), 3),
            "conversion_bound_ms_at_3.35TBps": round(conv_bytes / (HBM_TBS * 1e12) * 1e3, 3),
            "all_ms": {k: [round(t, 3) for t in v] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["c2", "c3", "m1"], choices=["c2", "c3", "m1"])
    ap.add_argument("--dtype", nargs="+", default=["float32", "bfloat16"], choices=["float32", "float16", "bfloat16"])
    ap.add_argument("--layout", nargs="+", default=["nchw", "nhwc"], choices=["nchw", "nhwc"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch

    import fpng_b200
    fpng_b200.fpng_init(0)
    name, power = card()
    for w in args.workload:
        for dt in (["bfloat16"] if w == "m1" else args.dtype):
            for lay in (["nchw"] if w == "m1" else args.layout):
                r = run(w, getattr(torch, dt), lay == "nchw", args.rounds, args.iters)
                r.update({"card": name, "power_limit": power, "rounds": args.rounds, "iters_per_round": args.iters})
                print(json.dumps(r), flush=True)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
