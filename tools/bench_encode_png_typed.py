"""Typed PNG encode (float32 / float16 / bfloat16 input written as 8- or 16-bit PNG samples by the conversion pre-pass) against the
torch chain followed by the uint8 / uint16 PNG encode, alternating in one process.

Workloads, from tests/pngenc_workloads.py:
  T1: E2 (256 x 640x480 depth maps) as float32 metres, written at 16 bits with scale 1000 (millimetres);
  T2: E3 (128 x 1920x1080 gray) as float16 in [0, 1], written at 8 bits with scale 255;
  T3: E4 (64 x 1920x1080 RGBA16) as bfloat16 NCHW in [-1, 1], written at 16 bits with scale = bias = 32767.5.
Arms, per workload:
  (a) encode_png_device of the pre-quantised uint8 / uint16 images (the floor);
  (b) q = nan_to_num(x.float() * s + b, nan=0).round().clamp(0, 2**D - 1).to(uint8 / uint16) on the whole batch in x's own
      layout (in place after the first op), then encode_png_device of q's per-image views (planar for NCHW);
  (c) encode_png_device(x views, scale=s, bias=b, depth=D).
Each round times `iters` calls of every arm with CUDA events, rounds alternate the arms, the median of the rounds is reported,
and (b) and (c) are compared byte for byte in every round.  Three profiled typed calls give the conversion kernel's time (encode
profile slot 9); its bytes are the elements read (x sizeof(T)) plus the samples written (x D / 8), against the H100 SXM data
sheet's 3.35 TB/s.  The card's name, power limit and SM clocks are read in the same run; one JSON line per workload.

    python tools/bench_encode_png_typed.py [--workload T1 T2 T3] [--rounds 5] [--iters 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import pngenc_workloads as pw  # noqa: E402

HBM_TBS = 3.35


def card():
    """name, power limit and SM clocks (current, max) of GPU 0, as nvidia-smi reports them"""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    return [v.strip() for v in q.stdout.splitlines()[0].split(",")] if q.returncode == 0 and q.stdout else ["unknown"] * 4


def chain(x, s, b, depth, channel_dim):
    """the cheapest eager form of the rule on a whole batch: one float32 temporary, the rest in place"""
    import torch
    shape = [1] * x.dim()
    shape[channel_dim] = len(s)
    st = torch.tensor(s, dtype=torch.float32, device=x.device).view(shape)
    bt = torch.tensor(b, dtype=torch.float32, device=x.device).view(shape)
    y = x.mul(st) if x.dtype == torch.float32 else x.float().mul_(st)
    y = y.add_(bt).nan_to_num_(nan=0.0).round_().clamp_(0, (1 << depth) - 1)
    return y.to(torch.uint8 if depth == 8 else torch.uint16)


def workload(name, dev):
    """(x: the whole batch as stored, per_image: a batch like x -> its [h, w, c] views, scale, bias, depth, channel dim of x)"""
    import torch
    imgs = np.stack(pw.workload({"T1": "E2", "T2": "E3", "T3": "E4"}[name]))          # [n, h, w, c] uint8 / uint16
    u = torch.from_numpy(imgs.astype(np.int32)).to(dev)
    if name == "T1":
        x = (u.float() / 1000.0).contiguous()                                           # metres, float32 NHWC
        s, b, depth, cdim = [1000.0], [0.0], 16, 3
    elif name == "T2":
        x = (u.float() / 255.0).to(torch.float16).contiguous()
        s, b, depth, cdim = [255.0], [0.0], 8, 3
    else:
        x = (u.float() / 32767.5 - 1.0).to(torch.bfloat16).permute(0, 3, 1, 2).contiguous()   # NCHW
        s, b, depth, cdim = [32767.5] * 4, [32767.5] * 4, 16, 1
    del u
    per_image = (lambda t: [t[i].permute(1, 2, 0) for i in range(t.shape[0])]) if cdim == 1 else (lambda t: list(t))
    return x, per_image, s, b, depth, cdim


def same(r1, r2):
    import torch
    (o1, f1, s1), (o2, f2, s2) = r1, r2
    if not (torch.equal(f1, f2) and torch.equal(s1, s2)):
        return False
    offs, sz = f1.cpu().numpy(), s1.cpu().numpy().astype(np.int64)
    return all(torch.equal(o1[offs[i]:offs[i] + sz[i]], o2[offs[i]:offs[i] + sz[i]]) for i in range(len(sz)))


def run(name, rounds, iters):
    import torch

    import fpng_b200
    from fpng_b200._lib import lib
    dev = torch.device("cuda", 0)
    x, per_image, s, b, depth, cdim = workload(name, dev)
    views = per_image(x)
    q_views = [t.contiguous() for t in per_image(chain(x, s, b, depth, cdim))]         # the floor's pre-quantised images
    arms = {
        "a": lambda: fpng_b200.encode_png_device(q_views),
        "b": lambda: fpng_b200.encode_png_device(per_image(chain(x, s, b, depth, cdim))),
        "c": lambda: fpng_b200.encode_png_device(views, scale=s, bias=b, depth=depth),
    }
    L = lib()
    L.fpngb_profile_enable.argtypes = [C.c_int]
    L.fpngb_profile_read.argtypes = [C.POINTER(C.c_float), C.c_int]
    for _ in range(2):                                                      # warm-up: workspace, conversion buffer, first launches
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
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
        identical.append(same(last["b"], last["c"]) and same(last["a"], last["c"]))
        del last
    ms = (C.c_float * 10)()
    L.fpngb_profile_read(ms, 10)
    L.fpngb_profile_enable(1)
    conv = []
    for _ in range(3):
        arms["c"]()
        assert L.fpngb_profile_read(ms, 10) == 1
        conv.append(float(ms[9]))
    L.fpngb_profile_enable(0)
    torch.cuda.synchronize()
    med = {k: statistics.median(v) for k, v in times.items()}
    u = statistics.median(conv)
    elems = x.numel()
    conv_bytes = elems * x.element_size() + elems * depth // 8
    return {"workload": name, "dtype": str(x.dtype).replace("torch.", ""), "depth": depth, "images": len(views),
            "shape_hwc": list(views[0].shape), "layout": "nchw" if cdim == 1 else "nhwc",
            "a_uint_encode_ms": round(med["a"], 3), "b_torch_chain_then_uint_encode_ms": round(med["b"], 3),
            "c_typed_encode_ms": round(med["c"], 3), "c_vs_b_speedup": round(med["b"] / med["c"], 3),
            "c_minus_a_ms": round(med["c"] - med["a"], 3), "a_b_c_equal_bytewise_every_round": all(identical),
            "conversion_kernel_ms": round(u, 3), "conversion_bytes": conv_bytes,
            "conversion_GBps": round(conv_bytes / (u * 1e-3) / 1e9, 1),
            "conversion_share_of_3.35TBps": round(conv_bytes / (u * 1e-3) / (HBM_TBS * 1e12), 3),
            "all_ms": {k: [round(t, 3) for t in v] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["T1", "T2", "T3"], choices=["T1", "T2", "T3"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch

    import fpng_b200
    fpng_b200.fpng_init(0)
    name, power, sm, sm_max = card()
    for w in args.workload:
        r = run(w, args.rounds, args.iters)
        r.update({"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max, "rounds": args.rounds,
                  "iters_per_round": args.iters})
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
