"""Strided device tensors: encode from NCHW planes and crops, decode into NCHW, against the copies callers make without them.

The images are bench.py's synthetic batch (same generator).  Arms, timed alternately in one process with CUDA events around
`--iters` back-to-back calls on the current stream (no host work inside the window):
  encode (a) contiguous NHWC, as bench.py;
         (b) NCHW source: permute(0, 2, 3, 1).contiguous() then encode -- what a caller had to do before strided input;
         (c) NCHW source encoded in place (planar loader);
         (d) a crop of a canvas 32 pixels wider, at a 16-byte aligned x offset (staged loaders) and at x offset 3 (direct
             loader);
  decode (e) decode_packed_device into contiguous NHWC;
         (f) (e) followed by permute(0, 3, 1, 2).contiguous() -- NCHW the old way;
         (g) decode_packed_device straight into an NCHW tensor.
Every encode arm's files are compared byte for byte with arm (a), (g) with (f), (e) with the input.  Prints one JSON line
per workload with the card's name and power limit, read in the same run.

    python tools/bench_strided.py [--workload c2 c3] [--rounds 5] [--iters 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

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


def run(wl_key: str, rounds: int, iters: int) -> dict:
    import torch

    import bench
    import fpng_b200

    wl = bench.WORKLOADS[wl_key]
    w, h, c, n, flags = wl["w"], wl["h"], wl["chans"], wl["images"], wl["flags"]
    dev = torch.device("cuda", 0)
    nhwc = bench.make_device_batch(wl, "g1", n, dev)
    nchw = nhwc.permute(0, 3, 1, 2).contiguous()
    canvas = torch.zeros((n, h, w + 32, c), dtype=torch.uint8, device=dev)
    canvas[:, :, 16:16 + w] = nhwc
    crop16 = canvas[:, :, 16:16 + w]
    crop3 = torch.zeros((n, h, w + 32, c), dtype=torch.uint8, device=dev)
    crop3[:, :, 3:3 + w] = nhwc
    crop3 = crop3[:, :, 3:3 + w]
    del canvas
    stride = (fpng_b200.max_encoded_size(w, h, c) + 15) // 16 * 16
    outs = {k: (torch.empty((n, stride), dtype=torch.uint8, device=dev), torch.empty((n,), dtype=torch.int32, device=dev))
            for k in ("a", "b", "c", "d16", "d3")}

    def enc(key, src):
        return lambda: fpng_b200.encode_batch_device(src, flags, out=outs[key][0], sizes=outs[key][1])

    arms = {
        "a_nhwc": enc("a", nhwc),
        "b_nchw_copy_then_encode": lambda: fpng_b200.encode_batch_device(nchw.permute(0, 2, 3, 1).contiguous(), flags,
                                                                         out=outs["b"][0], sizes=outs["b"][1]),
        "c_nchw_in_place": enc("c", nchw.permute(0, 2, 3, 1)),
        "d_crop_x16": enc("d16", crop16),
        "d_crop_x3": enc("d3", crop3),
    }
    # decode of arm (a)'s files, packed at the encode stride
    for f in arms.values():
        f()
    torch.cuda.synchronize()
    files, sizes = outs["a"]
    flat = files.view(-1)
    offsets = torch.arange(n, device=dev, dtype=torch.int64) * stride
    px_e = torch.empty((n, h, w, c), dtype=torch.uint8, device=dev)
    st = torch.empty((n,), dtype=torch.int32, device=dev)
    px_g = torch.empty((n, c, h, w), dtype=torch.uint8, device=dev)
    holder = {}

    def dec_e():
        fpng_b200.decode_packed_device(flat, offsets, sizes, w, h, c, c, out=px_e, status=st)

    def dec_f():
        fpng_b200.decode_packed_device(flat, offsets, sizes, w, h, c, c, out=px_e, status=st)
        holder["f"] = px_e.permute(0, 3, 1, 2).contiguous()

    def dec_g():
        fpng_b200.decode_packed_device(flat, offsets, sizes, w, h, c, c, out=px_g.permute(0, 2, 3, 1), status=st)

    arms.update({"e_decode_nhwc": dec_e, "f_decode_nhwc_then_permute": dec_f, "g_decode_nchw_in_place": dec_g})

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    for fn in arms.values():                                          # warm-up
        fn(); fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for r in range(rounds):                                           # alternating arms, order rotated every round
        keys = list(arms)
        keys = keys[r % len(keys):] + keys[: r % len(keys)]
        for k in keys:
            ms[k].append(timed(arms[k]))

    # correctness, after a fresh run of every arm
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    mask = torch.arange(stride, device=dev)[None, :] < (sizes.to(torch.int64) & 0xFFFFFFFF)[:, None]

    def same_files(key):
        o, s = outs[key]
        return bool(torch.equal(s, sizes)) and bool(torch.equal(torch.where(mask, o, 0), torch.where(mask, files, 0)))

    dec_e(); dec_f(); dec_g()
    torch.cuda.synchronize()
    checks = {
        "b_files_equal_a": same_files("b"), "c_files_equal_a": same_files("c"),
        "d_x16_files_equal_a": same_files("d16"), "d_x3_files_equal_a": same_files("d3"),
        "e_equals_input": bool(torch.equal(px_e, nhwc)) and bool((st == 0).all().item()),
        "g_equals_f": bool(torch.equal(px_g, holder["f"])),
    }
    name, power = card()
    summary = {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in ms.items()}
    return {
        "workload": wl["name"], "kind": "g1", "images": n, "card": name, "power_limit": power,
        "ms_per_call": summary, "checks": checks,
        "c_over_b": statistics.median(ms["c_nchw_in_place"]) / statistics.median(ms["b_nchw_copy_then_encode"]),
        "g_over_f": statistics.median(ms["g_decode_nchw_in_place"]) / statistics.median(ms["f_decode_nhwc_then_permute"]),
        "rounds": rounds, "iters_per_round": iters,
        "timing": "CUDA events around iters back-to-back calls on the current stream, per call",
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["c2", "c3"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_strided: no CUDA device")
    import fpng_b200
    fpng_b200.fpng_init(0)
    for k in args.workload:
        print(json.dumps(run(k, args.rounds, args.iters)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
