"""OpenAI CLIP's eval transform from packed PNG bytes: fpngb_decode_packed_views_device with interpolation="bicubic" against the
torch chain a caller runs without it, and against the same views call with bilinear interpolation (what bicubic costs).

Transform: Resize(224, BICUBIC, antialias=True) + CenterCrop(224) + Normalize(CLIP mean / std), bf16 NCHW output.
Workloads (those of bench_decode_views.py): M1, the 256 mixed files of bench_ragged_decode.py; C2, bench.py's 256 x 1920x1080
RGB batch packed by dist.compact.
Three arms, timed in alternating rounds:
  (a) decode_packed_views_device, resize_crop_views(info, 224, 224), interpolation="bicubic", every bound and pixel_cap given
      (no host synchronisation; the view table is built once);
  (b) the uint8 decode_packed_ragged_device, ragged_views (a read-back), then per file torchvision v2's resize(224, BICUBIC,
      antialias=True) and center_crop on the float image, the affine map and a cast into a preallocated NCHW batch;
  (c) (a) with interpolation="bilinear".
Times are host wall time per call ending in a device synchronise, medians over the rounds.  The largest difference between (a)
and (b) is reported on the 0-255 scale (torch's CUDA antialias kernel refuses some large downscales: such files are left out of
the comparison and counted).  Card name and power limit are read in the same run; one JSON line per workload.

    python tools/bench_decode_bicubic.py [--workload m1 c2] [--rounds 5] [--iters 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_decode_resized import c2_files, m1_files, packed  # noqa: E402
from bench_device_decode import card  # noqa: E402

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def timed(arms, rounds, iters):
    for fn in arms:
        fn()
    acc = [[] for _ in arms]
    for _ in range(rounds):
        for fn, a in zip(arms, acc):
            t0 = time.perf_counter()
            for _ in range(iters):
                fn()
            a.append((time.perf_counter() - t0) * 1e3 / iters)
    return acc


def run(name, files, rounds, iters):
    import torch
    import torchvision.transforms.v2.functional as F
    from torchvision.transforms import InterpolationMode

    import fpng_b200

    dev = torch.device("cuda", 0)
    data, offsets, sizes = packed(files, dev)
    info = fpng_b200.get_info_batch_device(data, offsets, sizes)
    dims = [(int(r[1]), int(r[2])) for r in info.cpu().numpy()]
    n, d, H, W = len(files), 3, 224, 224
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims),
                  pixel_cap=sum((w * h * d + 15) // 16 * 16 for w, h in dims))
    raw = torch.empty(bounds["pixel_cap"], dtype=torch.uint8, device=dev)
    rb = {k: v for k, v in bounds.items() if k != "pixel_cap"}
    views = fpng_b200.resize_crop_views(info, 224, 224)
    s, b = fpng_b200.normalize_scale_bias(CLIP_MEAN, CLIP_STD)
    st_, bt_ = torch.from_numpy(s).to(dev).view(3, 1, 1), torch.from_numpy(b).to(dev).view(3, 1, 1)
    out_a = torch.empty((n, d, H, W), dtype=torch.bfloat16, device=dev).permute(0, 2, 3, 1)
    out_b = torch.empty((n, d, H, W), dtype=torch.bfloat16, device=dev)
    out_c = torch.empty((n, d, H, W), dtype=torch.bfloat16, device=dev).permute(0, 2, 3, 1)
    kw = dict(dtype=torch.bfloat16, scale=s, bias=b, antialias=True)
    refused = set()

    def arm_a():
        fpng_b200.decode_packed_views_device(data, offsets, sizes, views, (H, W), d, out=out_a, interpolation="bicubic", **kw, **bounds)
        torch.cuda.synchronize()

    def arm_c():
        fpng_b200.decode_packed_views_device(data, offsets, sizes, views, (H, W), d, out=out_c, interpolation="bilinear", **kw, **bounds)
        torch.cuda.synchronize()

    def arm_b():
        px, oo, inf, st = fpng_b200.decode_packed_ragged_device(data, offsets, sizes, d, out=raw, **rb)
        for i, v in enumerate(fpng_b200.ragged_views(px, oo, inf, st, d)):
            try:
                x = F.center_crop(F.resize(v.permute(2, 0, 1).float(), 224, InterpolationMode.BICUBIC, antialias=True), [224, 224])
            except RuntimeError as e:                           # torch's CUDA antialias kernel refuses large downscales
                assert "shared memory" in str(e), e
                refused.add(i)
                continue
            out_b[i] = (x * st_ + bt_).to(torch.bfloat16)
        torch.cuda.synchronize()

    ta, tb, tc = timed([arm_a, arm_b, arm_c], rounds, iters)
    keep = [i for i in range(n) if i not in refused]
    to_255 = lambda t: (t.double() - bt_.double()) / st_.double()  # noqa: E731
    diff = float((to_255(out_a.permute(0, 3, 1, 2)[keep]) - to_255(out_b[keep])).abs().max())
    gpu, power = card()
    med = statistics.median
    return {"workload": name, "files": n, "canvas": [H, W], "dtype": "bfloat16",
            "a_views_bicubic_ms": med(ta), "a_min_max": [min(ta), max(ta)],
            "b_torch_chain_bicubic_ms": med(tb), "b_min_max": [min(tb), max(tb)],
            "c_views_bilinear_ms": med(tc), "c_min_max": [min(tc), max(tc)],
            "speedup_b_over_a": med(tb) / med(ta), "bicubic_over_bilinear": med(ta) / med(tc),
            "max_abs_diff_a_b_0_255": diff, "files_torch_refused": len(refused), "gpu": gpu, "power_limit": power}


def main():
    import torch

    import fpng_b200
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--workload", nargs="+", default=["m1", "c2"], choices=["m1", "c2"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    fpng_b200.fpng_init(0)
    dev = torch.device("cuda", 0)
    for w in a.workload:
        files = m1_files(dev) if w == "m1" else c2_files(dev)
        print(json.dumps(run(w.upper(), files, a.rounds, a.iters)), flush=True)


if __name__ == "__main__":
    main()
