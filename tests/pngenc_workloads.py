"""Seeded images for the PNG encode of gray, gray+alpha and 16-bit images (encode_png_device): the benchmark's workloads E1-E4
(tools/bench_png_encode.py) and the small corpus the tests compare the GPU with the oracle on.  One definition for both, so the
size bar the CPU test pins is the one the benchmark reports."""
from __future__ import annotations

import numpy as np


def label_mask(h, w, seed, labels=8, blobs=24):
    """A segmentation mask: background 0 and `blobs` overlapping ellipses of labels 1..labels-1."""
    rng = np.random.default_rng(seed)
    m = np.zeros((h, w), np.uint8)
    for _ in range(blobs):
        cy, cx = rng.integers(0, h), rng.integers(0, w)
        ry, rx = rng.integers(h // 16 + 1, h // 4 + 2), rng.integers(w // 16 + 1, w // 4 + 2)
        y0, y1, x0, x1 = max(cy - ry, 0), min(cy + ry + 1, h), max(cx - rx, 0), min(cx + rx + 1, w)
        yy, xx = np.ogrid[y0:y1, x0:x1]
        inside = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0
        m[y0:y1, x0:x1][inside] = rng.integers(1, labels)
    return m[..., None]


def depth_map(h, w, seed):
    """A 16-bit depth map in millimetres: a tilted plane with smooth relief, sensor noise and a near object with a sharp edge."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    ph = rng.uniform(0, 6.28)
    z = 2000 + 3 * yy + 1.5 * xx + 400 * np.sin(xx / 40 + ph) * np.cos(yy / 55) + rng.normal(0, 2, (h, w))
    cy, cx, r = rng.integers(h // 4, 3 * h // 4 + 1), rng.integers(w // 4, 3 * w // 4 + 1), max(min(h, w) // 6, 1)
    z[(xx - cx) ** 2 + (yy - cy) ** 2 < r * r] = 900
    return np.clip(z, 0, 65535).astype(np.uint16)[..., None]


def gradient_noise(h, w, seed):
    """8-bit gray: a diagonal gradient with +-3 noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    return np.clip((xx + yy) // 4 + rng.integers(-3, 4, (h, w)), 0, 255).astype(np.uint8)[..., None]


def rgba16(h, w, seed):
    """16-bit RGBA: colour gradients with +-40 noise and an opaque alpha channel."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([xx * 30, yy * 60, (xx + yy) * 15, np.full_like(xx, 65535)], -1)
    return np.clip(base + rng.integers(-40, 41, (h, w, 4)) * np.array([1, 1, 1, 0]), 0, 65535).astype(np.uint16)


# name: (image count, h, w, generator); image i of a workload is generator(h, w, seed=1000 * workload index + i)
WORKLOADS = {
    "E1": (256, 1024, 1024, label_mask),
    "E2": (256, 480, 640, depth_map),
    "E3": (128, 1080, 1920, gradient_noise),
    "E4": (64, 1080, 1920, rgba16),
}


def workload(name, count=None):
    """The first `count` images (all by default) of workload `name`, as [h, w, c] numpy arrays."""
    n, h, w, gen = WORKLOADS[name]
    k = list(WORKLOADS).index(name)
    return [gen(h, w, 1000 * k + i) for i in range(n if count is None else count)]


def corpus():
    """(name, image) pairs over the six formats of the new files: widths 1-33, one-row images, runs at and around
    floor(258 / B) pixels, smooth images (which take every filter), noise (which falls back to stored blocks)."""
    rng = np.random.default_rng(7)
    out = []
    for c, dt in ((1, np.uint8), (2, np.uint8), (1, np.uint16), (2, np.uint16), (3, np.uint16), (4, np.uint16)):
        B = c * np.dtype(dt).itemsize
        top = 256 if dt == np.uint8 else 65536
        tag = f"c{c}d{8 * np.dtype(dt).itemsize}"
        for w in range(1, 34):
            h = 1 + (w * 7) % 5
            out.append((f"{tag}_w{w}_levels", (rng.integers(0, 3, (h, w, c)) * (top // 3)).astype(dt)))
        out.append((f"{tag}_h1", rng.integers(0, 4, (1, 77, c)).astype(dt)))
        M = 258 // B
        for r in (M - 1, M, M + 1, 2 * M, 2 * M + 1, 3 * M - 1):
            row = np.zeros((3, r + 3, c), dt)
            row[:, 0] = 5
            row[:, r + 1:] = rng.integers(0, 200, (3, 2, c))
            row[1] += 1
            out.append((f"{tag}_run{r}", row))
        yy, xx = np.mgrid[0:40, 0:57]
        smooth = np.stack([(xx * 5 + yy * 3 + k * 11) % 256 for k in range(c)], -1) * (257 if dt == np.uint16 else 1)
        out.append((f"{tag}_smooth", smooth.astype(dt)))
        wave = np.stack([(128 + 100 * np.sin(xx / (5.0 + k) + yy / 7.0)) for k in range(c)], -1) * (257 if dt == np.uint16 else 1)
        out.append((f"{tag}_wave", wave.astype(dt)))
        out.append((f"{tag}_noise", rng.integers(0, top, (23, 31, c)).astype(dt)))
    return out
