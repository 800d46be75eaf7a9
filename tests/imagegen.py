"""Synthetic image generators shared by tests/ and bench.py (SURVEY.md section 8d).

G0 "gradient":        R = floor(255 x/(w-1)), G = floor(255 y/(h-1)), B = (x + y + i) & 255, A = G   (fpng_test -a swizzle,
                      src/fpng_test.cpp:1147-1152); RLE-dominated, out/in ~ 0.006.
G1 "gradient+noise":  G0 + per-channel uniform integer noise in [-3, 3] (MT19937, seed 1234 + i); literal-dominated,
                      out/in ~ 0.55-0.6.
G2 "random":          uniform bytes (MT19937); always lands on the stored-block fallback.
U<k> "uniform deltas": Up-filtered bytes uniform over k values; near-fixed-length Huffman codes when encoded 2-pass.
plus the mutation families of the reference's encoder fuzzers (src/fpng_test.cpp:381-615): colour runs, byte fills.
"""
from __future__ import annotations

import numpy as np


def gradient(w: int, h: int, chans: int, index: int = 0) -> np.ndarray:
    x = np.arange(w, dtype=np.int64)[None, :]
    y = np.arange(h, dtype=np.int64)[:, None]
    r = (255 * x) // max(w - 1, 1) + 0 * y
    g = (255 * y) // max(h - 1, 1) + 0 * x
    b = (x + y + index) & 255
    planes = [r, g, b] + ([g] if chans == 4 else [])
    return np.stack(planes, axis=-1).astype(np.uint8)


def gradient_noise(w: int, h: int, chans: int, index: int = 0, amp: int = 3) -> np.ndarray:
    rs = np.random.RandomState(1234 + index)
    base = gradient(w, h, chans, index).astype(np.int16)
    noise = rs.randint(-amp, amp + 1, size=base.shape).astype(np.int16)
    return ((base + noise) & 255).astype(np.uint8)


def random_bytes(w: int, h: int, chans: int, index: int = 0) -> np.ndarray:
    rs = np.random.RandomState(4321 + index)
    return rs.randint(0, 256, size=(h, w, chans), dtype=np.uint8)


def colour_runs(w: int, h: int, chans: int, seed: int = 0, max_run: int = 400) -> np.ndarray:
    """Random-length runs of one colour (exercises run splitting at 85/63 pixels and row boundaries)."""
    rs = np.random.RandomState(seed)
    img = np.empty((h * w, chans), dtype=np.uint8)
    i = 0
    while i < h * w:
        n = int(rs.randint(1, max_run))
        img[i:i + n] = rs.randint(0, 256, size=(chans,), dtype=np.uint8)
        i += n
    return img.reshape(h, w, chans)


def mutated(w: int, h: int, chans: int, seed: int) -> np.ndarray:
    """Gradient+noise with fills, xors and bit flips in the spirit of fuzz_test_encoder (src/fpng_test.cpp:381-615)."""
    rs = np.random.RandomState(seed)
    img = gradient_noise(w, h, chans, seed, amp=int(rs.randint(0, 4))).reshape(-1)
    for _ in range(int(rs.randint(1, 12))):
        kind = rs.randint(0, 4)
        pos = int(rs.randint(0, img.size))
        n = int(rs.randint(1, 259))
        if kind == 0:
            img[pos:pos + n] = rs.randint(0, 256)
        elif kind == 1:
            img[pos:pos + n] ^= np.uint8(rs.randint(1, 256))
        elif kind == 2:
            px = (pos // chans) * chans
            img[px:px + n * chans] = np.tile(rs.randint(0, 256, size=(chans,), dtype=np.uint8), n)[: max(0, min(n * chans, img.size - px))]
        else:
            img[pos] ^= np.uint8(1 << int(rs.randint(0, 8)))
    return img.reshape(h, w, chans)


KINDS = {"g0": gradient, "g1": gradient_noise, "g2": random_bytes}


def uniform_deltas(w: int, h: int, chans: int, k: int, index: int = 0) -> np.ndarray:
    """Image whose Up-filtered bytes are uniform over 0..k-1 (MT19937, seed 5678 + i): noisy low-bit-depth content.  Its
    2-pass Huffman table is close to a fixed-length code, which hardly resynchronises after a wrong start: the decoder's
    speculative subsequence starts (decode_scan_kernel) are mostly wrong and the link pass repairs them in chains."""
    rs = np.random.RandomState(5678 + index)
    return from_deltas(rs.randint(0, k, size=(h, w, chans)))


def make(kind: str, w: int, h: int, chans: int, index: int = 0) -> np.ndarray:
    if kind in KINDS:
        return KINDS[kind](w, h, chans, index)
    if kind[:1] == "u" and kind[1:].isdigit():                    # "u128", "u64", "u16", "u2"
        return uniform_deltas(w, h, chans, int(kind[1:]), index)
    if kind == "runs":
        return colour_runs(w, h, chans, index)
    if kind == "mut":
        return mutated(w, h, chans, index)
    if kind == "zero":
        return np.zeros((h, w, chans), np.uint8)
    raise KeyError(kind)


def from_deltas(delta: np.ndarray) -> np.ndarray:
    """Image whose Up-filtered rows (row 0: raw) equal `delta` (h, w, chans): running byte-wise sum down the rows."""
    return (np.cumsum(delta.astype(np.uint32), axis=0) & 255).astype(np.uint8)


def short_runs(w: int, h: int, chans: int, seed: int, palette) -> np.ndarray:
    """Filtered-domain pixels drawn channel-wise from `palette` with many runs of exactly 1-3 equal pixels: exercises the
    RGBA 1-pass "one-pixel match vs four literals" decision (src/fpng.cpp:1520-1528) in both directions."""
    rs = np.random.RandomState(seed)
    pal = np.asarray(palette, dtype=np.uint8)
    d = pal[rs.randint(0, len(pal), size=(h, w, chans))]
    rep = rs.rand(h, w) < 0.45
    for y in range(h):
        for x in range(1, w):
            if rep[y, x]:
                d[y, x] = d[y, x - 1]
    return from_deltas(d)


def trained_table_images(chans: int, sizes):
    """The fixed image set of tests/golden/trained_tables.json (name, w, h, pixels), built from the table's code sizes so
    that cheap and expensive literals both occur next to one-pixel matches."""
    order = np.argsort(np.asarray(sizes)[:256], kind="stable")
    cheap = [int(v) for v in order[:5]]
    pal_mixed = cheap + [int(order[40]), int(order[200])]
    out = []
    for i, (w, h, pal) in enumerate([(64, 20, cheap[:2]), (257, 9, cheap), (96, 33, pal_mixed), (16, 5, cheap[:1]), (130, 12, pal_mixed)]):
        out.append((f"short_runs_{i}", w, h, short_runs(w, h, chans, 100 + i, pal)))
    out.append(("g1", 128, 16, make("g1", 128, 16, chans, 3)))
    out.append(("runs", 200, 11, make("runs", 200, 11, chans, 5)))
    out.append(("zero", 70, 7, make("zero", 70, 7, chans, 0)))
    return out
