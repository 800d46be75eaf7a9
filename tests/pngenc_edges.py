"""Seeded edge images for the PNG encode of gray, gray+alpha and 16-bit images (encode_png_device, DESIGN §4.6).  Each image
names the construct of the encoder it exists to reach:

- stored:  stored-block files (FORCE_UNCOMPRESSED, and the natural fallback on noise) whose filtered stream spans at least three
           65535-byte blocks, with block boundaries on a row's filter byte, between the two bytes of a 16-bit sample and between
           two channels of a pixel, plus streams of exactly k * 65535 and k * 65535 + 1 bytes;
- tie:     a one-parameter family per class (a smooth image whose first k pixels are noise) around the k where the file turns
           from compressed to stored, including a member whose compressed zlib stream is exactly the stored one's length;
- wide:    rows of 32 * 37 + r pixels for every r in 0..31, with runs across 32-pixel steps and around floor(258 / B) pixels;
- limit:   the 2^24 width and height limits.

tests/test_encode_png_edges_cpu.py shows that the oracle's files really contain each construct; tests/test_encode_png_edges_gpu.py
holds the GPU's files to the oracle's."""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

BLOCK = 65535
FORCE_UNCOMPRESSED = 2

# name, channels, dtype: the six classes of the PNG row kernels
CLASSES = (("gray8", 1, np.uint8), ("ga8", 2, np.uint8), ("gray16", 1, np.uint16), ("ga16", 2, np.uint16),
           ("rgb16", 3, np.uint16), ("rgba16", 4, np.uint16))


@dataclass
class Edge:
    name: str
    img: np.ndarray                      # [h, w, c] uint8 / uint16
    flags: tuple                         # the flag values the image is encoded with
    construct: set = field(default_factory=set)
    expand: bool = False                 # every row is row 0: the GPU tests read it through expand (row stride 0)
    k: int = -1                          # tie: the number of noise pixels

    @property
    def B(self) -> int:
        return self.img.shape[2] * self.img.dtype.itemsize


def top(dt) -> int:
    return 256 if np.dtype(dt) == np.uint8 else 65536


def noise(rng, h, w, c, dt) -> np.ndarray:
    return rng.integers(0, top(dt), (h, w, c)).astype(dt)


def raw_size(w, h, B) -> int:
    """bytes of the filtered stream: a filter byte and w * B pixel bytes per row"""
    return (w * B + 1) * h


def zstored(w, h, B) -> int:
    raw = raw_size(w, h, B)
    return 2 + raw + 5 * ((raw + BLOCK - 1) // BLOCK) + 4


def boundary_kinds(w, h, c, es) -> set:
    """Where the stored-block boundaries (stream offsets 65535 k) fall in the filtered stream: 'filter' (a block starts with a
    row's filter byte), 'sample' (between the high and low byte of a 16-bit sample), 'channel' (between two channels of one
    pixel), 'pixel' (between two pixels); 'exact' for a stream of k * 65535 bytes, 'plus1' for k * 65535 + 1."""
    B = c * es
    n, raw = w * B + 1, raw_size(w, h, B)
    kinds = set()
    for s in range(BLOCK, raw, BLOCK):
        t = s % n
        if t == 0:
            kinds.add("filter")
            continue
        j = (t - 1) % B
        kinds.add("pixel" if j == 0 else ("sample" if es == 2 and j % 2 else "channel"))
    if raw % BLOCK == 0:
        kinds.add("exact")
    if raw % BLOCK == 1:
        kinds.add("plus1")
    return kinds


def _stored_shape(B, c, es, kind):
    """The smallest (w, h) from w = 61 up whose stream spans at least three blocks and has a boundary of `kind`."""
    for w in range(61, 1000):
        n = w * B + 1
        h0 = 2 * BLOCK // n + 1
        for h in range(h0, h0 + 16):
            if kind in boundary_kinds(w, h, c, es):
                return w, h
    raise AssertionError(kind)


def _plus1_shape(B):
    """(w, h) with a stream of k * 65535 + 1 bytes, k >= 3, smallest stream first."""
    best = None
    for w in range(1, 2000):
        n = w * B + 1
        for k in range(3, 64):
            if (k * BLOCK + 1) % n == 0 and (best is None or k < best[0]):
                best = (k, w, (k * BLOCK + 1) // n)
    return best[1], best[2]


def _exact_shape(B):
    """(w, h) with a stream of exactly 3 * 65535 bytes: 65535 = 3 * 5 * 17 * 257, and the row length w * B + 1 divides it."""
    for d in (257, 1285, 85, 771, 255, 51):
        if (d - 1) % B == 0:
            return (d - 1) // B, 3 * BLOCK // d
    raise AssertionError(B)


def stored_edges() -> list[Edge]:
    out = []
    rng = np.random.default_rng(2024)
    for name, c, dt in CLASSES:
        es = np.dtype(dt).itemsize
        B = c * es
        kinds = ["filter"] + (["sample"] if es == 2 else []) + (["channel"] if c > 1 else [])
        shapes = {k: _stored_shape(B, c, es, k) for k in kinds}
        shapes["exact"], shapes["plus1"] = _exact_shape(B), _plus1_shape(B)
        for kind, (w, h) in shapes.items():
            got = boundary_kinds(w, h, c, es)
            assert kind in got and raw_size(w, h, B) > 2 * BLOCK, (name, kind, w, h)
            out.append(Edge(f"stored_{name}_{kind}_{w}x{h}", noise(rng, h, w, c, dt), (0, FORCE_UNCOMPRESSED), {"stored"} | got))
        w, h = shapes["filter"]                                       # expand: one noise row repeated, so only forced stored
        row = noise(rng, 1, w, c, dt)
        out.append(Edge(f"stored_{name}_expand_{w}x{h}", np.repeat(row, h, axis=0), (FORCE_UNCOMPRESSED,),
                        {"stored"} | boundary_kinds(w, h, c, es), expand=True))
    return out


# ---- tie -------------------------------------------------------------------------------------------------------------------
TIE_H, TIE_W = 24, 40


def tie_image(c, dt, seed, k) -> np.ndarray:
    """A smooth image whose first k pixels in raster order are seeded noise."""
    yy, xx = np.mgrid[0:TIE_H, 0:TIE_W]
    img = np.stack([(xx // 3 + yy // 2 + 7 * j) % 256 for j in range(c)], -1) * (257 if np.dtype(dt) == np.uint16 else 1)
    img = img.astype(dt)
    flat = img.reshape(-1, c)
    flat[:k] = noise(np.random.default_rng(seed), TIE_H * TIE_W, 1, c, dt)[:k, 0]
    return img


def idat_info(png: bytes):
    """(zlib stream length, BTYPE of its first block) of a file of encode_png_device"""
    return struct.unpack(">I", png[33:37])[0], (png[43] >> 1) & 3


def tie_edges(oracle) -> list[Edge]:
    """Per class, bisect k to the last compressed member k* (k* + 1 is stored) and keep k* - 1 .. k* + 2.  Seeds are tried in
    order until k* is an exact tie (compressed stream length == stored length), which the rule zcomp <= zstored compresses."""
    out = []
    for name, c, dt in CLASSES:
        B = c * np.dtype(dt).itemsize
        zst = zstored(TIE_W, TIE_H, B)
        for seed in range(64):
            def btype(k):
                return idat_info(oracle.png_encode(tie_image(c, dt, seed, k)))[1]
            lo, hi = 0, TIE_H * TIE_W
            assert btype(lo) == 2 and btype(hi) == 0, (name, seed)
            while hi - lo > 1:
                m = (lo + hi) // 2
                lo, hi = (m, hi) if btype(m) == 2 else (lo, m)
            if idat_info(oracle.png_encode(tie_image(c, dt, seed, lo)))[0] == zst:
                break
        else:
            raise AssertionError(f"no exact tie for {name}")
        for k in range(lo - 1, lo + 3):
            tag = {lo: "tie", lo + 1: "first_stored"}.get(k, "near")
            out.append(Edge(f"tie_{name}_s{seed}_k{k}_{tag}", tie_image(c, dt, seed, k), (0,), {tag}, k=k))
    return out


# ---- wide rows -------------------------------------------------------------------------------------------------------------
def wide_image(c, dt, w, seed) -> np.ndarray:
    """Three rows of w pixels.  Row 0: runs that start at lane 31 of one 32-pixel step and end at lane 0 of a later one, runs
    of about floor(258 / B) * m +- 1 pixels (m = 1, 2) and a run to the end of the row, between noise pixels; row 1: noise;
    row 2: back-to-back runs of about floor(258 / B) * m +- 1 pixels, the last one cut by the row's end.  The noise has four
    levels, so that the files compress."""
    B = c * np.dtype(dt).itemsize
    M = 258 // B
    rng = np.random.default_rng(seed)
    img = (rng.integers(0, 4, (3, w, c)) * (top(dt) // 4 + 3)).astype(dt)   # 4-level noise: compressed files with flags 0
    val = noise(rng, 64, 1, c, dt)[:, 0]
    row = img[0]
    x, v = 0, 0
    # raw runs from lane 31 (filter 0) or lane 30 (sub, whose run of equal filtered pixels starts one later) to lane 0
    for lane, span in ((31, 34), (30, 35), (31, 66), (30, 67), (31, 2), (30, 3)):
        x += (lane - x) % 32
        row[x:x + span] = val[v]; v += 1
        x += span + 32
    # floor(258 / B) * m +- 1 pixels, raw and one longer (the run of equal sub-filtered pixels is one shorter)
    for L in (M - 1, M + 1, 2 * M - 1, 2 * M + 1, M, M + 2, 2 * M, 2 * M + 2):
        if x + L + 2 > w - 40:
            break
        row[x:x + L] = val[v]; v += 1
        x += L + 3
    row[w - 37:] = val[v]; v += 1                                  # a run that the row's last, partial step ends
    x, i, lens = 0, 0, (M - 1, 2 * M + 1, M + 1, 2 * M - 1, M, 2 * M + 2, M + 2, 2 * M)
    while x < w:
        L = lens[i % len(lens)]; i += 1
        img[2, x:x + L] = val[v % len(val)]; v += 1
        x += L
    return img


WIDE_BASE = 32 * 37


def wide_edges() -> list[Edge]:
    out = []
    for ci, (name, c, dt) in enumerate(CLASSES):
        for r in range(32):
            w = WIDE_BASE + r
            out.append(Edge(f"wide_{name}_w{w}", wide_image(c, dt, w, 100 * ci + r), (0, FORCE_UNCOMPRESSED), {f"residue{r}"}))
    return out


# ---- dimension limits ------------------------------------------------------------------------------------------------------
LIMIT = 1 << 24


def runs_image(h, w, c, dt, seed, run=300) -> np.ndarray:
    """An image whose raster order is runs of `run` equal pixels with seeded values, each tenth run noise instead."""
    rng = np.random.default_rng(seed)
    n = h * w
    vals = noise(rng, n // run + 1, 1, c, dt)[:, 0]
    px = np.repeat(vals, run, axis=0)[:n]
    idx = np.arange(n) // run
    sel = idx % 10 == 9
    px[sel] = noise(rng, int(sel.sum()), 1, c, dt)[:, 0]
    return px.reshape(h, w, c)


def limit_edges() -> list[Edge]:
    """gray8 1 x 2^24 and 2^24 x 1, gray16 1 x 2^24, RGBA16 2^24 x 1 (one 128 MiB row), all with runs."""
    return [
        Edge("limit_gray8_tall", runs_image(LIMIT, 1, 1, np.uint8, 1), (0,), {"tall"}),
        Edge("limit_gray8_wide", runs_image(1, LIMIT, 1, np.uint8, 2), (0,), {"wide"}),
        Edge("limit_gray16_tall", runs_image(LIMIT, 1, 1, np.uint16, 3), (0,), {"tall"}),
        Edge("limit_rgba16_wide", runs_image(1, LIMIT, 4, np.uint16, 4), (0,), {"wide"}),
    ]


# ---- past 32 bits ----------------------------------------------------------------------------------------------------------
BIG_H, BIG_W = 8192, 16384


def big_rgba16(h=BIG_H, seed=5) -> np.ndarray:
    """RGBA16 16384 x 8192 (1 GiB): smooth high bytes and noise low bytes, so the file stays compressed (the high bytes filter
    to runs of zeros) with a zlib stream past 2^29 bytes (the noise bytes cost 8 bits and more), where bit offsets pass 2^32."""
    rng = np.random.default_rng(seed)
    img = np.empty((h, BIG_W, 4), np.uint16)
    xx = np.arange(BIG_W, dtype=np.uint16)
    for y0 in range(0, h, 512):
        yy = np.arange(y0, y0 + 512, dtype=np.uint16)[:, None]
        for j in range(4):
            hi = ((xx[None] // 64 + yy // 32 + 40 * j) & 0xFF) << 8
            img[y0:y0 + 512, :, j] = hi | rng.integers(0, 256, (512, BIG_W), dtype=np.uint16)
    return img
