"""Test-side numpy model of the colour-type reduction rule of encode_png_device(reduce=True) (include/fpng_b200.h,
FPNGB_ENCODE_REDUCE; DESIGN §4.6 "Colour-type reduction"), written from the rule: the image's properties, the chosen format, the
palette order, and the existing call whose file the reduced file equals.  Only the tests and tools/bench scripts import it."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

FORMATS = ("gray", "palette", "ga", "rgb", "rgba")          # the rule's tie order


def pil_depth(k: int) -> int:
    return 1 if k <= 2 else 2 if k <= 4 else 4 if k <= 16 else 8


def hash_slot(key: int) -> int:
    """the slot of colour key R << 24 | G << 16 | B << 8 | A in the kernels' 512-slot sets (reduce_kernels.cu)"""
    return ((key * 0x9E3779B1) & 0xFFFFFFFF) >> 23


@dataclass
class Analysis:
    rep8: bool
    opaque: bool
    gray: bool
    lattice: int | None        # d in {1, 2, 4, 8} for a gray-valued, opaque, 8-bit representable image
    colours: np.ndarray | None  # uint32 [K] keys, None for more than 256


def analyse(img: np.ndarray) -> Analysis:
    """img: [h, w, c] uint8 or uint16"""
    a = np.asarray(img)
    c = a.shape[2]
    rep8 = a.dtype == np.uint8 or bool((a.astype(np.uint32) % 257 == 0).all())
    amax = 255 if a.dtype == np.uint8 else 65535
    opaque = c in (1, 3) or bool((a[..., c - 1] == amax).all())
    gray = c <= 2 or bool(((a[..., 0] == a[..., 1]) & (a[..., 0] == a[..., 2])).all())
    v8 = a.astype(np.uint32) if a.dtype == np.uint8 else a.astype(np.uint32) // 257
    lattice = None
    if gray and opaque and rep8:
        g = v8[..., 0]
        lattice = next(d for d in (1, 2, 4, 8) if (g % (255 // ((1 << d) - 1)) == 0).all())
    colours = None
    if rep8:
        r = v8[..., 0]
        gg, b = (r, r) if c <= 2 else (v8[..., 1], v8[..., 2])
        al = v8[..., c - 1] if c in (2, 4) else np.full_like(r, 255)
        keys = np.unique((r << 24 | gg << 16 | b << 8 | al).reshape(-1).astype(np.uint32))
        colours = keys if len(keys) <= 256 else None
    return Analysis(rep8, opaque, gray, lattice, colours)


def choose(img: np.ndarray):
    """(format, bits per pixel, sample depth) the rule picks: gray (depth d or 16), palette (depth p(K)), ga, rgb, rgba"""
    an = analyse(img)
    D = 8 if an.rep8 else 16
    cands = []
    if an.gray and an.opaque:
        cands.append(("gray", an.lattice, an.lattice) if an.rep8 else ("gray", 16, 16))
    if an.rep8 and an.colours is not None:
        p = pil_depth(len(an.colours))
        cands.append(("palette", p, p))
    if an.gray:
        cands.append(("ga", 2 * D, D))
    if an.opaque:
        cands.append(("rgb", 3 * D, D))
    cands.append(("rgba", 4 * D, D))
    return min(cands, key=lambda t: (t[1], FORMATS.index(t[0])))


def palette_order(keys: np.ndarray) -> np.ndarray:
    """the palette as uint8 [K, 4] RGBA: alpha below 255 first ascending by key, then the opaque ones ascending by RGB"""
    k = np.asarray(keys, dtype=np.uint64)
    order = np.lexsort((k, (k & 0xFF) == 0xFF))
    k = k[order].astype(np.uint32)
    return np.stack([(k >> 24) & 0xFF, (k >> 16) & 0xFF, (k >> 8) & 0xFF, k & 0xFF], axis=1).astype(np.uint8)


def reduced_call(img: np.ndarray):
    """The existing call whose file equals the reduced file: ("labels", ids [h, w] uint8, palette [K, 4] or None, depth) or
    ("png", reduced [h, w, c'] uint8 / uint16 array)."""
    a = np.asarray(img)
    c = a.shape[2]
    fmt, bits, depth = choose(a)
    v = a if depth == 16 else (a if a.dtype == np.uint8 else (a.astype(np.uint32) // 257).astype(np.uint8))
    if fmt == "palette":
        an = analyse(a)
        pal = palette_order(an.colours)
        v8 = v.astype(np.uint32)
        r = v8[..., 0]
        g, b = (r, r) if c <= 2 else (v8[..., 1], v8[..., 2])
        al = v8[..., c - 1] if c in (2, 4) else np.full_like(r, 255)
        key = r << 24 | g << 16 | b << 8 | al
        pk = pal.astype(np.uint32)
        pkeys = pk[:, 0] << 24 | pk[:, 1] << 16 | pk[:, 2] << 8 | pk[:, 3]
        order = np.argsort(pkeys)
        ids = order[np.searchsorted(pkeys[order], key)].astype(np.uint8)
        return ("labels", ids, pal, depth)
    if fmt == "gray" and depth < 8:
        return ("labels", (v[..., 0] // (255 // ((1 << depth) - 1))).astype(np.uint8), None, depth)
    chans = {"gray": [0], "ga": [0, c - 1], "rgb": [0, 1, 2], "rgba": [0, 1, 2, 3]}[fmt]
    return ("png", np.ascontiguousarray(v[..., chans]))

