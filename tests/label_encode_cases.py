"""Seeded corpus of label maps for the label-map PNG encode (fpngb_encode_label_ragged_device, DESIGN §4.6 "Label maps").  Each
case names the construct it reaches; tests/test_encode_labels_cpu.py checks with deflatetrace and PIL that the oracle's file for
it does reach that construct, and tests/test_encode_labels_gpu.py that the GPU writes the same bytes."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

FORCE_UNCOMPRESSED = 2


@dataclass
class Case:
    name: str
    ids: np.ndarray                 # [h, w] int64
    depth: int
    palette: np.ndarray | None      # uint8 [K, 3 | 4], None: gray
    flags: int = 0
    reaches: str = ""               # "residue", "stored", "forced", "trns-trimmed", "trns-present", "trns-absent", "K", "gray"


def voc_palette(k=256):
    """PASCAL VOC's colour map (the bit-interleaved one every VOC tool writes), first k entries"""
    pal = np.zeros((k, 3), np.uint8)
    for i in range(k):
        c, r, g, b = i, 0, 0, 0
        for j in range(8):
            r |= ((c >> 0) & 1) << (7 - j); g |= ((c >> 1) & 1) << (7 - j); b |= ((c >> 2) & 1) << (7 - j)
            c >>= 3
        pal[i] = (r, g, b)
    return pal


def blobs(rs, h, w, k):
    """a piecewise-constant map of k classes (compressible, like a segmentation)"""
    by, bx = max(1, h // 4), max(1, w // 5)
    coarse = rs.randint(0, k, size=((h + by - 1) // by, (w + bx - 1) // bx))
    return np.repeat(np.repeat(coarse, by, 0), bx, 1)[:h, :w].astype(np.int64)


def cases() -> list[Case]:
    rs = np.random.RandomState(2024)
    out = []
    # every w*d mod 8 residue, at each packed depth
    for d in (1, 2, 4):
        for w in range(8 // d, 2 * (8 // d)):
            out.append(Case(f"residue_d{d}_w{w}", blobs(rs, 300, w, 1 << d), d, None, reaches="residue"))
    # K across the depth boundaries of PIL's rule, RGB and RGBA palettes
    for k in (1, 2, 3, 4, 5, 16, 17, 256):
        d = 1 if k <= 2 else 2 if k <= 4 else 4 if k <= 16 else 8
        pal = rs.randint(0, 256, size=(k, 3)).astype(np.uint8)
        out.append(Case(f"K{k}_d{d}", blobs(rs, 37, 53, k), d, pal, reaches="K"))
    # tRNS: trimmed after the last non-opaque entry, present through the last entry, absent (opaque RGBA and RGB are covered above)
    pal = rs.randint(0, 256, size=(21, 4)).astype(np.uint8)
    pal[:, 3] = 255; pal[0, 3] = 0; pal[7, 3] = 128
    out.append(Case("trns_trimmed", blobs(rs, 40, 61, 21), 8, pal, reaches="trns-trimmed"))
    pal2 = pal.copy(); pal2[20, 3] = 3
    out.append(Case("trns_present", blobs(rs, 40, 61, 21), 8, pal2, reaches="trns-present"))
    pal3 = pal.copy(); pal3[:, 3] = 255
    out.append(Case("trns_absent_opaque_rgba", blobs(rs, 40, 61, 21), 8, pal3, reaches="trns-absent"))
    out.append(Case("voc_void", np.where(rs.rand(45, 70) < 0.1, 255, blobs(rs, 45, 70, 21)), 8, voc_palette(), reaches="K"))
    # stored: noise does not compress (fallback), and a compressible map with FPNGB_FORCE_UNCOMPRESSED
    out.append(Case("stored_fallback_d8", rs.randint(0, 256, size=(23, 97)).astype(np.int64), 8, None, reaches="stored"))
    out.append(Case("stored_fallback_d1", rs.randint(0, 2, size=(19, 300)).astype(np.int64), 1, None, reaches="stored"))
    out.append(Case("forced_d4_palette", blobs(rs, 30, 41, 16), 4, rs.randint(0, 256, (16, 4)).astype(np.uint8), FORCE_UNCOMPRESSED,
                    reaches="forced"))
    # gray at every depth, 16 bits included
    for d in (1, 2, 4, 8, 16):
        out.append(Case(f"gray_d{d}", blobs(rs, 29, 67, min(1 << d, 60000)) * (1 if d < 16 else 997) % (1 << d), d, None,
                        reaches="gray"))
    return out
