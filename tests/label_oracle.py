"""Test-only oracle of the label-map PNG files fpngb_encode_label_ragged_device writes (DESIGN §4.6 "Label maps"), written from
the format rules on top of the gray8 / gray16 PNG oracle (oracle/pngenc_oracle.py): pack the ids into row bytes, encode those
rows with that oracle, then put IHDR, PLTE and tRNS in front of its IDAT.  Only the tests and tools/bench scripts import it."""
from __future__ import annotations

import numpy as np


class LabelOracle:
    def __init__(self):
        from oracle.pngenc_oracle import PngEncodeOracle
        self.png = PngEncodeOracle()

    def label_encode(self, ids, depth, palette=None, flags=0):
        """The file fpngb_encode_label_ragged_device writes for ids, an [h, w] integer array, at `depth` bits (gray when palette
        is None, else a uint8 [K, 3 | 4] palette), written from the format rules of DESIGN §4.6 "Label maps": pack the rows,
        encode them with png_encode as a gray8 image ceil(w * depth / 8) wide (gray16 for depth 16), then put IHDR, PLTE and
        tRNS in front of that file's IDAT.  None when an id is out of range (the GPU call's size 0)."""
        a = np.asarray(ids).astype(np.int64)
        assert a.ndim == 2, a.shape
        h, w = a.shape
        limit = (1 << depth) if palette is None else len(palette)
        if a.size and (a.min() < 0 or a.max() >= limit):
            return None
        if depth == 16:
            packed = a.astype(np.uint16).reshape(h, w, 1)
        else:
            per = 8 // depth
            pad = (-w) % per
            v = np.concatenate([a, np.zeros((h, pad), np.int64)], axis=1).reshape(h, -1, per)
            shifts = np.array([8 - depth * (k + 1) for k in range(per)], dtype=np.int64)
            packed = (v << shifts).sum(axis=2).astype(np.uint8).reshape(h, -1, 1)
        body = self.png.png_encode(packed, flags)[33:]                   # the IDAT chunk and IEND of the packed rows
        chunks = [label_chunk(b"IHDR", w.to_bytes(4, "big") + h.to_bytes(4, "big") +
                              bytes([depth, 0 if palette is None else 3, 0, 0, 0]))]
        if palette is not None:
            pal = np.asarray(palette, dtype=np.uint8)
            chunks.append(label_chunk(b"PLTE", pal[:, :3].tobytes()))
            if pal.shape[1] == 4:
                opaque = pal[:, 3] == 255
                t = 0 if opaque.all() else int(np.nonzero(~opaque)[0][-1]) + 1
                if t:
                    chunks.append(label_chunk(b"tRNS", pal[:t, 3].tobytes()))
        return b"\x89PNG\r\n\x1a\n" + b"".join(chunks) + body

    def label_bound(self, w, h, depth, palette=None) -> int:
        """fpngb_max_label_encoded_size restated: the packed rows' bound plus the PLTE / tRNS chunk bytes"""
        pw, bpp = (w, 2) if depth == 16 else ((w * depth + 7) // 8, 1)
        extra = 0
        if palette is not None:
            pal = np.asarray(palette, dtype=np.uint8)
            extra = 12 + 3 * len(pal)
            if pal.shape[1] == 4 and (pal[:, 3] != 255).any():
                extra += 12 + int(np.nonzero(pal[:, 3] != 255)[0][-1]) + 1
        return self.png.max_encoded_size(pw, h, bpp) + extra


def label_chunk(kind: bytes, data: bytes) -> bytes:
    import zlib
    return len(data).to_bytes(4, "big") + kind + data + zlib.crc32(kind + data).to_bytes(4, "big")
