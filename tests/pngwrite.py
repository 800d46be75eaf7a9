"""A small PNG writer and numpy filter / unfilter model for the general-PNG decode tests: every row filter, any zlib level,
strategy, window size and flush, IDAT splits and extra chunks, all built from numpy and zlib (no imaging library)."""
from __future__ import annotations

import struct
import zlib

import numpy as np

COLOR_TYPE = {1: 0, 2: 4, 3: 2, 4: 6}          # channels -> IHDR color type
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}


def chunk(tag: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def ihdr(w, h, depth=8, ctype=2, comp=0, filt=0, interlace=0) -> bytes:
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, comp, filt, interlace))


SIG = b"\x89PNG\r\n\x1a\n"
IEND = chunk(b"IEND", b"")


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(img: np.ndarray, filters) -> bytes:
    """the filtered scanlines of img [h, w, c] uint8, row y with filter type filters[y]"""
    h, w, c = img.shape
    rows = img.reshape(h, w * c).astype(np.int32)
    out = np.zeros((h, w * c + 1), np.uint8)
    prev = np.zeros(w * c, np.int32)
    z = np.zeros(c, np.int32)
    for y in range(h):
        cur, ft = rows[y], int(filters[y])
        a = np.concatenate([z, cur[:-c]])
        cc = np.concatenate([z, prev[:-c]])
        pred = [0 * cur, a, prev, (a + prev) // 2, paeth(a, prev, cc)][ft]
        out[y, 0] = ft
        out[y, 1:] = (cur - pred) & 255
        prev = cur
    return out.tobytes()


def unfilter(raw: bytes, w: int, h: int, c: int):
    """numpy model of the decoder's unfilter: [h, w, c] uint8, or None when a filter byte is above 4"""
    stride = w * c + 1
    buf = np.frombuffer(raw, np.uint8).reshape(h, stride).astype(np.int32)
    out = np.zeros((h, w * c), np.int32)
    prev = np.zeros(w * c, np.int32)
    for y in range(h):
        ft, f = int(buf[y, 0]), buf[y, 1:]
        if ft > 4:
            return None
        if ft in (0, 2):
            cur = (f + (prev if ft == 2 else 0)) & 255
        else:
            cur = np.zeros(w * c, np.int32)
            for x in range(w * c):
                a = cur[x - c] if x >= c else 0
                b = prev[x]
                cc = prev[x - c] if x >= c else 0
                pred = a if ft == 1 else (a + b) // 2 if ft == 3 else int(paeth(np.int32(a), np.int32(b), np.int32(cc)))
                cur[x] = (f[x] + pred) & 255
        out[y] = cur
        prev = cur
    return out.reshape(h, w, c).astype(np.uint8)


def row_filters(h: int, mode, seed: int = 0):
    if mode == "random":
        return np.random.RandomState(seed).randint(0, 5, h)
    return np.full(h, int(mode))


def compress(data: bytes, level=6, strategy="default", wbits=15, flush=None) -> bytes:
    """zlib stream of data; flush = (zlib flush mode, [split points]) flushes mid-stream at those byte offsets"""
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, STRATEGIES[strategy])
    if not flush:
        return co.compress(data) + co.flush()
    mode, points = flush
    out, at = b"", 0
    for p in points:
        out += co.compress(data[at:p]) + co.flush(mode)
        at = p
    return out + co.compress(data[at:]) + co.flush()


def split_idat(z: bytes, split=None, seed: int = 0):
    """IDAT payloads: one chunk (None), 1-byte chunks ("bytes"), random sizes ("random"), random sizes with zero-length chunks
    between ("zeros"), or fixed-size chunks (an int)"""
    if split is None:
        return [z]
    if split == "bytes":
        return [z[i:i + 1] for i in range(len(z))]
    if isinstance(split, int):
        return [z[i:i + split] for i in range(0, len(z), split)] or [b""]
    rs = np.random.RandomState(seed)
    parts, at = [], 0
    while at < len(z):
        k = int(rs.randint(1, 64))
        parts.append(z[at:at + k])
        at += k
        if split == "zeros" and rs.randint(0, 3) == 0:
            parts.append(b"")
    return parts


def make_png(img: np.ndarray, filters="random", level=6, strategy="default", wbits=15, flush=None, split=None, seed=0,
             before=(), between=(), after=(), z=None) -> bytes:
    """a PNG of img [h, w, c] (c = 1 gray, 2 gray+alpha, 3, 4); before / after: extra chunks before / after the IDAT run,
    between: chunks after the first IDAT chunk (which break the run); z replaces the zlib stream"""
    h, w, c = img.shape
    if z is None:
        z = compress(filter_rows(img, row_filters(h, filters, seed)), level, strategy, wbits, flush)
    parts = [chunk(b"IDAT", p) for p in split_idat(z, split, seed)]
    body = parts[:1] + list(between) + parts[1:]
    return SIG + ihdr(w, h, ctype=COLOR_TYPE[c]) + b"".join(before) + b"".join(body) + b"".join(after) + IEND


def gray(img: np.ndarray) -> np.ndarray:
    return img[..., :1].copy()


def gray_alpha(img4: np.ndarray) -> np.ndarray:
    return img4[..., [0, 3]].copy()


def expand(img: np.ndarray, desired: int) -> np.ndarray:
    """the decoder's channel mapping (PIL's convert("RGB") / convert("RGBA"))"""
    h, w, c = img.shape
    if c in (1, 2):
        rgb = np.repeat(img[..., :1], 3, axis=2)
        alpha = img[..., 1:2] if c == 2 else np.full((h, w, 1), 255, np.uint8)
    else:
        rgb = img[..., :3]
        alpha = img[..., 3:4] if c == 4 else np.full((h, w, 1), 255, np.uint8)
    return rgb if desired == 3 else np.concatenate([rgb, alpha], axis=2)


def source(kind: str, w: int, h: int, c: int, index: int = 0) -> np.ndarray:
    """an imagegen image with c channels"""
    import imagegen
    if c == 1:
        return gray(imagegen.make(kind, w, h, 3, index))
    if c == 2:
        return gray_alpha(imagegen.make(kind, w, h, 4, index))
    return imagegen.make(kind, w, h, c, index)
