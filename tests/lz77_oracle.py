"""ctypes front-end of tests/cpp/lz77_oracle.c, the TEST-ONLY C restatement of the LZ77 mode of the PNG encode
(FPNGB_LZ77_CHAIN, include/fpng_b200.h "LZ77").  It builds tests/cpp/liblz77_oracle.so from that file and oracle/png_encode_oracle.c,
which it includes.  Only the tests and tools/bench scripts import it."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "lz77_oracle.c")
DEPS = [SRC, os.path.join(HERE, "..", "oracle", "png_encode_oracle.c"), os.path.join(HERE, "..", "oracle", "fpng_oracle.c")]
SO = os.path.join(HERE, "cpp", "liblz77_oracle.so")
INFO_KEYS = ("n", "tokens", "dist_syms", "stored", "zcomp", "zstored", "rows_crossed", "max_dist")
STAT_KEYS = ("rows_crossed", "max_dist", "len258", "cut_at_segment")


def build(force: bool = False) -> str:
    if force or not os.path.exists(SO) or any(os.path.getmtime(SO) < os.path.getmtime(s) for s in DEPS):
        tmp = SO + ".building"
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-o", tmp, SRC])
        os.replace(tmp, SO)
    return SO


_L = None


def lib():
    global _L
    if _L is None:
        L = C.CDLL(build())
        L.lz77_encode.restype = C.c_size_t
        L.lz77_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                  C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.lz77_parse.restype = C.c_size_t
        L.lz77_parse.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t]
        L.oracle_init()
        _L = L
    return _L


def chunk(kind: bytes, data: bytes) -> bytes:
    return len(data).to_bytes(4, "big") + kind + data + zlib.crc32(kind + data).to_bytes(4, "big")


def container(w, h, depth, color_type, palette=None) -> bytes:
    """signature, IHDR, a palette's PLTE and tRNS, then the IDAT length (patched by the encoder) and type"""
    parts = [b"\x89PNG\r\n\x1a\n", chunk(b"IHDR", w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([depth, color_type, 0, 0, 0]))]
    if palette is not None:
        pal = np.asarray(palette, dtype=np.uint8)
        parts.append(chunk(b"PLTE", pal[:, :3].tobytes()))
        if pal.shape[1] == 4:
            opaque = pal[:, 3] == 255
            t = 0 if opaque.all() else int(np.nonzero(~opaque)[0][-1]) + 1
            if t:
                parts.append(chunk(b"tRNS", pal[:t, 3].tobytes()))
    return b"".join(parts) + b"\0\0\0\0IDAT"


def encode_rows(rows: np.ndarray, B: int, hdr: bytes, K: int, flags: int = 0, want_info: bool = False):
    """The LZ77-mode file of h rows (uint8 [h, R], PNG byte order) filtered at distance B behind the container header hdr."""
    rows = np.ascontiguousarray(rows, dtype=np.uint8)
    h, R = rows.shape
    cap = len(hdr) + 2 + (R + 1) * h + 5 * (((R + 1) * h + 65534) // 65535) + 4 + 16
    out = np.empty(cap, dtype=np.uint8)
    info = np.zeros(8, dtype=np.uint64)
    stats = np.zeros(4, dtype=np.uint64)
    hb = np.frombuffer(hdr, dtype=np.uint8)
    n = lib().lz77_encode(rows.ctypes.data, R, h, B, hb.ctypes.data, len(hdr), flags, K, out.ctypes.data, cap, info.ctypes.data,
                          stats.ctypes.data)
    assert n, "lz77_encode"
    data = out[:n].tobytes()
    if not want_info:
        return data
    d = dict(zip(INFO_KEYS, map(int, info)))
    d.update(zip(STAT_KEYS, map(int, stats)))
    return data, d


def parse(S: bytes, K: int):
    """the rule's tokens for a given stream S (no filtering): a literal is an int, a match a (length, distance) pair"""
    a = np.frombuffer(S, dtype=np.uint8)
    ln = np.zeros(max(len(S), 1), np.uint16)
    ds = np.zeros(max(len(S), 1), np.uint16)
    n = lib().lz77_parse(a.ctypes.data, len(S), K, ln.ctypes.data, ds.ctypes.data, len(ln))
    return [(int(l), int(d)) if l else int(d) for l, d in zip(ln[:n], ds[:n])]


def image_rows(img: np.ndarray):
    """(rows in PNG byte order, B) of an [h, w, c] uint8 / uint16 image"""
    a = np.ascontiguousarray(img)
    h, w, c = a.shape
    if a.dtype == np.uint16:
        return a.astype(">u2").view(np.uint8).reshape(h, w * c * 2), 2 * c
    return a.reshape(h, w * c), c


def png_encode(img: np.ndarray, K: int, flags: int = 0, want_info: bool = False):
    """The file encode_png_device(lz77=K) writes for img, [h, w, c] uint8 or uint16 (c 1..4)"""
    h, w, c = img.shape
    rows, B = image_rows(img)
    return encode_rows(rows, B, container(w, h, 8 * img.dtype.itemsize, (0, 4, 2, 6)[c - 1]), K, flags, want_info)


def label_rows(ids: np.ndarray, depth: int):
    """(packed rows, B) of a label map: MSB-first ids for depth < 16, big-endian uint16 for depth 16"""
    a = np.asarray(ids).astype(np.int64)
    h, w = a.shape
    if depth == 16:
        return a.astype(">u2").view(np.uint8).reshape(h, 2 * w), 2
    per = 8 // depth
    v = np.concatenate([a, np.zeros((h, (-w) % per), np.int64)], axis=1).reshape(h, -1, per)
    shifts = np.array([8 - depth * (k + 1) for k in range(per)], dtype=np.int64)
    return (v << shifts).sum(axis=2).astype(np.uint8), 1


def label_encode(ids: np.ndarray, depth: int, K: int, palette=None, flags: int = 0):
    """The file encode_labels_device(lz77=K) writes for ids [h, w] (all in range)"""
    h, w = np.asarray(ids).shape
    rows, B = label_rows(ids, depth)
    return encode_rows(rows, B, container(w, h, depth, 0 if palette is None else 3, palette), K, flags)
