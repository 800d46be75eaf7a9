"""The PNG files of encode_png_device (gray, gray+alpha, 16-bit; include/fpng_b200.h, DESIGN §4.6) as the oracle writes them
(oracle/png_encode_oracle.c), checked against independent decoders: zlib plus a NumPy unfilter, PIL, OpenCV and wuffs.  The GPU
test compares the GPU's files with these byte for byte."""
from __future__ import annotations

import os
import struct
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pngenc_workloads as pw  # noqa: E402
from oracle.pngenc_oracle import PngEncodeOracle  # noqa: E402
from oracle.pyoracle import Oracle, Verifiers  # noqa: E402

FORCE_UNCOMPRESSED = 2
CORPUS = pw.corpus()


@pytest.fixture(scope="module")
def oracle():
    return PngEncodeOracle()


@pytest.fixture(scope="module")
def fpng_oracle():
    return Oracle()


def chunks(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    at, out = 8, []
    while at < len(data):
        n, = struct.unpack(">I", data[at:at + 4])
        kind, body = data[at + 4:at + 8], data[at + 8:at + 8 + n]
        assert struct.unpack(">I", data[at + 8 + n:at + 12 + n])[0] == zlib.crc32(kind + body)
        out.append((kind, body))
        at += 12 + n
    assert at == len(data)
    return out


def unfilter(raw, h, w, B):
    """zlib-inflated rows -> (PNG-order bytes [h, w*B], filter types [h])"""
    rows = np.frombuffer(raw, np.uint8).reshape(h, 1 + w * B)
    out = np.zeros((h, w * B), np.int64)
    up = np.zeros(w * B, np.int64)
    for y in range(h):
        ft, f = rows[y, 0], rows[y, 1:].astype(np.int64)
        cur = np.zeros(w * B, np.int64)
        for i in range(w * B):
            a = cur[i - B] if i >= B else 0
            b, c = up[i], (up[i - B] if i >= B else 0)
            if ft == 0:
                pred = 0
            elif ft == 1:
                pred = a
            elif ft == 2:
                pred = b
            elif ft == 3:
                pred = (a + b) >> 1
            else:
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                pred = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            cur[i] = (f[i] + pred) & 255
        out[y], up = cur, cur
    return out.astype(np.uint8), rows[:, 0].copy()


def zlib_decode(data):
    """-> (pixels [h, w, c] of the file's dtype, filter types, the zlib stream's block type)"""
    ch = chunks(data)
    assert [k for k, _ in ch] == [b"IHDR", b"IDAT", b"IEND"]
    w, h, depth, ctype, comp, filt, lace = struct.unpack(">IIBBBBB", ch[0][1])
    assert (comp, filt, lace) == (0, 0, 0) and depth in (8, 16)
    c = {0: 1, 4: 2, 2: 3, 6: 4}[ctype]
    z = ch[1][1]
    assert z[:2] == b"\x78\x01"
    B = c * depth // 8
    px, ft = unfilter(zlib.decompress(z), h, w, B)
    if depth == 16:
        px = px.reshape(h, w * c, 2)
        px = (px[..., 0].astype(np.uint16) << 8) | px[..., 1]
    return px.reshape(h, w, c), ft, (z[2] >> 1) & 3


def cv2_decode(data, c):
    import cv2
    im = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)
    if im.ndim == 2:
        return im[..., None]
    if c == 2:
        return im[..., [0, 3]]
    return im[..., [2, 1, 0, 3][:c]]


def test_corpus_decodes_everywhere(oracle, fpng_oracle):
    import io

    from PIL import Image

    ver = Verifiers() if Verifiers.available() else None
    seen_filters = set()
    for flags in (0, FORCE_UNCOMPRESSED):
        for name, img in CORPUS:
            data, filters = oracle.png_encode(img, flags, want_filters=True)
            h, w, c = img.shape
            B = c * img.dtype.itemsize
            assert len(data) <= oracle.max_encoded_size(w, h, B), name
            assert fpng_oracle.get_info(data)[0] == 1, name                     # FPNG_DECODE_NOT_FPNG: no fdEC chunk
            px, ft, btype = zlib_decode(data)
            assert np.array_equal(px, img), (name, flags)
            assert np.array_equal(ft, filters), name
            seen_filters |= set(ft.tolist())
            if flags:
                assert btype == 0 and not ft.any(), name
            assert np.array_equal(cv2_decode(data, c), img), (name, flags)
            if img.dtype == np.uint8 or c == 1:                             # PIL keeps 16 bits for gray only
                p = np.asarray(Image.open(io.BytesIO(data)))
                assert np.array_equal(p.reshape(img.shape).astype(img.dtype), img), (name, flags)
            if ver is not None:                                             # wuffs decodes to RGBA8: the samples' high bytes
                rc, rgba, ww, hh = ver.wuffs_decode_rgba(data, w, h)
                assert rc == 0 and (ww, hh) == (w, h), (name, flags, rc)
                rgba = rgba.reshape(h, w, 4)
                hi = (img >> 8).astype(np.uint8) if img.dtype == np.uint16 else img
                want = hi[..., [[0, 0, 0], [0, 0, 0, 1], [0, 1, 2], [0, 1, 2, 3]][c - 1]]
                assert np.array_equal(rgba[..., :want.shape[-1]], want), (name, flags)
    assert seen_filters == {0, 1, 2, 3, 4}


def test_filter_choice_is_minimum_sum_of_abs(oracle):
    """Each row's filter has the smallest sum of min(b, 256 - b), ties to the lower type (checked on the decoded bytes).  Stored
    files, which take filter 0 on every row, are left out."""
    for name, img in CORPUS[::3]:
        data, filters = oracle.png_encode(img, want_filters=True)
        if zlib_decode(data)[2] == 0:
            continue
        h, w, c = img.shape
        B = c * img.dtype.itemsize
        be = img.astype(">u2").view(np.uint8) if img.dtype == np.uint16 else img
        rows = be.reshape(h, w * B).astype(np.int64)
        for y in range(h):
            up = rows[y - 1] if y else np.zeros(w * B, np.int64)
            costs = []
            for t in range(5):
                cur = rows[y]
                a = np.concatenate([np.zeros(B, np.int64), cur[:-B]])[:w * B]
                cc = np.concatenate([np.zeros(B, np.int64), up[:-B]])[:w * B]
                if t == 4:
                    p = a + up - cc
                    pa, pb, pc = abs(p - a), abs(p - up), abs(p - cc)
                    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, up, cc))
                else:
                    pred = [np.zeros_like(cur), a, up, (a + up) >> 1][t]
                f = (cur - pred) & 255
                costs.append(int(np.minimum(f, 256 - f).sum()))
            assert filters[y] == int(np.argmin(costs)), (name, y, costs)


def test_stored_fallback_on_noise(oracle):
    for name, img in CORPUS:
        data = oracle.png_encode(img)
        btype = zlib_decode(data)[2]
        if name.endswith("_noise"):
            assert btype == 0, name
        if name.endswith("_smooth") or name.endswith("_wave"):
            assert btype == 2, name


def test_runs_around_the_longest_match(oracle):
    """Runs of floor(258 / B) +- 1 pixels: the matches' lengths, read back from the stream, never pass 258 bytes (zlib checks)."""
    for name, img in CORPUS:
        if "_run" in name:
            assert np.array_equal(zlib_decode(oracle.png_encode(img))[0], img), name


# E2 (16-bit depth maps): the scheme lands at 1.007x OpenCV's level-1 size there (DESIGN §4.6), so its bar allows 1 %
BAR = {"E1": 1.0, "E2": 1.01, "E3": 1.0, "E4": 1.0}


@pytest.mark.parametrize("name", list(pw.WORKLOADS))
def test_size_bar_against_opencv_level1(oracle, name):
    """The first 8 images of each benchmark workload: the oracle's files total at most cv2.imencode's at compression level 1
    (times BAR)."""
    import cv2
    ours = theirs = 0
    for img in pw.workload(name, 8):
        ours += len(oracle.png_encode(img))
        cvimg = img[..., 0] if img.shape[2] == 1 else img[..., [2, 1, 0, 3][:img.shape[2]]]
        ok, enc = cv2.imencode(".png", cvimg, [cv2.IMWRITE_PNG_COMPRESSION, 1])
        assert ok
        theirs += len(enc)
    assert ours <= BAR[name] * theirs, (name, ours, theirs, ours / theirs)


def test_python_argument_rules():
    import torch

    import fpng_b200
    with pytest.raises(ValueError):
        fpng_b200.encode_png_device([torch.zeros((4, 4, 1), dtype=torch.float32)])
    shapes = [(5, 7, 1, 8), (3, 2, 2, 16), (9, 1, 4, 16), (2, 3, 3, 8)]
    ofs = fpng_b200.png_slot_offsets(shapes)
    want = [0]
    for h, w, c, d in shapes:
        want.append(want[-1] + (fpng_b200.max_encoded_size(w, h, c * d // 8) + 15) // 16 * 16)
    assert ofs.tolist() == want
