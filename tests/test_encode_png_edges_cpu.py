"""The edge images of tests/pngenc_edges.py as the oracle encodes them (oracle/png_encode_oracle.c): each file decodes to its
image through zlib plus a NumPy unfilter (PIL for the 2^24 gray limits), and each image reaches the construct it names, read back
from the Deflate stream by tests/deflatetrace.py, which is first checked against zlib.  tests/test_encode_png_edges_gpu.py holds
the GPU's files to the oracle's on the same images."""
from __future__ import annotations

import os
import sys
import zlib
from collections import defaultdict

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import deflatetrace as dt  # noqa: E402
import pngenc_edges as pe  # noqa: E402
import pngenc_workloads as pw  # noqa: E402
from oracle.pngenc_oracle import PngEncodeOracle  # noqa: E402


@pytest.fixture(scope="module")
def oracle():
    return PngEncodeOracle()


def chunks(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    at, out = 8, []
    while at < len(data):
        n = int.from_bytes(data[at:at + 4], "big")
        kind, body = data[at + 4:at + 8], data[at + 8:at + 8 + n]
        assert int.from_bytes(data[at + 8 + n:at + 12 + n], "big") == zlib.crc32(kind + body)
        out.append((kind, body))
        at += 12 + n
    assert at == len(data)
    return out


def zstream(png: bytes) -> bytes:
    ch = chunks(png)
    assert [k for k, _ in ch] == [b"IHDR", b"IDAT", b"IEND"]
    z = ch[1][1]
    assert z[:2] == b"\x78\x01"
    return z


def unfilter(raw: bytes, h, w, B):
    """Inflated stream -> PNG-order bytes [h, w * B]; filters 0-2 whole-row, 3 and 4 pixel by pixel over the B bytes."""
    rows = np.frombuffer(raw, np.uint8).reshape(h, 1 + w * B)
    out = np.zeros((h, w, B), np.uint8)
    up = np.zeros((w, B), np.int64)
    for y in range(h):
        ft, f = rows[y, 0], rows[y, 1:].reshape(w, B).astype(np.int64)
        if ft == 0:
            cur = f
        elif ft == 1:
            cur = np.cumsum(f, axis=0) & 255
        elif ft == 2:
            cur = (f + up) & 255
        else:
            cur = np.zeros((w, B), np.int64)
            a = c = np.zeros(B, np.int64)
            for x in range(w):
                b = up[x]
                if ft == 3:
                    pred = (a + b) >> 1
                else:
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
                a = cur[x] = (f[x] + pred) & 255
                c = b
        out[y], up = cur, cur
    return out.reshape(h, w * B), rows[:, 0].copy()


def to_pixels(be, h, w, c, dtype):
    if np.dtype(dtype) == np.uint16:
        be = be.reshape(h, w * c, 2)
        return ((be[..., 0].astype(np.uint16) << 8) | be[..., 1]).reshape(h, w, c)
    return be.reshape(h, w, c)


def decode(png: bytes, img):
    """-> (pixels, filter types, Trace) of one file, checked against zlib and the IDAT length / IHDR"""
    h, w, c = img.shape
    z = zstream(png)
    raw = zlib.decompress(z)
    t = dt.trace(z)
    assert t.data == raw and t.end_byte + 4 == len(z)
    be, ft = unfilter(raw, h, w, c * img.dtype.itemsize)
    return to_pixels(be, h, w, c, img.dtype), ft, t


def test_trace_equals_zlib_on_corpus(oracle):
    """The trace reader inflates every corpus file as zlib does and ends where the Adler-32 starts."""
    n = 0
    for flags in (0, 1, pe.FORCE_UNCOMPRESSED):
        for name, img in pw.corpus():
            z = zstream(oracle.png_encode(img, flags))
            t = dt.trace(z)
            assert t.data == zlib.decompress(z), (name, flags)
            assert t.end_byte + 4 == len(z), (name, flags)
            assert int.from_bytes(z[-4:], "big") == zlib.adler32(t.data)
            assert all(b.btype in (0, 2) for b in t.blocks)
            if t.blocks[0].btype == 2:                         # one dynamic block whose codes the tokens re-expand to
                out = bytearray()
                for tok in t.blocks[0].tokens:
                    if isinstance(tok, int):
                        out.append(tok)
                    else:
                        for _ in range(tok[0]):
                            out.append(out[-tok[1]])
                assert bytes(out) == t.data
            n += 1
    print(f"trace == zlib on {n} corpus files")


def block_boundary_kinds(t: dt.Trace, w, h, c, es):
    """The boundary kinds (pngenc_edges.boundary_kinds) of the stored blocks actually in the stream."""
    B = c * es
    n = w * B + 1
    kinds = set()
    for b in t.blocks[1:]:
        s = b.out_start
        r = s % n
        if r == 0:
            kinds.add("filter")
        else:
            j = (r - 1) % B
            kinds.add("pixel" if j == 0 else ("sample" if es == 2 and j % 2 else "channel"))
    if t.blocks[-1].stored_len == pe.BLOCK:
        kinds.add("exact")
    if t.blocks[-1].stored_len == 1:
        kinds.add("plus1")
    return kinds


def test_stored_edges(oracle):
    seen = defaultdict(set)
    for e in pe.stored_edges():
        h, w, c = e.img.shape
        es = e.img.dtype.itemsize
        raw = pe.raw_size(w, h, e.B)
        for flags in e.flags:
            png = oracle.png_encode(e.img, flags)
            px, ft, t = decode(png, e.img)
            assert np.array_equal(px, e.img), (e.name, flags)
            if t.blocks[0].btype != 0:
                assert flags == 0 and e.B == 1, (e.name, "only gray8 noise may compress")   # 8-bit codes win on short rows
                continue
            assert not ft.any()
            assert all(b.btype == 0 for b in t.blocks) and t.blocks[-1].final and not any(b.final for b in t.blocks[:-1])
            nblk = -(-raw // pe.BLOCK)
            assert len(t.blocks) == nblk >= 3, e.name
            assert [b.stored_len for b in t.blocks] == [pe.BLOCK] * (nblk - 1) + [raw - pe.BLOCK * (nblk - 1)], e.name
            assert len(zstream(png)) == pe.zstored(w, h, e.B)
            kinds = block_boundary_kinds(t, w, h, c, es)
            assert kinds | {"stored"} == e.construct, (e.name, kinds)
            name = e.name.split("_")[1]
            seen[name] |= kinds | {"natural" if flags == 0 else "forced"} | ({"expand"} if e.expand else set())
    for name, c, dtype in pe.CLASSES:
        want = {"filter", "exact", "plus1", "forced", "natural", "expand"}
        want |= {"sample"} if np.dtype(dtype).itemsize == 2 else set()
        want |= {"channel"} if c > 1 else set()
        assert want <= seen[name], (name, want - seen[name])
        print(f"stored {name}: hit {sorted(seen[name])}")


def test_tie_edges(oracle):
    """Per class: the member k* whose compressed stream is exactly as long as the stored one is compressed (zcomp <= zstored),
    k* + 1 is stored, and every member decodes."""
    fam = defaultdict(list)
    for e in pe.tie_edges(oracle):
        fam[e.name.split("_")[1]].append(e)
    assert sorted(fam) == sorted(n for n, _, _ in pe.CLASSES)
    for name, members in fam.items():
        gaps = []
        for e in members:
            h, w, _ = e.img.shape
            png = oracle.png_encode(e.img)
            px, _, t = decode(png, e.img)
            assert np.array_equal(px, e.img), e.name
            zlen, btype = pe.idat_info(png)
            zst = pe.zstored(w, h, e.B)
            if "tie" in e.construct:
                assert btype == 2 and zlen == zst, (e.name, zlen, zst)
            if "first_stored" in e.construct:
                assert btype == 0 and zlen == zst, e.name
            gaps.append((e.k, "compressed" if btype == 2 else "stored", zst - zlen if btype == 2 else None))
        print(f"tie {name}: zstored {zst}; (k, kind, zstored - zcomp): {gaps}")


def runs_of(row_px):
    """maximal runs [s, e] (e > s) of equal pixels in one filtered row [w, B]"""
    eq = np.all(row_px[1:] == row_px[:-1], axis=1)
    out, s = [], None
    for x, q in enumerate(eq, start=1):
        if q and s is None:
            s = x - 1
        if not q and s is not None:
            out.append((s, x - 1)); s = None
    if s is not None:
        out.append((s, len(row_px) - 1))
    return out


def row_tokens(t: dt.Trace, n, h):
    """the tokens of each row (n = stream bytes per row); no match may cross a row"""
    rows = [[] for _ in range(h)]
    at = 0
    for tok in t.blocks[0].tokens:
        L = 1 if isinstance(tok, int) else tok[0]
        assert at // n == (at + L - 1) // n, "a match crosses a row"
        rows[at // n].append((at % n, tok))
        at += L
    return rows


def test_wide_edges(oracle):
    hit = defaultdict(set)
    for e in pe.wide_edges():
        h, w, c = e.img.shape
        B = e.B
        M = 258 // B
        for flags in e.flags:
            png = oracle.png_encode(e.img, flags)
            px, ft, t = decode(png, e.img)
            assert np.array_equal(px, e.img), (e.name, flags)
            if flags:
                assert all(b.btype == 0 for b in t.blocks)
                continue
            assert len(t.blocks) == 1 and t.blocks[0].btype == 2, e.name
            n = w * B + 1
            filt = np.frombuffer(t.data, np.uint8).reshape(h, n)[:, 1:].reshape(h, w, B)
            rows = row_tokens(t, n, h)
            name = e.name.split("_")[1]
            for y in range(h):
                runs = runs_of(filt[y])
                if any(s % 32 == 31 and e_ % 32 == 0 for s, e_ in runs):
                    hit[name].add("lane31_to_lane0")
                last_at, last = rows[y][-1]
                if not isinstance(last, int) and last_at + last[0] == n and w % 32:
                    hit[name].add(f"tail_match_in_partial_step_r{w % 32}")
                lens = {tok[0] for _, tok in rows[y] if not isinstance(tok, int)}
                if M * B in lens:
                    hit[name].add("full_match")
                for s, e_ in runs_of(e.img[y].astype(np.int64)):              # runs of equal image pixels
                    for m in (1, 2):
                        if e_ - s + 1 in (M * m - 1, M * m + 1):
                            hit[name].add(f"run_M*{m}+-1")
            if w % 32 == 0 and any(not isinstance(r[-1][1], int) and r[-1][0] + r[-1][1][0] == n for r in rows):
                hit[name].add("tail_match_in_full_step")
    for name, _, _ in pe.CLASSES:
        want = {"lane31_to_lane0", "full_match", "run_M*1+-1", "run_M*2+-1", "tail_match_in_full_step"}
        want |= {f"tail_match_in_partial_step_r{r}" for r in range(1, 32)}
        assert want <= hit[name], (name, sorted(want - hit[name]))
        print(f"wide {name}: every residue 0..31 ends its row in a match; also {sorted(h for h in hit[name] if 'step_r' not in h)}")


def test_limit_edges(oracle):
    """The 2^24 limits compress, carry their size in IHDR and decode (PIL for gray, zlib plus the sub unfilter for RGBA16)."""
    import io
    import struct

    from PIL import Image
    for e in pe.limit_edges():
        h, w, c = e.img.shape
        png = oracle.png_encode(e.img)
        assert struct.unpack(">II", png[16:24]) == (w, h)
        zlen, btype = pe.idat_info(png)
        assert btype == 2, e.name
        if c == 1:
            got = np.asarray(Image.open(io.BytesIO(png))).reshape(h, w, 1).astype(e.img.dtype)
        else:
            raw = zlib.decompress(zstream(png))
            assert h == 1 and raw[0] in (0, 1, 4), e.name                # row 0: paeth of (a, 0, 0) is a, as sub
            f = np.frombuffer(raw, np.uint8)[1:].reshape(w, e.B)
            be = f if raw[0] == 0 else (np.cumsum(f, axis=0, dtype=np.uint8))
            got = to_pixels(be, h, w, c, e.img.dtype)
        assert np.array_equal(got, e.img), e.name
        print(f"limit {e.name}: {w}x{h}, zlib stream {zlen} bytes of {pe.zstored(w, h, e.B)} stored")
