"""The general-PNG walk (fpngb_get_png_info, the host instantiation of png_walk) on the CPU: one status per walk rule from
hand-edited chunks with correct CRCs, agreement with PIL on PIL- and OpenCV-written files, and fpng files' rows equal to
get_info_ex's.  The test PNG writer and its numpy unfilter model are pinned against PIL's decoder."""
import io
import json
import os
import struct
import zlib

import numpy as np
import pytest

import imagegen
import pngwrite
from pngwrite import IEND, SIG, chunk, ihdr

NOT_PNG, HEADER_CRC, INVALID_DIMS, CHUNK_PARSING, INVALID_IDAT, UNSUPPORTED = 3, 4, 5, 7, 8, 104
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "anypng")


def info(data):
    import fpng_b200
    return fpng_b200.get_png_info(data)


def idat(img, **kw):
    h = img.shape[0]
    return chunk(b"IDAT", pngwrite.compress(pngwrite.filter_rows(img, pngwrite.row_filters(h, "random")), **kw))


IMG = pngwrite.source("g1", 9, 5, 3)
PAD = chunk(b"tEXt", b"padding\0" + b"x" * 24)     # keeps short cases above the walk's minimum file size


def flip_last(b: bytes) -> bytes:
    return b[:-1] + bytes([b[-1] ^ 1])


def test_valid_files_every_color_type():
    for c in (1, 2, 3, 4):
        img = pngwrite.source("g1", 13, 7, c, c)
        png = pngwrite.make_png(img, split=17)
        st, w, h, cc, ofs, ln = info(png)
        assert (st, w, h, cc) == (0, 13, 7, c)
        assert png[ofs + 4:ofs + 8] == b"IDAT"
        assert ln == sum(len(p) for p in pngwrite.split_idat(pngwrite.compress(pngwrite.filter_rows(
            img, pngwrite.row_filters(7, "random"))), 17))


@pytest.mark.parametrize("field,value", [(0, 16), (0, 4), (0, 1), (1, 3), (1, 1), (1, 5), (2, 1), (3, 1), (4, 1)])
def test_ihdr_variants_are_unsupported(field, value):
    fields = [8, 2, 0, 0, 0]                      # depth, color type, compression, filter method, interlace
    fields[field] = value
    png = SIG + ihdr(9, 5, *fields) + idat(IMG) + IEND
    assert info(png)[0] == UNSUPPORTED


def test_walk_rules():
    body = idat(IMG)
    good = SIG + ihdr(9, 5) + body + IEND
    assert info(good)[0] == 0
    cases = {
        "unknown critical chunk": (SIG + ihdr(9, 5) + chunk(b"ABCD", b"x") + body + IEND, UNSUPPORTED),
        "second IHDR": (SIG + ihdr(9, 5) + ihdr(9, 5) + body + IEND, UNSUPPORTED),
        "tRNS in RGB": (SIG + ihdr(9, 5) + chunk(b"tRNS", b"\0\1\0\2\0\3") + body + IEND, UNSUPPORTED),
        "PLTE in RGB": (SIG + ihdr(9, 5) + chunk(b"PLTE", b"\1\2\3" * 4) + body + chunk(b"PLTE", b"\1\2\3") + IEND, 0),
        "ancillary chunks": (SIG + ihdr(9, 5) + chunk(b"gAMA", b"\0\1\x86\xa0") + chunk(b"tEXt", b"k\0v") + body +
                             chunk(b"zzZz", b"") + IEND, 0),
        "bad ancillary CRC": (SIG + ihdr(9, 5) + flip_last(chunk(b"gAMA", b"\0\1\x86\xa0")) + body + IEND, HEADER_CRC),
        "no IDAT": (SIG + ihdr(9, 5) + PAD + IEND, INVALID_IDAT),
        "one data byte": (SIG + ihdr(9, 5) + PAD + chunk(b"IDAT", b"\x78") + IEND, INVALID_IDAT),
        "zero-length IDATs": (SIG + ihdr(9, 5) + chunk(b"IDAT", b"") + body + chunk(b"IDAT", b"") + IEND, 0),
        "IDAT run broken": (SIG + ihdr(9, 5) + body + chunk(b"tEXt", b"k\0v") + chunk(b"IDAT", b"") + IEND, CHUNK_PARSING),
        "no IEND": (SIG + ihdr(9, 5) + body, CHUNK_PARSING),
        "width 0": (SIG + ihdr(0, 5) + body + IEND, INVALID_DIMS),
        "too many pixels": (SIG + ihdr(1 << 16, 1 << 15) + body + IEND, INVALID_DIMS),
        "bad signature": (b"\x89PNG\r\n\x1a\x0b" + ihdr(9, 5) + body + IEND, NOT_PNG),
        "bad IHDR CRC": (SIG + flip_last(ihdr(9, 5)) + body + IEND, HEADER_CRC),
    }
    for name, (png, want) in cases.items():
        assert info(png)[0] == want, name
    # tRNS in gray: unsupported; in gray+alpha / RGBA it is ignored (the file has alpha already)
    for c, want in ((1, UNSUPPORTED), (2, 0), (4, 0)):
        img = pngwrite.source("g0", 6, 4, c)
        png = pngwrite.make_png(img, before=[chunk(b"tRNS", b"\0\1")])
        assert info(png)[0] == want, c
    # PLTE in a gray file
    png = pngwrite.make_png(pngwrite.source("g0", 6, 4, 1), before=[chunk(b"PLTE", b"\1\2\3")])
    assert info(png)[0] == UNSUPPORTED


def test_split_idat_offsets_and_lengths():
    img = pngwrite.source("g1", 31, 17, 4)
    z = pngwrite.compress(pngwrite.filter_rows(img, pngwrite.row_filters(17, "random")))
    for split in (None, "bytes", "random", "zeros", 7):
        png = pngwrite.make_png(img, z=z, split=split, before=[chunk(b"pHYs", b"\0" * 9)])
        st, w, h, c, ofs, ln = info(png)
        assert (st, w, h, c, ln) == (0, 31, 17, 4, len(z)), split
        assert png[ofs + 4:ofs + 8] == b"IDAT" and ofs == 8 + 25 + 21


def test_fpng_files_keep_get_info_ex_rows(oracle):
    import fpng_b200
    for i, (kind, w, h, c) in enumerate([("g1", 40, 6, 3), ("g0", 200, 20, 4), ("runs", 300, 7, 3), ("g2", 31, 9, 4)]):
        png = oracle.encode(imagegen.make(kind, w, h, c, i), w, h, c, 0)
        assert info(png) == fpng_b200.get_info_ex(png)
        assert info(png)[0] == 0


def test_writer_and_unfilter_model_match_pil():
    from PIL import Image
    for c, mode in ((1, "L"), (2, "LA"), (3, "RGB"), (4, "RGBA")):
        for filters in ("random", 0, 1, 2, 3, 4):
            img = pngwrite.source("g1", 23, 11, c, c)
            png = pngwrite.make_png(img, filters=filters, split="random")
            pil = np.asarray(Image.open(io.BytesIO(png)))
            assert Image.open(io.BytesIO(png)).mode == mode
            np.testing.assert_array_equal(pil.reshape(img.shape), img)
            raw = zlib.decompress(b"".join(pngwrite.split_idat(pngwrite.compress(pngwrite.filter_rows(
                img, pngwrite.row_filters(11, filters))))))
            np.testing.assert_array_equal(pngwrite.unfilter(raw, 23, 11, c), img)
            for d, conv in ((3, "RGB"), (4, "RGBA")):
                np.testing.assert_array_equal(np.asarray(Image.open(io.BytesIO(png)).convert(conv)), pngwrite.expand(img, d))


def test_golden_files_agree_with_pil():
    from PIL import Image
    with open(os.path.join(GOLDEN, "manifest.json")) as f:
        manifest = json.load(f)
    modes = {1: "L", 2: "LA", 3: "RGB", 4: "RGBA"}
    for m in manifest:
        data = open(os.path.join(GOLDEN, m["file"]), "rb").read()
        im = Image.open(io.BytesIO(data))
        st, w, h, c, ofs, ln = info(data)
        assert (st, w, h, c) == (0, m["w"], m["h"], m["chans"]), m["file"]
        assert im.size == (w, h) and im.mode == modes[c], m["file"]
        img = pngwrite.source(m["kind"], m["w"], m["h"], m["chans"], m["index"])
        np.testing.assert_array_equal(np.asarray(im).reshape(img.shape), img)
        assert struct.unpack(">I", data[ofs:ofs + 4])[0] <= ln
