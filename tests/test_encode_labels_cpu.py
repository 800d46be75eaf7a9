"""The label-map PNG format (DESIGN §4.6 "Label maps") on the oracle: PIL reads every corpus file back to its ids, palette and
transparency; each case reaches the construct it names; the slot bound holds; encode_labels_device's argument errors."""
from __future__ import annotations

import io
import zlib

import numpy as np
import pytest
from PIL import Image

import deflatetrace
from label_encode_cases import cases

CASES = cases()


@pytest.fixture(scope="module")
def penc():
    from label_oracle import LabelOracle
    return LabelOracle()


def chunks(f):
    out, p = [], 8
    while p < len(f):
        n = int.from_bytes(f[p:p + 4], "big")
        kind, data = f[p + 4:p + 8], f[p + 8:p + 8 + n]
        assert zlib.crc32(kind + data) == int.from_bytes(f[p + 8 + n:p + 12 + n], "big"), kind
        out.append((kind, data))
        p += 12 + n
    return out


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_pil_reads_oracle_file(penc, case):
    f = penc.label_encode(case.ids, case.depth, case.palette, case.flags)
    im = Image.open(io.BytesIO(f))
    im.load()                                                            # PIL checks every chunk CRC on load
    h, w = case.ids.shape
    assert im.size == (w, h)
    kinds = [k for k, _ in chunks(f)]
    assert kinds[0] == b"IHDR" and kinds[-2:] == [b"IDAT", b"IEND"] and kinds.count(b"IDAT") == 1
    ihdr = chunks(f)[0][1]
    assert ihdr[8] == case.depth and ihdr[9] == (0 if case.palette is None else 3) and ihdr[10:] == b"\0\0\0"
    if case.palette is not None:
        assert im.mode == "P" and np.array_equal(np.asarray(im).astype(np.int64), case.ids)
        k = len(case.palette)
        assert np.array_equal(np.array(im.getpalette()[:3 * k], np.uint8).reshape(k, 3), case.palette[:, :3])
        alpha = case.palette[:, 3] if case.palette.shape[1] == 4 else np.full(k, 255, np.uint8)
        t = int(np.nonzero(alpha != 255)[0][-1]) + 1 if (alpha != 255).any() else 0
        assert kinds[1] == b"PLTE" and (b"tRNS" in kinds) == (t > 0)
        if t:
            assert im.info["transparency"] == alpha[:t].tobytes()
        else:
            assert "transparency" not in im.info
    elif case.depth in (1, 8):
        got = np.asarray(im).astype(np.int64)
        assert np.array_equal(got, case.ids), case.name
    else:
        # every other gray depth: the IDAT inflates to the packed rows (filters undone by PIL above is not exposed for 2/4/16)
        assert im.mode in ("L", "I", "I;16", "I;16B")


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_reaches_its_construct(penc, case):
    f = penc.label_encode(case.ids, case.depth, case.palette, case.flags)
    cs = chunks(f)
    idat = [d for k, d in cs if k == b"IDAT"][0]
    tr = deflatetrace.trace(idat)
    h, w = case.ids.shape
    rowbytes = w * 2 if case.depth == 16 else (w * case.depth + 7) // 8
    assert len(tr.data) == h * (rowbytes + 1)
    stored = all(b.btype == 0 for b in tr.blocks)
    if case.reaches in ("stored", "forced"):
        assert stored, case.name
        assert all(tr.data[y * (rowbytes + 1)] == 0 for y in range(h))  # filter 0 on every row
    else:
        assert not stored and [b.btype for b in tr.blocks] == [2], case.name
    if case.reaches == "residue" or case.depth < 8:
        r = (w * case.depth) % 8
        if r:                                                             # the last byte's unused low bits are zero
            raw = penc.label_encode(case.ids, case.depth, case.palette, FORCE := 2)
            data = deflatetrace.trace([d for k, d in chunks(raw) if k == b"IDAT"][0]).data
            last = np.frombuffer(data, np.uint8).reshape(h, rowbytes + 1)[:, -1]
            assert (last & ((1 << (8 - r)) - 1) == 0).all(), (case.name, FORCE)
    kinds = [k for k, _ in cs]
    if case.reaches == "trns-trimmed":
        t = dict(cs)[b"tRNS"]
        assert len(t) == 8 and len(case.palette) == 21
    if case.reaches == "trns-present":
        assert len(dict(cs)[b"tRNS"]) == 21
    if case.reaches == "trns-absent":
        assert b"tRNS" not in kinds and case.palette.shape[1] == 4


def test_residues_and_palette_sizes_covered():
    res = {(c.depth, (c.ids.shape[1] * c.depth) % 8) for c in CASES if c.reaches == "residue"}
    assert res == {(d, r) for d in (1, 2, 4) for r in range(0, 8, d)}
    assert {len(c.palette) for c in CASES if c.reaches == "K"} >= {1, 2, 3, 4, 5, 16, 17, 256}
    assert {c.reaches for c in CASES} >= {"stored", "forced", "trns-trimmed", "trns-present", "trns-absent"}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_slot_bound_holds(penc, case):
    h, w = case.ids.shape
    bound = penc.label_bound(w, h, case.depth, case.palette)
    for flags in (0, 2):
        assert len(penc.label_encode(case.ids, case.depth, case.palette, flags)) <= bound


def test_out_of_range_has_no_file(penc):
    ids = np.zeros((4, 5), np.int64)
    ids[3, 4] = 4
    assert penc.label_encode(ids, 2, None) is None
    assert penc.label_encode(ids, 8, np.zeros((4, 3), np.uint8)) is None
    ids[3, 4] = -1
    assert penc.label_encode(ids, 8, None) is None


def test_python_argument_errors():
    import torch

    import fpng_b200 as g
    m = torch.zeros((4, 5), dtype=torch.uint8)
    pal = np.zeros((3, 3), np.uint8)
    bad = [
        dict(images=[m], depth=1),                                        # a CPU tensor
        dict(images=[], depth=1),
        dict(images=[m], palette=np.zeros((3, 2), np.uint8)),
        dict(images=[m], palette=np.zeros((0, 3), np.uint8)),
        dict(images=[m], palette=np.zeros((257, 3), np.uint8)),
        dict(images=[m], palette=np.zeros((3, 3), np.float32)),
        dict(images=[m], palette=[pal, pal]),
        dict(images=[m], depth=[1, 2]),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            g.encode_labels_device(**kw)
