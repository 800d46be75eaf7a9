"""GPU tests of the all-formats decode (FPNGB_PNG_ALL_FORMATS / FPNGB_RESIZE_ALL_PNG_FORMATS, all_formats=True): palette,
1/2/4/16-bit, color-keyed and Adam7 files decoded in the packed ragged and resized calls.  Files come from tests/pngwrite_formats.py
(every format, filter and padding) and tests/golden/anypng_formats (PIL and OpenCV); expected pixels from its numpy model, which
test_decode_png_formats_cpu.py pins against PIL, libpng, lodepng and wuffs."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

import pngwrite
import pngwrite_formats as pf
from pngwrite import IEND, SIG, chunk, ihdr
from test_decode_device_gpu import to_device
from test_decode_png_gpu import fpng_file
from test_decode_ragged_gpu import pack_at

pytestmark = pytest.mark.gpu

HEADER_CRC, INVALID_IDAT, ADLER, UNSUPPORTED = 4, 8, 102, 104
GUARD = 0xA5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "anypng_formats")


def run(gpu, files, d, rs=None, dtype=None, scale=None, bias=None, all_formats=True, any_png=True):
    """one ragged call (all bounds given, no host sync inside) into a guard-filled output; returns (views, status, info, raw)"""
    import torch
    rs = rs or np.random.RandomState(0)
    buf, offs = pack_at(files, rs, False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    infos = [gpu.get_png_info(f, all_formats=True) for f in files]
    mw = max([i[1] for i in infos] + [1])
    mh = max([i[2] for i in infos] + [1])
    es = 1 if dtype is None else torch.empty((), dtype=dtype).element_size()
    cap = max(16, sum((i[1] * i[2] * d * es + 15) // 16 * 16 for i in infos if i[0] == 0))
    raw = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out = raw[:cap].view(dtype) if es > 1 else raw[:cap]
    _, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=out, max_file_size=max(len(f) for f in files),
                                                      max_w=mw, max_h=mh, scale=scale, bias=bias, any_png=any_png,
                                                      all_formats=all_formats)
    torch.cuda.synchronize()
    return gpu.ragged_views(out, oo, info, st, d), st.cpu().numpy(), info.cpu().numpy(), raw


SHAPES = [(1, 1), (1, 2), (2, 1), (2, 2), (3, 3), (4, 5), (5, 4), (7, 9), (8, 8), (9, 7), (1, 17), (17, 1), (13, 17), (17, 17),
          (11, 3), (15, 16)]


def combo_cases(ctype, depth, il, t, seed):
    rs = np.random.RandomState(seed)
    out = [pf.case(rs, w, h, ctype, depth, il, t, seed=seed + k) for k, (w, h) in enumerate(SHAPES)]
    out += [pf.case(rs, 19, 11, ctype, depth, il, t, filters=ft, seed=seed + ft) for ft in range(5)]
    return out


@pytest.mark.parametrize("combo", pf.combos(), ids=lambda c: "t%d_d%d_i%d_%s" % (c[0], c[1], c[2], "trns" if c[3] else "plain"))
@pytest.mark.parametrize("d", [3, 4])
def test_every_format(gpu, combo, d):
    ctype, depth, il, t = combo
    cases = combo_cases(ctype, depth, il, t, 100 * ctype + depth + 7 * il + 3 * t)
    views, st, info, raw = run(gpu, [c[0] for c in cases], d)
    for k, (png, s, plte, trns) in enumerate(cases):
        h, w = s.shape[:2]
        assert st[k] == 0, (k, st[k])
        assert tuple(info[k][:4]) == (0, w, h, pf.info_chans(ctype, trns))
        np.testing.assert_array_equal(views[k].cpu().numpy(), pf.model_u8(s, ctype, depth, d, plte, trns), err_msg=str((k, w, h)))


@pytest.mark.parametrize("il", [0, 1])
def test_large_files(gpu, il):
    rs = np.random.RandomState(5 + il)
    cases = [pf.case(rs, 640, 480, ctype, depth, il, t, seed=k)
             for k, (ctype, depth, t) in enumerate([(3, 8, True), (3, 4, False), (0, 1, False), (0, 16, True), (2, 16, False), (6, 16, False),
                                                     (4, 8, False), (2, 8, True)])]
    for d in (3, 4):
        views, st, _, _ = run(gpu, [c[0] for c in cases], d)
        for k, (png, s, plte, trns) in enumerate(cases):
            f = pf.parse(png)
            assert st[k] == 0
            np.testing.assert_array_equal(views[k].cpu().numpy(), pf.model_u8(s, f["ctype"], f["depth"], d, plte, trns), err_msg=str(k))


@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
def test_typed_output(gpu, dtype):
    import torch
    T = getattr(torch, dtype)
    rs = np.random.RandomState(21)
    cases = []
    for k, (ctype, depth, il, t) in enumerate(pf.combos()):
        for (w, h) in [(3, 2), (9, 13)]:
            cases.append((ctype, depth) + pf.case(rs, w, h, ctype, depth, il, t, seed=k))
    for d in (3, 4):
        s_, b_ = [0.5, 1.0 / 255, 2.0, 0.25][:d], [-1.0, 0.0, 3.5, 0.125][:d]
        views, st, _, _ = run(gpu, [c[2] for c in cases], d, dtype=T, scale=s_, bias=b_)
        for k, (ctype, depth, png, s, plte, trns) in enumerate(cases):
            assert st[k] == 0
            v = torch.from_numpy(pf.model_values(s, ctype, depth, d, plte, trns))
            want = (v * torch.tensor(s_) + torch.tensor(b_)).to(T)
            assert torch.equal(views[k].cpu(), want), (dtype, d, k, ctype, depth)


def test_16bit_float_rule(gpu):
    """v = s / 257: every 16-bit value is recovered from float32 output, and 257 * k decodes to exactly k"""
    import torch
    s = np.arange(65536, dtype=np.uint32).reshape(256, 256, 1)
    files = [pf.make_png(s, 0, 16, il) for il in (0, 1)]
    k = (np.arange(256, dtype=np.uint32) * 257).reshape(16, 16, 1)
    files.append(pf.make_png(k, 0, 16))
    views, st, _, _ = run(gpu, files, 3, dtype=torch.float32)
    assert (st == 0).all()
    for i in (0, 1):
        v = views[i].cpu().numpy()[..., 0]
        assert np.array_equal(np.round(v * np.float32(257.0)).astype(np.int64), s[..., 0].astype(np.int64))
    assert np.array_equal(views[2].cpu().numpy()[..., 1], np.arange(256, dtype=np.float32).reshape(16, 16))


def test_edge_cases(gpu):
    rs = np.random.RandomState(3)
    # palette index past the entries: (0, 0, 0), alpha 255 past the short tRNS
    s = rs.randint(0, 16, (9, 11, 1)).astype(np.uint32)
    plte = rs.randint(0, 256, (5, 3)).astype(np.uint8)
    trns = bytes([10, 20])
    oor = pf.make_png(s, 3, 4, 0, plte, trns)
    oor_i = pf.make_png(s, 3, 4, 1, plte, trns)
    # a 16-bit key that matches only in its high byte: opaque
    g = np.array([[[0x1234], [0x1299], [0x1234]]], np.uint32)
    key = pf.make_png(g, 0, 16, trns=struct.pack(">H", 0x1234 ^ 0x00FF))
    key_hit = pf.make_png(g, 0, 16, trns=struct.pack(">H", 0x1234))
    rgb = np.array([[[0x0102, 0x0304, 0x0506], [0x0102, 0x0304, 0x05FF]]], np.uint32)
    key_rgb = pf.make_png(rgb, 2, 16, trns=struct.pack(">HHH", 0x0102, 0x0304, 0x0506))
    # a key above the depth never matches
    g8 = np.array([[[0], [255]]], np.uint32)
    key_big = pf.make_png(g8, 0, 8, trns=struct.pack(">H", 0x100))
    views, st, _, _ = run(gpu, [oor, oor_i, key, key_hit, key_rgb, key_big], 4)
    assert list(st) == [0] * 6
    want = pf.model_u8(s, 3, 4, 4, plte, trns)
    assert (want[s[..., 0] >= 5] == [0, 0, 0, 255]).all()
    for i in (0, 1):
        np.testing.assert_array_equal(views[i].cpu().numpy(), want)
    assert views[2].cpu().numpy()[0, :, 3].tolist() == [255, 255, 255]
    assert views[3].cpu().numpy()[0, :, 3].tolist() == [0, 255, 0]
    assert views[4].cpu().numpy()[0, :, 3].tolist() == [0, 255]
    assert views[5].cpu().numpy()[0, :, 3].tolist() == [255, 255]


def bad_streams():
    """(name, png): ext files whose stream breaks a rule after the inflate"""
    rs = np.random.RandomState(8)
    s = rs.randint(0, 4, (13, 17, 1)).astype(np.uint32)
    plte = rs.randint(0, 256, (4, 3)).astype(np.uint8)
    raw = bytearray(pf.raw_stream(s, 3, 2, 1))
    # the first row of pass 7 (y0 = 1, 7 rows of 1 + ceil(17 * 2 / 8) bytes): its filter byte
    at = sum(ph * (1 + (pw * 2 + 7) // 8) for (_, _, _, _, pw, ph) in pf.passes(17, 13, 1)[:6])
    bad7 = bytearray(raw)
    bad7[at] = 5
    bad7_last = bytearray(raw)
    bad7_last[len(raw) - 1 - (17 * 2 + 7) // 8] = 9
    return {"pass7 filter": pf.make_png(s, 3, 2, 1, plte, z=zlib.compress(bytes(bad7))),
            "pass7 last row filter": pf.make_png(s, 3, 2, 1, plte, z=zlib.compress(bytes(bad7_last))),
            "one byte short": pf.make_png(s, 3, 2, 1, plte, z=zlib.compress(bytes(raw[:-1]))),
            "one byte long": pf.make_png(s, 3, 2, 1, plte, z=zlib.compress(bytes(raw) + b"\0")),
            "16-bit short": pf.make_png(s, 0, 16, 0, z=zlib.compress(pf.raw_stream(s, 0, 16)[:-1]))}


def test_bad_streams(gpu):
    cases = bad_streams()
    good = pf.case(np.random.RandomState(1), 9, 9, 3, 2, 1)
    files = list(cases.values()) + [good[0]]
    for d in (3, 4):
        views, st, info, raw = run(gpu, files, d)
        assert list(st) == [INVALID_IDAT] * len(cases) + [0], st
        # every file is placed (17 x 13 each, then the good 9 x 9 one); only the good file's bytes are written
        r = raw.cpu().numpy()
        at = len(cases) * ((17 * 13 * d + 15) // 16 * 16)
        assert (r[:at] == GUARD).all() and (r[at + 9 * 9 * d:] == GUARD).all()
        np.testing.assert_array_equal(views[-1].cpu().numpy(), pf.model_u8(good[1], 3, 2, d, good[2], good[3]))


def test_mixed_batch_flag_on_off(gpu):
    rs = np.random.RandomState(17)
    items = []
    for k in range(6):
        png, img = fpng_file(gpu, int(rs.randint(1, 60)), int(rs.randint(1, 30)), 3 + k % 2, k)
        items.append(("fpng", png, img))
    for k in range(6):
        img = pngwrite.source("g1", int(rs.randint(1, 40)), int(rs.randint(1, 20)), 1 + k % 4, k)
        items.append(("png", pngwrite.make_png(img, seed=k), img))
    for k, (ctype, depth, il, t) in enumerate(pf.combos()[::3]):
        png, s, plte, trns = pf.case(rs, int(rs.randint(1, 30)), int(rs.randint(1, 30)), ctype, depth, il, t, seed=k)
        items.append(("ext", png, (s, ctype, depth, plte, trns)))
    items.append(("bad", bad_streams()["pass7 filter"], None))
    items.append(("bad8", pngwrite.make_png(pngwrite.source("g1", 8, 8, 3), z=zlib.compress(b"\0" * 10)), None))
    rs.shuffle(items)
    files = [it[1] for it in items]
    for d in (3, 4):
        on_v, on_st, _, _ = run(gpu, files, d, rs=np.random.RandomState(d))
        off_v, off_st, _, _ = run(gpu, files, d, rs=np.random.RandomState(d), all_formats=False)
        for k, (kind, png, ref) in enumerate(items):
            if kind in ("fpng", "png"):
                assert on_st[k] == off_st[k] == 0
                assert np.array_equal(on_v[k].cpu().numpy(), off_v[k].cpu().numpy())
            elif kind == "ext":
                s, ctype, depth, plte, trns = ref
                ext = depth != 8 or pf.parse(png)["interlace"] or ctype == 3 or trns is not None
                assert on_st[k] == 0 and off_st[k] == (UNSUPPORTED if ext else 0)
                np.testing.assert_array_equal(on_v[k].cpu().numpy(), pf.model_u8(s, ctype, depth, d, plte, trns))
            elif kind == "bad":
                assert on_st[k] == INVALID_IDAT and off_st[k] == UNSUPPORTED
            else:
                assert on_st[k] == off_st[k] == INVALID_IDAT


def test_verify(gpu):
    rs = np.random.RandomState(4)
    good = [pf.case(rs, 11, 7, ctype, depth, il, t, seed=k)[0] for k, (ctype, depth, il, t) in enumerate(pf.combos()[::4])]
    g = good[0]
    ofs = gpu.get_png_info(g, all_formats=True)[4]
    n = struct.unpack(">I", g[ofs:ofs + 4])[0]
    bad_crc = bytearray(g)
    bad_crc[ofs + 8 + n] ^= 1                                                # the IDAT chunk's CRC
    zz = zlib.compress(pf.raw_stream(np.zeros((7, 11, 1), np.uint32), 0, 16))
    bad_adler = pf.make_png(np.zeros((7, 11, 1), np.uint32), 0, 16, z=zz[:-4] + bytes([zz[-4] ^ 1]) + zz[-3:])
    raw = bytearray(pf.raw_stream(np.zeros((7, 11, 1), np.uint32), 0, 16))
    raw[0] = 7
    zb = zlib.compress(bytes(raw))
    bad_both = pf.make_png(np.zeros((7, 11, 1), np.uint32), 0, 16, z=zb[:-4] + bytes([zb[-4] ^ 1]) + zb[-3:])
    files = good + [bytes(bad_crc), bad_adler, bad_both]
    gpu.set_decode_verify(True)
    try:
        n0 = gpu.launch_count()
        _, st, _, _ = run(gpu, files, 4)
        assert gpu.launch_count() - n0 == 17
    finally:
        gpu.set_decode_verify(False)
    assert list(st) == [0] * len(good) + [HEADER_CRC, ADLER, INVALID_IDAT], st
    _, st, _, _ = run(gpu, files, 4)
    assert list(st) == [0] * len(good) + [0, 0, INVALID_IDAT]


def test_launch_counts_and_flags(gpu):
    import torch
    import ctypes as C
    from fpng_b200._lib import lib
    rs = np.random.RandomState(2)
    files = [pf.case(rs, 9, 5, 3, 8)[0], pf.case(rs, 9, 5, 0, 16, 1)[0]]
    n0 = gpu.launch_count()
    _, st, _, _ = run(gpu, files, 3, all_formats=False)
    assert (st == UNSUPPORTED).all() and gpu.launch_count() - n0 == 14
    n0 = gpu.launch_count()
    _, st, _, _ = run(gpu, files, 3)
    assert (st == 0).all() and gpu.launch_count() - n0 == 15
    buf, offs = pack_at(files, rs, False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    info = torch.empty((2, 6), dtype=torch.int32, device="cuda")
    out = torch.empty(1024, dtype=torch.uint8, device="cuda")
    oo = torch.empty(3, dtype=torch.int64, device="cuda")
    stt = torch.empty(2, dtype=torch.int32, device="cuda")
    n0 = gpu.launch_count()
    for flags in (2, 3, 0x100):
        assert lib().fpngb_get_png_info_batch_device_ex(data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), 2, flags, info.data_ptr(),
                                                        None) == 1
        assert lib().fpngb_decode_packed_png_device_ex(data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), 2, 4096, 64,
                                                       64, 3, out.data_ptr(), 1024, oo.data_ptr(), info.data_ptr(), flags, None,
                                                       stt.data_ptr(), None) == 1
    assert gpu.launch_count() == n0
    on = gpu.get_info_batch_device(data, offsets, sizes, any_png=True, all_formats=True).cpu().numpy()
    assert [tuple(r) for r in on] == [gpu.get_png_info(f, all_formats=True) for f in files]
    off = gpu.get_info_batch_device(data, offsets, sizes, any_png=True).cpu().numpy()
    assert list(off[:, 0]) == [UNSUPPORTED, UNSUPPORTED]


def test_resized_all_formats(gpu):
    """the resized call reads the uint8 values: a 16-bit file resizes exactly as the 8-bit file of its high bytes"""
    import torch
    rs = np.random.RandomState(6)
    s16 = rs.randint(0, 65536, (37, 53, 4)).astype(np.uint32)
    f16 = pf.make_png(s16, 6, 16, 1)
    f8 = pngwrite.make_png((s16 >> 8).astype(np.uint8))
    p, s, plte, trns = pf.case(rs, 53, 37, 3, 4, 1, True)
    f_pal = p
    files = [f16, f8, f_pal, pngwrite.make_png(pf.model_u8(s, 3, 4, 4, plte, trns))]
    buf, offs = pack_at(files, rs, False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    for dt in (torch.uint8, torch.float32):
        n0 = gpu.launch_count()
        out, info, st = gpu.decode_packed_resized_device(data, offsets, sizes, (20, 30), 4, any_png=True, all_formats=True, dtype=dt,
                                                         max_file_size=max(len(f) for f in files), max_w=53, max_h=37,
                                                         pixel_cap=4 * 53 * 37 * 4 + 64)
        torch.cuda.synchronize()
        assert gpu.launch_count() - n0 == 16
        assert (st.cpu().numpy() == 0).all()
        o = out.cpu()
        assert torch.equal(o[0], o[1]) and torch.equal(o[2], o[3])
    _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (20, 30), 4, any_png=True, max_file_size=max(len(f) for f in files),
                                                max_w=53, max_h=37, pixel_cap=4 * 53 * 37 * 4 + 64)
    assert list(st.cpu().numpy()) == [UNSUPPORTED, 0, UNSUPPORTED, 0]


def test_streams_no_sync(gpu):
    """two all-formats calls on two streams overlap, with every bound given (no host synchronisation inside the calls)"""
    import torch
    rs = np.random.RandomState(12)
    halves = []
    for h in range(2):
        cs = []
        for k in range(300):
            ctype, depth, il, t = pf.combos()[k % len(pf.combos())]
            cs.append(pf.case(rs, int(rs.randint(1, 40)), int(rs.randint(1, 40)), ctype, depth, il, t, seed=k))
        halves.append(cs)
    packs = []
    for cs in halves:
        fs = [c[0] for c in cs]
        buf, offs = pack_at(fs, rs, False)
        packs.append(to_device(buf, offs, [len(f) for f in fs]))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    res = []
    for (data, offsets, sizes), s, cs in zip(packs, (s1, s2), halves):
        with torch.cuda.stream(s):
            out = torch.empty((40 * 40 * 4 + 16) * len(cs), dtype=torch.uint8, device="cuda")
            res.append(gpu.decode_packed_ragged_device(data, offsets, sizes, 4, out=out, max_file_size=max(len(c[0]) for c in cs),
                                                       max_w=40, max_h=40, any_png=True, all_formats=True))
    torch.cuda.synchronize()
    for (out, oo, info, st), cs in zip(res, halves):
        assert (st.cpu().numpy() == 0).all()
        vs = gpu.ragged_views(out, oo, info, st, 4)
        for k in range(0, len(cs), 3):
            png, s, plte, trns = cs[k]
            f = pf.parse(png)
            np.testing.assert_array_equal(vs[k].cpu().numpy(), pf.model_u8(s, f["ctype"], f["depth"], 4, plte, trns))


def golden():
    with open(os.path.join(GOLDEN, "manifest.json")) as f:
        manifest = json.load(f)
    return [open(os.path.join(GOLDEN, m["file"]), "rb").read() for m in manifest]


@pytest.mark.parametrize("d", [3, 4])
def test_golden_files(gpu, d):
    import torch
    files = golden()
    views, st, _, _ = run(gpu, files, d)
    assert (st == 0).all()
    fviews, fst, _, _ = run(gpu, files, d, dtype=torch.float32)
    assert (fst == 0).all()
    for k, png in enumerate(files):
        f = pf.parse(png)
        np.testing.assert_array_equal(views[k].cpu().numpy(), pf.model_u8(f["samples"], f["ctype"], f["depth"], d, f["plte"], f["trns"]))
        v = pf.model_values(f["samples"], f["ctype"], f["depth"], d, f["plte"], f["trns"])
        assert np.array_equal(fviews[k].cpu().numpy(), v)
