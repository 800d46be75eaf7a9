"""GPU tests of the general-PNG decode (fpngb_decode_packed_png_device, FPNGB_RESIZE_ANY_PNG): PNGs from any zlib stream decoded
in the packed ragged and resized calls.  Expected pixels are the source images (tests/pngwrite.py writes the files from numpy and
zlib; tests/golden/anypng holds libpng- and PIL-written files of seeded imagegen images), or for corrupted streams zlib's output
run through the numpy unfilter model.  fpng files in the same call must decode exactly as without any_png."""
import json
import os
import struct
import zlib

import numpy as np
import pytest

import pngwrite
from pngwrite import IEND, SIG, chunk, ihdr
from test_decode_device_gpu import to_device
from test_decode_ragged_gpu import pack_at
from test_decode_resized_gpu import corpus as resized_corpus

pytestmark = pytest.mark.gpu

NOT_FPNG, HEADER_CRC, INVALID_IDAT, OUT_OF_SPACE, ADLER, UNSUPPORTED = 1, 4, 8, 101, 102, 104
PENDING = 0x7FFFFFF0
GUARD = 0xA5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "anypng")


def run(gpu, files, d, rs=None, out_cap=None, dtype=None, scale=None, bias=None, any_png=True):
    """one ragged call (all bounds given) over files packed at random 4-byte-aligned offsets into a guard-filled output;
    returns (views or None per file, status, info, out_offsets, out tensor)"""
    import torch
    rs = rs or np.random.RandomState(0)
    buf, offs = pack_at(files, rs, False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    infos = [gpu.get_png_info(f) for f in files]
    mw = max([i[1] for i in infos] + [1])
    mh = max([i[2] for i in infos] + [1])
    es = 1 if dtype is None else torch.empty((), dtype=dtype).element_size()
    if out_cap is None:
        out_cap = max(16, sum((i[1] * i[2] * d * es + 15) // 16 * 16 for i in infos if i[0] == 0))
    odt = torch.uint8 if dtype is None else dtype
    raw = torch.full((out_cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out = raw[:out_cap].view(odt) if es > 1 else raw[:out_cap]
    _, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, out=out, max_file_size=max(len(f) for f in files),
                                                      max_w=mw, max_h=mh, scale=scale, bias=bias, any_png=any_png)
    torch.cuda.synchronize()
    views = gpu.ragged_views(out, oo, info, st, d)
    return views, st.cpu().numpy(), info.cpu().numpy(), oo.cpu().numpy().view(np.uint64), raw


def check_pixels(gpu, cases, d):
    """cases: [(png, expected [h, w, c] image)]; every file decodes with status 0 to expand(image, d)"""
    views, st, info, _, _ = run(gpu, [c[0] for c in cases], d)
    for k, (png, img) in enumerate(cases):
        assert st[k] == 0, (k, st[k])
        assert tuple(info[k][:4]) == (0, img.shape[1], img.shape[0], img.shape[2])
        np.testing.assert_array_equal(views[k].cpu().numpy(), pngwrite.expand(img, d), err_msg=str(k))


def corpus():
    out = []
    shapes = [(1, 1), (1, 9), (9, 1), (13, 7), (31, 3), (1000, 7), (7, 1000), (640, 480)]
    k = 0
    for (w, h) in shapes:
        for c in (1, 2, 3, 4):
            if w * h > 10000 and c != 3:
                continue
            img = pngwrite.source(("g1", "g0", "runs")[k % 3], w, h, c, k)
            out.append((pngwrite.make_png(img, seed=k), img))
            k += 1
    img = pngwrite.source("g1", 41, 13, 3, 5)
    for filters in (0, 1, 2, 3, 4):
        out.append((pngwrite.make_png(img, filters=filters), img))
    for level in (0, 1, 6, 9):
        for strategy in pngwrite.STRATEGIES:
            c = 1 + (level + len(strategy)) % 4
            im = pngwrite.source("g1", 57, 19, c, level)
            out.append((pngwrite.make_png(im, level=level, strategy=strategy, seed=level), im))
    for wbits in range(9, 16):
        im = pngwrite.source("runs", 300, 11, 4, wbits)
        out.append((pngwrite.make_png(im, wbits=wbits, level=9), im))
    big = pngwrite.source("g1", 200, 40, 3, 3)
    n = 40 * 601
    for mode in (zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
        out.append((pngwrite.make_png(big, flush=(mode, [n // 5, n // 2, n // 2 + 1])), big))
    for split in ("bytes", "random", "zeros", 8192):
        out.append((pngwrite.make_png(big if split != "bytes" else img, split=split), big if split != "bytes" else img))
    out.append((pngwrite.make_png(img, before=[chunk(b"PLTE", b"\1\2\3" * 5), chunk(b"gAMA", b"\0\1\x86\xa0")],
                                  between=[], after=[chunk(b"tEXt", b"k\0v"), chunk(b"PLTE", b"\4\5\6")]), img))
    return out


@pytest.mark.parametrize("d", [3, 4])
def test_hand_written_corpus(gpu, d):
    check_pixels(gpu, corpus(), d)


def golden():
    with open(os.path.join(GOLDEN, "manifest.json")) as f:
        manifest = json.load(f)
    return [(open(os.path.join(GOLDEN, m["file"]), "rb").read(), pngwrite.source(m["kind"], m["w"], m["h"], m["chans"], m["index"]))
            for m in manifest]


@pytest.mark.parametrize("d", [3, 4])
def test_real_encoder_output(gpu, d):
    check_pixels(gpu, golden(), d)


@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
def test_typed_output(gpu, dtype):
    import torch
    T = getattr(torch, dtype)
    cases = corpus()[:20] + golden()[:10]
    for d in (3, 4):
        s, b = [0.5, 1.0 / 255, 2.0, 0.25][:d], [-1.0, 0.0, 3.5, 0.125][:d]
        views, st, _, _, _ = run(gpu, [c[0] for c in cases], d, dtype=T, scale=s, bias=b)
        for k, (_, img) in enumerate(cases):
            assert st[k] == 0
            u8 = torch.from_numpy(pngwrite.expand(img, d))
            want = (u8.float() * torch.tensor(s) + torch.tensor(b)).to(T)
            assert torch.equal(views[k].cpu(), want), (dtype, d, k)


def fpng_file(gpu, w, h, c, k):
    import imagegen
    img = imagegen.make(("g1", "g0", "runs")[k % 3], w, h, c, k)
    ok, png = gpu.fpng_encode_image_to_memory(img, w, h, c)
    assert ok
    return png, img


def test_mixed_batch(gpu):
    rs = np.random.RandomState(7)
    items = []
    for k in range(12):
        png, img = fpng_file(gpu, int(rs.randint(1, 90)), int(rs.randint(1, 40)), 3 + k % 2, k)
        items.append(("fpng", png, img))
    for k, (png, img) in enumerate(corpus()[:30:2]):
        items.append(("png", png, img))
    bad = pngwrite.make_png(pngwrite.source("g1", 8, 8, 3), z=zlib.compress(b"\0" * 10))
    items += [("bad", bad, None), ("bad", SIG + ihdr(4, 4, depth=16) + chunk(b"IDAT", b"xx") + IEND + b"\0" * 20, None)]
    rs.shuffle(items)
    files = [it[1] for it in items]
    for d in (3, 4):
        views, st, info, oo, raw = run(gpu, files, d, rs=np.random.RandomState(d))
        ref_views, ref_st, _, _, _ = run(gpu, files, d, rs=np.random.RandomState(d), any_png=False)
        at = 0
        for k, (kind, png, img) in enumerate(items):
            if kind == "fpng":
                assert st[k] == ref_st[k] == 0
                assert np.array_equal(views[k].cpu().numpy(), ref_views[k].cpu().numpy())
            elif kind == "png":
                assert st[k] == 0 and ref_st[k] == NOT_FPNG
                np.testing.assert_array_equal(views[k].cpu().numpy(), pngwrite.expand(img, d))
            else:
                assert st[k] in (INVALID_IDAT, UNSUPPORTED) and ref_st[k] == NOT_FPNG
            assert oo[k] == at
            if info[k][0] == 0:
                at += (int(info[k][1]) * int(info[k][2]) * d + 15) // 16 * 16
        assert oo[-1] == at
        r = raw.cpu().numpy()
        mask = np.ones(r.size, bool)
        for k in range(len(items)):
            if st[k] == 0:
                mask[int(oo[k]):int(oo[k]) + int(info[k][1]) * int(info[k][2]) * d] = False
        assert (r[mask] == GUARD).all()
        assert not (st == PENDING).any()
    # a small out_cap: a suffix of the placed files gets OUT_OF_SPACE
    views, st, info, oo, _ = run(gpu, files, 4, out_cap=int(oo[-1]) // 2)
    placed = [k for k in range(len(items)) if info[k][0] == 0]
    oos = [st[k] == OUT_OF_SPACE for k in placed]
    assert any(oos) and oos == sorted(oos)


def stream_cases():
    """(name, png): streams every decoder must reject with FAILED_INVALID_IDAT"""
    img = pngwrite.source("g1", 17, 9, 3)
    raw = pngwrite.filter_rows(img, pngwrite.row_filters(9, "random"))
    z = zlib.compress(raw, 9)
    cases = {
        "truncated": z[:len(z) // 2],
        "extra output": zlib.compress(raw + b"\0"),
        "short output": zlib.compress(raw[:-1]),
        "filter byte 5": zlib.compress(b"\5" + raw[1:]),
        "fdict": bytes([0x78, 0xBB]) + z[2:],
        "bad fcheck": bytes([0x78, 0x9D]) + z[2:],
        "cm 7": bytes([0x77]) + z[1:],
        # a fixed block whose first symbol is a match of distance 1 (nothing written yet): 0x78 0x01, then BFINAL 1, BTYPE 01,
        # length code 257 (0000001), distance code 0 (00000)
        "distance too far": bytes([0x78, 0x01]) + bytes(pack_bits([(1, 1), (1, 2), (rev(0b0000001, 7), 7), (0, 5), (0, 7)])),
        "block type 3": bytes([0x78, 0x01, 0x07, 0, 0, 0, 0]),
    }
    return {k: pngwrite.make_png(img, z=v) for k, v in cases.items()}


def rev(v, n):
    return int(format(v, f"0{n}b")[::-1], 2)


def pack_bits(fields):
    acc, nb, out = 0, 0, []
    for v, n in fields:
        acc |= v << nb
        nb += n
    while nb > 0:
        out.append(acc & 255)
        acc >>= 8
        nb -= 8
    return out


def test_bad_streams(gpu):
    cases = stream_cases()
    _, st, _, _, _ = run(gpu, list(cases.values()), 4)
    for (name, _), s in zip(cases.items(), st):
        assert s == INVALID_IDAT, name


def test_unsupported(gpu):
    body = chunk(b"IDAT", zlib.compress(b"\0" * 20))
    files = [SIG + ihdr(4, 4, *f) + body + IEND for f in ([16, 2, 0, 0, 0], [8, 3, 0, 0, 0], [4, 0, 0, 0, 0], [8, 2, 0, 0, 1],
                                                          [1, 0, 0, 0, 0], [8, 6, 1, 0, 0], [8, 6, 0, 1, 0])]
    files.append(SIG + ihdr(4, 4) + chunk(b"tRNS", b"\0\1\0\2\0\3") + body + IEND)
    files.append(SIG + ihdr(4, 4) + chunk(b"ABCD", b"") + body + IEND)
    _, st, _, _, _ = run(gpu, files, 3)
    assert (st == UNSUPPORTED).all(), st


def test_bit_flips_match_zlib(gpu):
    rs = np.random.RandomState(3)
    files, want = [], []
    for k in range(300):
        c = 1 + k % 4
        w, h = int(rs.randint(1, 12)), int(rs.randint(1, 8))
        img = pngwrite.source(("g1", "runs")[k % 2], w, h, c, k)
        raw = pngwrite.filter_rows(img, pngwrite.row_filters(h, "random", k))
        z = bytearray(pngwrite.compress(raw, level=int(rs.randint(0, 10)), strategy=list(pngwrite.STRATEGIES)[k % 5]))
        pos = int(rs.randint(2, max(3, len(z) - 4)))
        z[pos] ^= 1 << int(rs.randint(0, 8))
        do = zlib.decompressobj(-15)
        try:
            out = do.decompress(bytes(z[2:]))
            ok = do.eof and len(out) == h * (w * c + 1)
        except zlib.error:
            ok = False
        exp = pngwrite.unfilter(out, w, h, c) if ok else None
        files.append(pngwrite.make_png(img, z=bytes(z)))
        want.append(exp)
    for d in (3, 4):
        views, st, _, _, _ = run(gpu, files, d)
        for k, exp in enumerate(want):
            if exp is None:
                assert st[k] == INVALID_IDAT, k
            else:
                assert st[k] == 0, k
                np.testing.assert_array_equal(views[k].cpu().numpy(), pngwrite.expand(exp, d))


def test_verify(gpu):
    img = pngwrite.source("g1", 50, 20, 4)
    z = pngwrite.compress(pngwrite.filter_rows(img, pngwrite.row_filters(20, "random")))
    good = pngwrite.make_png(img, z=z, split=100)
    parts = [chunk(b"IDAT", p) for p in pngwrite.split_idat(z, 100)]
    mid = len(parts) // 2
    bad_crc = SIG + ihdr(50, 20, ctype=6) + b"".join(parts[:mid]) + parts[mid][:-1] + bytes([parts[mid][-1] ^ 1]) + \
        b"".join(parts[mid + 1:]) + IEND
    bad_adler = pngwrite.make_png(img, z=z[:-1] + bytes([z[-1] ^ 1]))
    no_adler = pngwrite.make_png(img, z=z[:-4])
    files = [good, bad_crc, bad_adler, no_adler]
    try:
        gpu.set_decode_verify(True)
        views, st, _, _, _ = run(gpu, files, 4)
        assert list(st) == [0, HEADER_CRC, ADLER, ADLER]
        np.testing.assert_array_equal(views[0].cpu().numpy(), img)
    finally:
        gpu.set_decode_verify(False)
    views, st, _, _, _ = run(gpu, files, 4)
    assert list(st) == [0, 0, 0, 0]
    for v in views:
        np.testing.assert_array_equal(v.cpu().numpy(), img)


def test_any_png_off_is_untouched(gpu):
    files = [c[0] for c in corpus()[:8]]
    n0 = gpu.launch_count()
    _, st, _, _, _ = run(gpu, files, 3, any_png=False)
    assert (st == NOT_FPNG).all()
    assert gpu.launch_count() - n0 == 11
    n0 = gpu.launch_count()
    _, st, _, _, _ = run(gpu, files, 3)
    assert (st == 0).all()
    assert gpu.launch_count() - n0 == 14


def test_resized_any_png(gpu):
    import torch
    cases = corpus()[:24]
    files = [c[0] for c in cases]
    buf, offs = pack_at(files, np.random.RandomState(1), False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    # identity: every file is its own size, so resize to one common shape only for equal shapes; use 1x1 crops of a pixel
    rs = np.random.RandomState(2)
    boxes = []
    for png, img in cases:
        h, w = img.shape[:2]
        t, l = int(rs.randint(0, h)), int(rs.randint(0, w))
        boxes.append([t, l, 1, 1])
    bx = torch.tensor(boxes, dtype=torch.int32, device="cuda")
    for d in (3, 4):
        out, info, st = gpu.decode_packed_resized_device(data, offsets, sizes, (1, 1), d, boxes=bx, any_png=True)
        assert (st.cpu().numpy() == 0).all()
        o = out.cpu().numpy()
        for k, (png, img) in enumerate(cases):
            t, l = boxes[k][:2]
            np.testing.assert_array_equal(o[k, 0, 0], pngwrite.expand(img, d)[t, l])
        # planar float output of the same identity crops
        nchw = torch.empty((len(files), d, 1, 1), dtype=torch.float32, device="cuda").permute(0, 2, 3, 1)
        out2, _, st2 = gpu.decode_packed_resized_device(data, offsets, sizes, (1, 1), d, boxes=bx, any_png=True, out=nchw,
                                                        scale=[2.0] * d, bias=[1.0] * d)
        assert (st2.cpu().numpy() == 0).all()
        np.testing.assert_array_equal(out2.cpu().numpy(), o.astype(np.float32) * 2 + 1)
    # without any_png the general files are not decoded
    _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (1, 1), 3, boxes=bx, max_file_size=max(len(f) for f in files),
                                                max_w=1000, max_h=1000, pixel_cap=1 << 24)
    assert (st.cpu().numpy() == NOT_FPNG).all()


def test_resized_any_png_matches_model(gpu):
    import torch
    from test_decode_resized_gpu import check_values
    from test_decode_resized_cpu import resize_model
    img = pngwrite.source("g1", 97, 61, 3, 1)
    files = [pngwrite.make_png(img, seed=s) for s in range(4)]
    buf, offs = pack_at(files, np.random.RandomState(1), False)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    boxes = [[0, 0, 61, 97], [5, 7, 40, 33], [10, 0, 20, 97], [0, 50, 61, 47]]
    bx = torch.tensor(boxes, dtype=torch.int32, device="cuda")
    for dt in (torch.uint8, torch.float32):
        for aa in (True, False):
            out, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (32, 48), 3, boxes=bx, any_png=True, dtype=dt,
                                                          antialias=aa)
            assert (st.cpu().numpy() == 0).all()
            got = out.cpu().float().numpy()
            for k, b in enumerate(boxes):
                check_values(got[k], resize_model(img, 32, 48, aa, b), dt, [1.0] * 3, [0.0] * 3)


def test_scale_and_streams(gpu):
    import torch
    rs = np.random.RandomState(9)
    files, imgs = [], []
    for k in range(4096):
        c = 1 + k % 4
        img = pngwrite.source(("g1", "g0", "runs")[k % 3], int(rs.randint(1, 17)), int(rs.randint(1, 9)), c, k)
        files.append(pngwrite.make_png(img, seed=k, level=int(rs.randint(0, 10))))
        imgs.append(img)
    views, st, _, _, _ = run(gpu, files, 4)
    assert (st == 0).all()
    for k in range(0, 4096, 7):
        np.testing.assert_array_equal(views[k].cpu().numpy(), pngwrite.expand(imgs[k], 4))
    # two calls overlapping on two streams
    halves = [files[:2048], files[2048:]]
    packs = []
    for fs in halves:
        buf, offs = pack_at(fs, rs, False)
        packs.append(to_device(buf, offs, [len(f) for f in fs]))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    res = []
    for (data, offsets, sizes), s, fs in zip(packs, (s1, s2), halves):
        with torch.cuda.stream(s):
            out = torch.empty((sum((im.shape[0] * im.shape[1] * 4 + 15) // 16 * 16 for im in imgs),), dtype=torch.uint8, device="cuda")
            r = gpu.decode_packed_ragged_device(data, offsets, sizes, 4, out=out, max_file_size=max(len(f) for f in fs), max_w=16,
                                                max_h=8, any_png=True)
            res.append(r)
    torch.cuda.synchronize()
    for (out, oo, info, st), fs, base in zip(res, halves, (0, 2048)):
        assert (st.cpu().numpy() == 0).all()
        vs = gpu.ragged_views(out, oo, info, st, 4)
        for k in range(0, len(fs), 5):
            np.testing.assert_array_equal(vs[k].cpu().numpy(), pngwrite.expand(imgs[base + k], 4))


def test_resized_rejected_calls(gpu, oracle):
    """fpngb_decode_packed_resized_device's call-level checks next to FPNGB_RESIZE_ANY_PNG (4): the unknown bits 2 and 8 are still
    rejected, and ANY_PNG with or without FPNGB_RESIZE_ANTIALIAS is accepted"""
    import torch
    import ctypes as C
    from fpng_b200._lib import PixelFormat, lib
    files = resized_corpus(oracle)[:3]
    buf, offs = pack_at(files, np.random.RandomState(0), True)
    data, offsets, sizes = to_device(buf, offs, [len(f) for f in files])
    out = torch.full((3, 8, 8, 4), -5.0, dtype=torch.float32, device="cuda")
    st = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    info = torch.full((3, 6), -7, dtype=torch.int32, device="cuda")
    fmt = PixelFormat(); fmt.dtype = 1; fmt.scale[:] = [1.0] * 4
    bad_fmt = PixelFormat(); bad_fmt.dtype = 9
    nan_fmt = PixelFormat(); nan_fmt.dtype = 1; nan_fmt.scale[:] = [float("nan")] * 4
    o = out.data_ptr()

    def args(**kw):
        a = dict(base=data.data_ptr(), bb=data.numel(), n=3, mfs=1 << 20, mw=1 << 12, mh=1 << 12, cap=1 << 24, boxes=None, ow=8, oh=8,
                 d=4, flags=1, fmt=C.byref(fmt), out=o, strides=(8 * 8 * 16, 8 * 16, 16, 4))
        a.update(kw)
        return (a["base"], a["bb"], offsets.data_ptr(), sizes.data_ptr(), a["n"], a["mfs"], a["mw"], a["mh"], a["cap"], a["boxes"],
                a["ow"], a["oh"], a["d"], a["flags"], a["fmt"], a["out"], *a["strides"], info.data_ptr(), st.data_ptr(), None)

    cases = [(dict(n=0), 1), (dict(n=65536), 1), (dict(ow=0), 1), (dict(oh=0), 1), (dict(ow=(1 << 24) + 1), 1), (dict(oh=(1 << 24) + 1), 1),
             (dict(d=2), 1), (dict(d=5), 1), (dict(flags=2), 1), (dict(flags=8), 1), (dict(flags=6), 1), (dict(fmt=C.byref(bad_fmt)), 1), (dict(fmt=C.byref(nan_fmt)), 1),
             (dict(out=None), 1), (dict(base=None), 1), (dict(mfs=0), 1), (dict(mw=0), 1), (dict(mh=(1 << 24) + 1), 1),
             (dict(strides=(8 * 8 * 16, 8 * 16, 8, 4)), 1), (dict(strides=(8 * 16, 8 * 16, 16, 4)), 1),
             (dict(base=data.data_ptr() + 2), 5), (dict(out=o + 2), 5), (dict(strides=(8 * 8 * 16, 8 * 16 + 2, 16, 4)), 5)]
    before = gpu.launch_count()
    for kw, rc in cases:
        assert lib().fpngb_decode_packed_resized_device(*args(**kw)) == rc, kw
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out.cpu().numpy() == -5).all() and (st.cpu().numpy() == -7).all() and (info.cpu().numpy() == -7).all()
    # the same arguments are accepted as they are
    assert lib().fpngb_decode_packed_resized_device(*args()) == 0
    torch.cuda.synchronize()
    assert (st.cpu().numpy() == 0).all() and gpu.launch_count() - before == 12
    # with FPNGB_RESIZE_ANY_PNG: the same call, three launches more
    for k, flags in enumerate((5, 4)):
        assert lib().fpngb_decode_packed_resized_device(*args(flags=flags)) == 0
        torch.cuda.synchronize()
        assert (st.cpu().numpy() == 0).all() and gpu.launch_count() - before == 12 + 15 * (k + 1)
