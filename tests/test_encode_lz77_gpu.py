"""GPU tests of the LZ77 mode of the PNG encode (encode_png_device / encode_labels_device with lz77=K, FPNGB_LZ77_CHAIN): every
file must equal the oracle's (tests/cpp/lz77_oracle.c) byte for byte, decode back on the GPU, and leave the bytes after the
call's slots untouched."""
import numpy as np
import pytest

import lz77_oracle as lo

pytestmark = pytest.mark.gpu

INVALID_ARG = 1
GUARD = 0xA5


@pytest.fixture(scope="module")
def fp():
    import fpng_b200
    fpng_b200.fpng_init(0)
    return fpng_b200


def dev(img):
    import torch
    return torch.from_numpy(np.ascontiguousarray(img)).cuda()


def files(out, offsets, sizes):
    import torch
    torch.cuda.synchronize()
    data, ofs, sz = out.cpu().numpy(), offsets.cpu().numpy(), sizes.cpu().numpy().astype(np.int64)
    return [data[ofs[i]:ofs[i] + sz[i]].tobytes() for i in range(len(sz))]


def guarded_out(fp, shapes, bound=None):
    import torch
    total = int((bound or fp.png_slot_offsets)(shapes)[-1])
    buf = torch.full((total + 64,), GUARD, dtype=torch.uint8, device="cuda")
    return buf, total


def structured(rs, h, w, c, dtype=np.uint8):
    """blocks of repeated content, a few noisy rows, and rows that repeat far above: matches at every distance"""
    top = 255 if dtype == np.uint8 else 65535
    tile = rs.integers(0, top + 1, (8, 8, c), dtype=np.int64)
    img = np.tile(tile, (h // 8 + 1, w // 8 + 1, 1))[:h, :w]
    img[h // 3:h // 3 + 2] = rs.integers(0, top + 1, (min(2, h - h // 3), w, c))
    img[(2 * h) // 3:] = img[:h - (2 * h) // 3]
    return img.astype(dtype)


CLASSES = [(1, np.uint8), (2, np.uint8), (3, np.uint8), (4, np.uint8), (1, np.uint16), (2, np.uint16), (3, np.uint16), (4, np.uint16)]


def check(fp, imgs, K, flags=0, views=None):
    shapes = [(i.shape[0], i.shape[1], i.shape[2], 8 * i.dtype.itemsize) for i in imgs]
    buf, total = guarded_out(fp, shapes)
    out, offsets, sizes = fp.encode_png_device(views if views is not None else [dev(i) for i in imgs], flags, out=buf[:total], lz77=K)
    got = files(out, offsets, sizes)
    assert offsets.cpu().numpy().tolist() == fp.png_slot_offsets(shapes).tolist()
    for k, img in enumerate(imgs):
        assert got[k] == lo.png_encode(img, K, flags), (k, img.shape, img.dtype, K, flags)
    assert (buf[total:].cpu().numpy() == GUARD).all()
    return out, offsets, sizes


@pytest.mark.parametrize("K", [1, 8, 128])
def test_every_class_matches_oracle(fp, K):
    rs = np.random.default_rng(K)
    imgs = [structured(rs, h, w, c, dt) for (c, dt) in CLASSES for (h, w) in ((1, 1), (3, 5), (37, 61), (130, 257))]
    check(fp, imgs, K)


def test_forced_stored_and_noise(fp):
    rs = np.random.default_rng(1)
    imgs = [structured(rs, 40, 50, c, dt) for (c, dt) in CLASSES] + [rs.integers(0, 256, (64, 64, 3), dtype=np.uint8)]
    check(fp, imgs, 8, 2)
    check(fp, imgs, 8, 0)


def test_segments_and_window(fp):
    """streams of 16383, 16384, 16385 and 3 * 16384 + 1 bytes, a multi-segment image with 32 KiB distances, an all-equal image"""
    rs = np.random.default_rng(2)
    imgs = []
    for n in (16383, 16384, 16385, 3 * 16384 + 1):          # one row of n - 1 gray8 pixels
        row = np.tile(rs.integers(0, 256, 300, dtype=np.uint8), n // 300 + 1)[:n - 1]
        imgs.append(row.reshape(1, n - 1, 1))
    far = rs.integers(0, 256, (1, 32767, 1), dtype=np.uint8)
    imgs.append(np.concatenate([far, far, far], axis=0))      # rows 32768 bytes apart (filter byte included)
    imgs.append(np.full((300, 700, 4), 7, np.uint8))
    imgs.append(structured(rs, 300, 300, 2, np.uint8))
    for K in (1, 2, 256):
        check(fp, imgs, K)


def test_views_and_round_trip(fp):
    """crops and CHW views match the oracle on their pixels, and every file decodes back through the all-formats decoder (the
    uint8 output holds each sample's high byte; gray is replicated to RGB, alpha the file lacks is not compared)"""
    import torch
    rs = np.random.default_rng(3)
    t = dev(structured(rs, 90, 140, 4, np.uint8))
    t16 = dev(structured(rs, 50, 60, 3, np.uint16))
    views = [t[5:80, 7:120], t.permute(2, 0, 1).contiguous().permute(1, 2, 0), t16[3:40, 1:59],
             t16.permute(2, 0, 1).contiguous().permute(1, 2, 0)]
    imgs = [v.cpu().numpy() for v in views] + [structured(rs, 70, 33, c, np.uint8) for c in (1, 2)]
    views = views + [dev(i) for i in imgs[4:]]
    out, offsets, sizes = check(fp, imgs, 32, views=views)
    px, pofs, _, status = fp.decode_packed_ragged_device(out, offsets[:-1].contiguous(), sizes, 4, any_png=True, all_formats=True)
    torch.cuda.synchronize()
    assert not status.any().item()
    px, pofs = px.cpu().numpy(), pofs.cpu().numpy()
    for k, img in enumerate(imgs):
        h, w, c = img.shape
        cols = [[0, 0, 0], [0, 0, 0, 1], [0, 1, 2], [0, 1, 2, 3]][c - 1]
        u8 = px.view(np.uint8)[pofs[k]:pofs[k] + 4 * h * w].reshape(h, w, 4)[..., :len(cols)]
        hi = (img >> 8).astype(np.uint8) if img.dtype == np.uint16 else img
        assert np.array_equal(u8, hi[..., cols]), (k, img.shape, img.dtype)


def test_labels_match_oracle(fp):
    import torch
    rs = np.random.default_rng(4)
    cases = []
    for depth, pal in ((1, None), (2, None), (4, None), (16, None), (2, rs.integers(0, 256, (3, 4), dtype=np.uint8)),
                       (8, rs.integers(0, 256, (200, 3), dtype=np.uint8))):
        limit = (1 << depth) if pal is None else len(pal)
        ids = np.tile(rs.integers(0, limit, (9, 13)), (20, 30))[:170, :333]
        cases.append((ids, depth, pal))
    for K in (1, 16):
        imgs = [dev(ids.astype(np.int64 if d == 16 or k % 2 else np.uint8)) for k, (ids, d, _) in enumerate(cases)]
        out, offsets, sizes = fp.encode_labels_device(imgs, palette=[p for _, _, p in cases], depth=[d for _, d, _ in cases], lz77=K)
        got = files(out, offsets, sizes)
        for k, (ids, d, pal) in enumerate(cases):
            assert got[k] == lo.label_encode(ids, d, K, pal), (k, d, K)


def test_reduce_and_typed(fp):
    import torch
    rs = np.random.default_rng(5)
    mask = (structured(rs, 60, 70, 1, np.uint8) > 128).astype(np.uint8) * 255
    rgb = np.repeat(mask, 3, axis=2)
    opaque = np.concatenate([rs.integers(0, 256, (60, 70, 3), dtype=np.uint8), np.full((60, 70, 1), 255, np.uint8)], axis=2)
    out, offsets, sizes = fp.encode_png_device([dev(rgb), dev(opaque)], reduce=True, lz77=8)
    got = files(out, offsets, sizes)
    assert got[0] == lo.label_encode((mask[:, :, 0] // 255).astype(np.int64), 1, 8)
    assert got[1] == lo.png_encode(opaque[:, :, :3], 8)
    f = structured(rs, 50, 40, 3, np.uint8)
    for depth, dt in ((8, np.uint8), (16, np.uint16)):
        out, offsets, sizes = fp.encode_png_device([dev(f.astype(np.float32))], depth=depth, lz77=8)
        assert files(out, offsets, sizes)[0] == lo.png_encode(f.astype(dt), 8)


def test_many_images_two_streams(fp):
    import torch
    rs = np.random.default_rng(6)
    imgs = [structured(rs, int(rs.integers(1, 20)), int(rs.integers(1, 40)), 1 + k % 4, np.uint8) for k in range(4096)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    res = []
    for part, s in ((imgs[:2048], s1), (imgs[2048:], s2)):
        with torch.cuda.stream(s):
            res.append(fp.encode_png_device([dev(i) for i in part], lz77=4))
    torch.cuda.synchronize()
    for part, r in zip((imgs[:2048], imgs[2048:]), res):
        got = files(*r)
        for k in range(0, len(part), 97):
            assert got[k] == lo.png_encode(part[k], 4)


def test_compressed_equals_stored_tie(fp):
    """an image whose compressed stream is exactly as long as the stored one stays compressed (zcomp <= zstored)"""
    from test_encode_lz77_cpu import tie_row
    check(fp, [tie_row().reshape(1, -1, 1)], 8)


def test_label_indices_round_trip(fp):
    import torch
    rs = np.random.default_rng(9)
    cases = [(np.tile(rs.integers(0, 1 << d, (7, 11)), (9, 21))[:60, :200], d) for d in (1, 2, 4, 8, 16)]
    imgs = [dev(ids.astype(np.int64)) for ids, _ in cases]
    out, offsets, sizes = fp.encode_labels_device(imgs, depth=[d for _, d in cases], lz77=8)
    got = files(out, offsets, sizes)
    for k, (ids, d) in enumerate(cases):
        assert got[k] == lo.label_encode(ids, d, 8), (k, d)
    px, pofs, info, st = fp.decode_packed_ragged_device(out, offsets[:-1].contiguous(), sizes, 1, indices=True, any_png=True,
                                                        all_formats=True, native=True, dtype=torch.uint16)
    views = fp.ragged_views(px, pofs, info, st, 1)
    for k, (ids, d) in enumerate(cases):
        assert np.array_equal(views[k].cpu().numpy()[..., 0].astype(np.int64), ids), (k, d)


def big_image():
    """16-bit RGBA, 8192 x 18432: smooth high bytes, random low bytes.  Its stream S is 1.21 GB and codes to about 0.8 GB, so the
    compressed stream passes 2^29 bytes and the segments' bit offsets pass 2^32"""
    h, w = 18432, 8192
    rs = np.random.default_rng(29)
    img = np.empty((h, w, 4), np.uint16)
    hi = ((np.arange(w)[None, :] // 64 + np.arange(h)[:, None] // 64) & 0xFF).astype(np.uint16) << 8
    for c in range(4):
        img[:, :, c] = hi | rs.integers(0, 256, (h, w), dtype=np.uint16)
    return img


def test_stream_past_2_pow_29(fp):
    import torch
    img = big_image()
    want, d = lo.png_encode(img, 1, want_info=True)
    assert d["stored"] == 0 and d["zcomp"] > 1 << 29
    shapes = [(img.shape[0], img.shape[1], 4, 16)]
    buf, total = guarded_out(fp, shapes)
    out, offsets, sizes = fp.encode_png_device([dev(img)], out=buf[:total], lz77=1)
    torch.cuda.synchronize()
    n = int(sizes[0])
    got = buf[:n].cpu().numpy()
    w = np.frombuffer(want, np.uint8)
    same = n == len(want) and np.array_equal(got, w)
    assert same, (n, len(want), int(np.argmax(got[:min(n, len(w))] != w[:min(n, len(w))])))
    assert (buf[total:].cpu().numpy() == GUARD).all()


def test_rejections(fp):
    import ctypes as C
    from fpng_b200._lib import lib
    t = dev(np.zeros((4, 4, 1), np.uint8))
    with pytest.raises(Exception):
        fp.encode_png_device([t], 1, lz77=8)                  # FPNG_ENCODE_SLOWER with a chain depth
    with pytest.raises(ValueError):
        fp.encode_png_device([t], lz77=257)
    out = dev(np.zeros(4096, np.uint8))
    offsets = dev(np.zeros(2, np.int64))
    sizes = dev(np.zeros(1, np.int32))
    ptrs = np.array([t.data_ptr()], np.uint64)
    dims = np.array([4, 4, 1, 8], np.uint32)
    for flags in (257 << 16, 511 << 16, (8 << 16) | 1, 1 << 25):
        rc = lib().fpngb_encode_png_ragged_device(1, ptrs.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p), None, flags,
                                                  out.data_ptr(), 4096, offsets.data_ptr(), sizes.data_ptr(), None)
        assert rc == INVALID_ARG, flags
