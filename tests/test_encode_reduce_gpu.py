"""encode_png_device(reduce=True) (FPNGB_ENCODE_REDUCE) on the GPU: every reduced file is byte-identical to the existing call's file
on the model-reduced input (tests/reduce_model.py), the files decode back to the input pixels (our decoder and PIL), and the
analysis holds at its colour-count, hash, CTA, size, layout, stream and launch edges."""
from __future__ import annotations

import ctypes as C
import io

import numpy as np
import pytest

from reduce_model import choose, hash_slot, reduced_call

pytestmark = pytest.mark.gpu

GUARD = 0xA5
SLOWER, FORCE = 1, 2


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda().view(
        torch.uint16 if a.dtype == np.uint16 else torch.uint8)


def files_of(out, offsets, sizes):
    import torch
    torch.cuda.synchronize()
    o, s, raw = offsets.cpu().numpy(), sizes.cpu().numpy(), out.cpu().numpy()
    return [raw[o[i]:o[i] + s[i]].tobytes() for i in range(len(s))]


def reduce_encode(gpu, images, flags=0, guard=64, stream=None):
    """one reduce call into a guard-filled buffer; returns (files, guard bytes past the total, sizes)"""
    import torch
    shapes = [(t.shape[0], t.shape[1], t.shape[2], 8 * t.element_size()) for t in images]
    total = int(gpu.reduced_slot_offsets(shapes)[-1])
    raw = torch.full((total + guard,), GUARD, dtype=torch.uint8, device="cuda")
    out, offsets, sizes = gpu.encode_png_device(images, flags=flags, out=raw[:total], reduce=True, stream=stream)
    files = files_of(out, offsets, sizes)
    assert int(offsets[-1]) == total
    return files, raw[total:].cpu().numpy(), sizes.cpu().numpy()


def expected_file(gpu, img, flags):
    """the existing call's file on the model-reduced input"""
    call = reduced_call(img)
    if call[0] == "labels":
        _, ids, pal, depth = call
        out, offsets, sizes = gpu.encode_labels_device([dev(ids)], palette=pal, depth=depth, flags=flags & FORCE)
    else:
        out, offsets, sizes = gpu.encode_png_device([dev(call[1])], flags=flags)
    return files_of(out, offsets, sizes)[0]


def corpus():
    """seeded images reaching every format of the rule, from every input channel count and depth"""
    rng = np.random.default_rng(7)
    im = []
    h, w = 23, 37
    im.append(np.zeros((h, w, 1), np.uint8))                                          # gray 1-bit (constant 0)
    im.append(np.full((h, w, 1), 100, np.uint8))                                      # palette 1-bit
    im.append(rng.integers(0, 2, (h, w, 3), dtype=np.uint8).repeat(1, 2)[..., :1].repeat(3, 2) * 255)   # RGB binary mask: gray 1
    im.append((rng.integers(0, 4, (h, w, 1)) * 85).astype(np.uint8))                  # gray 2-bit
    im.append((rng.integers(0, 16, (h, w, 1)) * 17).astype(np.uint8).repeat(3, 2))    # gray 4-bit from RGB
    im.append(rng.integers(0, 256, (h, w, 1), dtype=np.uint8).repeat(3, 2))           # grey scan as RGB: gray8
    cols = rng.integers(0, 256, (19, 3), dtype=np.uint8)
    im.append(cols[rng.integers(0, 19, (h, w))])                                      # 19-colour segmentation: palette 8
    cols4 = rng.integers(0, 256, (5, 4), dtype=np.uint8)
    im.append(cols4[rng.integers(0, 5, (h, w))])                                      # RGBA palette 4-bit with tRNS
    im.append(cols[:3][rng.integers(0, 3, (h, w))])                                   # palette 2-bit
    ga = np.stack([rng.integers(0, 256, (h, w)), rng.integers(0, 256, (h, w))], 2).astype(np.uint8)
    im.append(ga)                                                                     # GA8
    rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    rgba[..., 3] = 255
    im.append(rgba)                                                                   # opaque RGBA: fpng RGB
    im.append(rng.integers(0, 256, (h, w, 4), dtype=np.uint8))                        # RGBA stays (fpng)
    im.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))                        # RGB stays (fpng)
    g4 = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    g4[..., 1] = g4[..., 0]; g4[..., 2] = g4[..., 0]
    im.append(g4)                                                                     # gray-valued RGBA: GA8
    im.append(rng.integers(0, 65536, (h, w, 1), dtype=np.uint16))                     # gray16 stays
    im.append(rng.integers(0, 65536, (h, w, 3), dtype=np.uint16).astype(np.uint16))  # RGB16 stays
    r16 = rng.integers(0, 65536, (h, w, 4), dtype=np.uint16)
    r16[..., 3] = 65535
    im.append(r16)                                                                    # RGBA16 opaque: RGB16
    g16 = rng.integers(0, 65536, (h, w, 3), dtype=np.uint16)
    g16[..., 1] = g16[..., 0]; g16[..., 2] = g16[..., 0]
    im.append(g16)                                                                    # gray-valued RGB16: gray16
    ga16 = rng.integers(0, 65536, (h, w, 4), dtype=np.uint16)
    ga16[..., 1] = ga16[..., 0]; ga16[..., 2] = ga16[..., 0]
    im.append(ga16)                                                                   # GA16
    im.append((rng.integers(0, 256, (h, w, 4)) * 257).astype(np.uint16))              # 16-bit, multiples of 257: RGBA8 fpng
    im.append((rng.integers(0, 256, (h, w, 2)) * 257).astype(np.uint16))              # GA16 of multiples of 257: GA8
    im.append((cols[rng.integers(0, 19, (h, w))].astype(np.uint16) * 257))            # 16-bit palette
    im.append((rng.integers(0, 4, (h, w, 1)) * 85 * 257).astype(np.uint16))           # 16-bit gray 2-bit
    im.append(rng.integers(0, 65536, (h, w, 4), dtype=np.uint16))                     # RGBA16 stays
    return im


CORPUS = corpus()


def test_corpus_reaches_every_format():
    got = {(f, d) for f, _, d in map(choose, CORPUS)}
    want = {("gray", 1), ("gray", 2), ("gray", 4), ("gray", 8), ("gray", 16), ("palette", 1), ("palette", 2), ("palette", 4),
            ("palette", 8), ("ga", 8), ("ga", 16), ("rgb", 8), ("rgb", 16), ("rgba", 8), ("rgba", 16)}
    assert want <= got, want - got


@pytest.mark.parametrize("flags", [0, SLOWER, FORCE])
def test_byte_identity_mixed_and_single(gpu, flags):
    want = [expected_file(gpu, a, flags) for a in CORPUS]
    files, tail, _ = reduce_encode(gpu, [dev(a) for a in CORPUS], flags)
    assert (tail == GUARD).all()
    for i, (f, w) in enumerate(zip(files, want)):
        assert f == w, (i, choose(CORPUS[i]))
    for i, a in enumerate(CORPUS):
        files, tail, _ = reduce_encode(gpu, [dev(a)], flags)
        assert files[0] == want[i] and (tail == GUARD).all(), i


def decode_native(gpu, files, chans, dtype=None):
    import torch
    sizes = [len(f) for f in files]
    ofs = np.zeros(len(files) + 1, np.int64)
    ofs[1:] = np.cumsum([(s + 15) // 16 * 16 for s in sizes])
    buf = np.zeros(int(ofs[-1]), np.uint8)
    for f, o in zip(files, ofs):
        buf[o:o + len(f)] = np.frombuffer(f, np.uint8)
    data, offsets = torch.from_numpy(buf).cuda(), torch.from_numpy(ofs).cuda()
    sz = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    out, oo, info, status = gpu.decode_packed_ragged_device(data, offsets, sz, chans, any_png=True, all_formats=True, native=True,
                                                            dtype=dtype)
    torch.cuda.synchronize()
    assert (status.cpu().numpy() == 0).all()
    return out, oo.cpu().numpy(), info.cpu().numpy()


def test_round_trip_decoder_and_pil(gpu):
    import torch
    from PIL import Image
    files, _, _ = reduce_encode(gpu, [dev(a) for a in CORPUS])
    for a, f in zip(CORPUS, files):
        c = a.shape[2]
        if a.dtype == np.uint8:
            out, oo, info = decode_native(gpu, [f], c)
            px = out.cpu().numpy()[oo[0]:oo[0] + a.size].reshape(a.shape)
            assert (px == a).all(), choose(a)
            mode = {1: "L", 2: "LA", 3: "RGB", 4: "RGBA"}[c]
            assert (np.asarray(Image.open(io.BytesIO(f)).convert(mode)).reshape(a.shape) == a).all(), choose(a)
        else:
            out, oo, info = decode_native(gpu, [f], c, torch.uint16)
            px = out.view(torch.uint8).cpu().numpy()[oo[0]:oo[0] + 2 * a.size].view(np.uint16).reshape(a.shape)
            assert (px == a).all(), choose(a)
        assert info[0, 0] == 0 and (info[0, 1], info[0, 2]) == (a.shape[1], a.shape[0])


def test_cv2_reads_16bit(gpu):
    cv2 = pytest.importorskip("cv2")
    sixteen = [a for a in CORPUS if a.dtype == np.uint16 and choose(a)[2] == 16]
    files, _, _ = reduce_encode(gpu, [dev(a) for a in sixteen])
    for a, f in zip(sixteen, files):
        got = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_UNCHANGED)
        got = got.reshape(a.shape[0], a.shape[1], -1)
        if got.shape[2] >= 3:                                                          # BGR(A) -> RGB(A)
            got = got[..., [2, 1, 0] + ([3] if got.shape[2] == 4 else [])]
        c_out = got.shape[2]
        ref = a[..., :c_out] if c_out != 2 else a[..., [0, a.shape[2] - 1]]
        assert got.dtype == np.uint16 and (got == ref).all()


# ---- edges ------------------------------------------------------------------------------------------------------------------------
def check(gpu, imgs, flags=0):
    files, tail, _ = reduce_encode(gpu, [dev(a) for a in imgs], flags)
    assert (tail == GUARD).all()
    for a, f in zip(imgs, files):
        assert f == expected_file(gpu, a, flags), choose(a)
    return files


def distinct_colours(k, seed=0):
    rng = np.random.default_rng(seed)
    keys = rng.choice(1 << 24, k, replace=False).astype(np.uint32)
    return np.stack([keys >> 16, (keys >> 8) & 255, keys & 255], 1).astype(np.uint8)


def test_256_and_257_colours_last_pixel(gpu):
    cols = distinct_colours(257, 1)
    a = np.repeat(cols[:256], 200, axis=0).reshape(400, 128, 3)                        # 51200 pixels, several CTAs
    b = a.copy()
    b[-1, -1] = cols[256]                                                              # the 257th colour at the last pixel only
    assert choose(a)[0] == "palette" and choose(b)[0] == "rgb"
    check(gpu, [a, b])


def test_ctas_below_256_image_above(gpu):
    cols = distinct_colours(600, 2)
    a = np.concatenate([np.repeat(cols[200 * k:200 * k + 200], 41, axis=0)[:8192] for k in range(3)]).reshape(96, 256, 3)
    assert choose(a)[0] == "rgb"                                                       # each 8192-pixel CTA sees 200 colours
    check(gpu, [a])


def test_zero_ff_and_hash_collisions(gpu):
    ks = np.arange(0x11223344, 0x11223344 + 100000, dtype=np.uint64)
    slots = ((ks * 0x9E3779B1) & 0xFFFFFFFF) >> 23
    same = ks[slots == slots[0]][:10]                                                  # colours that share a slot
    assert len(same) == 10 and len({hash_slot(int(k)) for k in same}) == 1
    keys = np.array([0x00000000, 0xFFFFFFFF] + [int(k) for k in same], np.uint32)
    cols = np.stack([keys >> 24, (keys >> 16) & 255, (keys >> 8) & 255, keys & 255], 1).astype(np.uint8)
    a = cols[np.random.default_rng(3).integers(0, len(cols), (33, 47))]
    assert choose(a) == ("palette", 4, 4)
    check(gpu, [a])
    check(gpu, [np.zeros((5, 9, 4), np.uint8), np.full((5, 9, 4), 255, np.uint8)])


def test_transparent_pixels_keep_their_rgb(gpu):
    a = np.zeros((8, 8, 4), np.uint8)
    a[..., 0] = np.arange(64).reshape(8, 8)                                            # 64 colours, all alpha 0
    assert choose(a) == ("palette", 8, 8)
    files = check(gpu, [a])
    out, oo, _ = decode_native(gpu, files, 4)
    assert (out.cpu().numpy()[:a.size].reshape(a.shape) == a).all()


def test_extreme_shapes(gpu):
    rng = np.random.default_rng(4)
    check(gpu, [rng.integers(0, 256, (1, 1, c), dtype=np.uint8) for c in (1, 2, 3, 4)])
    wide = np.zeros((1, 1 << 24, 1), np.uint8)
    wide[0, ::3] = 255
    tall = (rng.integers(0, 3, (1 << 24, 1, 3)) * 100).astype(np.uint8)
    check(gpu, [wide, tall])


def test_16k_palette_image(gpu):
    import torch
    n = 16384
    lut = torch.tensor(distinct_colours(200, 5), device="cuda")
    idx = (torch.arange(n, device="cuda").view(-1, 1) * 7 + torch.arange(n, device="cuda").view(1, -1) * 3) % 200
    img = lut[idx]                                                                     # 768 MiB RGB, 200 colours
    del idx
    files, tail, sizes = reduce_encode(gpu, [img], FORCE)
    assert (tail == GUARD).all()
    f = files[0]
    assert f[24:26] == bytes([8, 3])                                                   # palette, depth 8
    out, oo, info = decode_native(gpu, [f], 3)
    assert torch.equal(out[:img.numel()].view(n, n, 3), img)


def test_layouts_strided_chw_expand(gpu):
    import torch
    rng = np.random.default_rng(6)
    cols = torch.tensor(distinct_colours(9, 6), device="cuda")
    full = cols[torch.tensor(rng.integers(0, 9, (40, 60)), device="cuda")]
    crop = full[3:30, 5:50]                                                            # strided rows
    chw = full.permute(2, 0, 1).contiguous().permute(1, 2, 0)                          # planar
    exp = full[:1].expand(25, -1, -1)                                                  # stride-0 rows
    rgba = torch.cat([full, torch.full_like(full[..., :1], 255)], 2)[..., :3]         # an RGB view of RGBA pixels
    imgs = [crop, chw, exp]
    files, tail, _ = reduce_encode(gpu, imgs)
    for t, f in zip(imgs, files):
        assert f == expected_file(gpu, t.cpu().numpy(), 0)
    with pytest.raises(Exception):
        gpu.encode_png_device([rgba], reduce=True)


def test_thousands_mixed(gpu):
    rng = np.random.default_rng(8)
    imgs = []
    for i in range(3000):
        a = CORPUS[i % len(CORPUS)]
        y, x = rng.integers(0, 10), rng.integers(0, 10)
        imgs.append(a[y:y + 1 + rng.integers(0, 13), x:x + 1 + rng.integers(0, 27)])
    files, tail, _ = reduce_encode(gpu, [dev(a) for a in imgs], 0)
    assert (tail == GUARD).all()
    for i in range(0, 3000, 7):
        assert files[i] == expected_file(gpu, imgs[i], 0), i


def test_canaries_past_slots(gpu):
    import torch
    imgs = [dev(a) for a in CORPUS[:8]]
    shapes = [(t.shape[0], t.shape[1], t.shape[2], 8 * t.element_size()) for t in imgs]
    ofs = gpu.reduced_slot_offsets(shapes)
    raw = torch.full((int(ofs[-1]) + 256,), GUARD, dtype=torch.uint8, device="cuda")
    out, offsets, sizes = gpu.encode_png_device(imgs, out=raw[:int(ofs[-1])], reduce=True)
    torch.cuda.synchronize()
    r, s = raw.cpu().numpy(), sizes.cpu().numpy()
    for i in range(len(imgs)):
        assert (r[ofs[i] + s[i]:ofs[i + 1]] == GUARD).all(), i
    assert (r[int(ofs[-1]):] == GUARD).all()


def test_side_stream_after_writer(gpu):
    import torch
    a = CORPUS[6]
    want = expected_file(gpu, a, 0)
    src = dev(a)
    side = torch.cuda.Stream()
    t = torch.zeros_like(src)
    with torch.cuda.stream(side):
        torch.cuda._sleep(2_000_000)
        t.copy_(src)                                                                   # a kernel that writes the input
        files, tail, _ = reduce_encode(gpu, [t], 0, stream=side.cuda_stream)
    assert files[0] == want


def test_launches_and_profile_slots(gpu):
    import torch
    L = gpu.api.lib()
    L.fpngb_profile_enable.argtypes = [C.c_int]
    L.fpngb_profile_read.argtypes = [C.POINTER(C.c_float), C.c_int]
    ms = (C.c_float * 11)()
    img_pal, img_rgb = dev(CORPUS[6]), dev(CORPUS[12])
    gpu.encode_png_device([img_pal], reduce=True)
    torch.cuda.synchronize()
    n0 = gpu.launch_count()
    gpu.encode_png_device([img_rgb], reduce=True)                                      # RGB stays: analysis 2 + fpng route
    n1 = gpu.launch_count()
    gpu.encode_png_device([img_rgb])
    n2 = gpu.launch_count()
    assert n1 - n0 == 2 + (n2 - n1)
    gpu.encode_png_device([img_pal], reduce=True)                                      # palette: analysis 2 + conversion 1 + PNG
    n3 = gpu.launch_count()
    assert n3 - n2 == 2 + 1 + 3 + 4
    L.fpngb_profile_read(ms, 11)
    L.fpngb_profile_enable(1)
    try:
        gpu.encode_png_device([img_pal], reduce=True)
        torch.cuda.synchronize()
        assert L.fpngb_profile_read(ms, 11) == 1 and ms[10] > 0 and ms[9] > 0
        gpu.encode_png_device([img_rgb], reduce=True)
        torch.cuda.synchronize()
        assert L.fpngb_profile_read(ms, 11) == 1 and ms[10] > 0 and ms[9] == 0
    finally:
        L.fpngb_profile_enable(0)


def test_rejections(gpu):
    import torch
    from fpng_b200._lib import FpngB200Error
    L = gpu.api.lib()
    img = dev(CORPUS[0])
    n = 1
    ptrs = np.array([img.data_ptr()], np.uint64)
    dims = np.array([[img.shape[1], img.shape[0], 1, 8]], np.uint32)
    out = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    offsets = torch.zeros(2, dtype=torch.int64, device="cuda")
    sizes = torch.zeros(1, dtype=torch.int32, device="cuda")
    fmt = gpu.api.PixelFormat()
    rc = L.fpngb_encode_png_ragged_device_typed(n, ptrs.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p), None,
                                                C.byref(fmt), gpu.FPNGB_ENCODE_REDUCE, out.data_ptr(), out.numel(), offsets.data_ptr(), sizes.data_ptr(),
                                                None)
    assert rc == 1
    small = int(gpu.reduced_slot_offsets([(img.shape[0], img.shape[1], 1, 8)])[-1]) - 16
    with pytest.raises(FpngB200Error):
        gpu.encode_png_device([img], out=out[:small], reduce=True)
    huge = torch.zeros(1, 256, 4, dtype=torch.uint8, device="cuda").expand(1 << 24, -1, -1)  # bound above 2^31 - 1
    with pytest.raises(FpngB200Error):
        gpu.encode_png_device([huge], out=out, reduce=True)
