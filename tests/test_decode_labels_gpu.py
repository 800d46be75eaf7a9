"""GPU tests of the label-map decode: raw-sample output in the any-PNG ragged and resized decodes (FPNGB_PNG_INDEX,
FPNGB_RESIZE_INDEX, indices=True) and the nearest-neighbour resized decode (FPNGB_RESIZE_NEAREST / _EXACT, interpolation=).
Expected values come from the numpy models of test_decode_labels_cpu.py (pinned there against PIL and torch's CPU
F.interpolate), applied to the samples the test wrote or to the ragged decode's output; torch's CUDA F.interpolate is a second
check where it has the dtype."""
import ctypes as C

import numpy as np
import pytest

import pngwrite_formats as pf
from test_decode_labels_cpu import golden_label_files, index_model, nearest_src
from test_decode_native_gpu import as_np, packed
from test_decode_png_gpu import fpng_file

pytestmark = pytest.mark.gpu

GUARD = 0xA5
NOT_INDEXED, BAD_CROP, SHAPE_MISMATCH, CRC = 105, 103, 100, 4
SHAPES = [(1, 1), (2, 3), (5, 4), (9, 7), (17, 1), (13, 17), (33, 5), (70, 9)]
FULL = dict(any_png=True, all_formats=True, native=True)


def ragged_index(gpu, files, dtype, max_w=None, max_h=None, seed=0):
    """one indices=True ragged call with every bound given into a guard-filled buffer; returns (views, status, out_offsets, raw)"""
    import torch
    T = getattr(torch, dtype)
    data, offsets, sizes = packed(files, seed)
    infos = [gpu.get_png_info(f, all_formats=True) for f in files]
    es = T.itemsize
    cap = max(16, sum((i[1] * i[2] * es + 15) // 16 * 16 for i in infos if i[0] == 0))
    raw = torch.full((cap + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out = raw[:cap].view(T) if es > 1 else raw[:cap]
    _, oo, info, st = gpu.decode_packed_ragged_device(
        data, offsets, sizes, 1, out=out, max_file_size=max(len(f) for f in files), indices=True,
        max_w=max_w or max([i[1] for i in infos] + [1]), max_h=max_h or max([i[2] for i in infos] + [1]), **FULL)
    torch.cuda.synchronize()
    return gpu.ragged_views(out, oo, info, st, 1), st.cpu().numpy(), oo.cpu().numpy(), raw.cpu().numpy()


def check_untouched(raw, oo, st):
    """every byte outside the files the call decoded keeps the guard"""
    mask = np.ones(raw.size, bool)
    for i in np.nonzero(st == 0)[0]:
        mask[oo[i]:oo[i + 1]] = False
    assert (raw[mask] == GUARD).all()


# ---- 1. index decode ----------------------------------------------------------------------------------------------------------------
LABEL_COMBOS = [c for c in pf.combos() if c[0] in (0, 3)]


@pytest.mark.parametrize("combo", LABEL_COMBOS, ids=lambda c: "t%d_d%d_i%d_%s" % (c[0], c[1], c[2], "trns" if c[3] else "plain"))
def test_index_every_label_format(gpu, combo):
    ctype, depth, il, t = combo
    rs = np.random.RandomState(300 + 100 * ctype + depth + 7 * il + 3 * t)
    cases = [pf.case(rs, w, h, ctype, depth, il, t, seed=k) for k, (w, h) in enumerate(SHAPES)]
    cases += [pf.case(rs, 19, 11, ctype, depth, il, t, filters=ft, seed=50 + ft) for ft in range(5)]
    files = [c[0] for c in cases]
    for dtype in ("uint8", "uint16"):
        views, st, oo, raw = ragged_index(gpu, files, dtype)
        if depth == 16 and dtype == "uint8":                                    # not truncated: no space, nothing written
            assert (st == NOT_INDEXED).all() and (oo == 0).all() and (raw == GUARD).all()
            continue
        assert (st == 0).all(), st
        for k, (png, s, plte, trns) in enumerate(cases):
            assert np.array_equal(as_np(views[k]).astype(np.int64), s[..., :1].astype(np.int64)), (dtype, k, s.shape)
        check_untouched(raw, oo, st)


def test_index_golden_files(gpu):
    files = [open(p, "rb").read() for p in golden_label_files()]
    for dtype in ("uint8", "uint16"):
        views, st, _, _ = ragged_index(gpu, files, dtype)
        assert (st == 0).all()
        for k, f in enumerate(files):
            assert np.array_equal(as_np(views[k])[..., 0].astype(np.int64), index_model(f)), (dtype, k)


def not_indexed_files(gpu, rs):
    out = [pf.case(rs, 9, 5, ctype, depth, il, t)[0] for ctype in (2, 4, 6) for depth in (8, 16) for il in (0, 1)
           for t in ((False, True) if ctype == 2 else (False,))]
    out += [fpng_file(gpu, 12, 7, c, k)[0] for k, c in enumerate((3, 4))]
    return out


def test_not_indexed_files_take_no_space(gpu):
    rs = np.random.RandomState(21)
    files = not_indexed_files(gpu, rs)
    for dtype in ("uint8", "uint16"):
        views, st, oo, raw = ragged_index(gpu, files, dtype, max_w=64, max_h=64)
        assert (st == NOT_INDEXED).all() and (oo == 0).all() and (raw == GUARD).all(), st


def test_index_mixed_batch_and_out_of_range_palette_indices(gpu):
    rs = np.random.RandomState(22)
    labels = []
    for k in range(12):
        ctype, depth, il, t = LABEL_COMBOS[int(rs.randint(len(LABEL_COMBOS)))]
        if depth == 16:
            depth = 8
        labels.append(pf.case(rs, int(rs.randint(1, 40)), int(rs.randint(1, 30)), ctype, depth, il, t, seed=k)[:2])
    # indices at or past the palette's entry count are stored as they are
    s = rs.randint(0, 256, (6, 10, 1)).astype(np.uint32)
    labels.append((pf.make_png(s, 3, 8, plte=rs.randint(0, 256, (3, 3)), trns=b"\x00\x10"), s))
    others = not_indexed_files(gpu, rs)
    order = rs.permutation(len(labels) + len(others))
    files = [(labels + [(f, None) for f in others])[j] for j in order]
    for dtype in ("uint8", "uint16"):
        views, st, oo, raw = ragged_index(gpu, [f for f, _ in files], dtype)
        for k, (f, s) in enumerate(files):
            if s is None:
                assert st[k] == NOT_INDEXED and oo[k + 1] == oo[k], k
            else:
                assert st[k] == 0 and np.array_equal(as_np(views[k]).astype(np.int64), s.astype(np.int64)), (dtype, k)
        check_untouched(raw, oo, st)


def damaged_crc(gpu, f):
    _, _, _, _, io, il = gpu.get_png_info(f, all_formats=True)
    b = bytearray(f)
    b[io + 8 + il] ^= 0x10
    return bytes(b)


def test_status_order_with_verify_on_and_off(gpu):
    """FPNGB_DECODE_NOT_INDEXED comes right after the walk: before the shape check and the verified IDAT CRC"""
    rs = np.random.RandomState(23)
    lab = pf.case(rs, 8, 6, 3, 4)[0]
    rgb = pf.case(rs, 8, 6, 2, 8)[0]
    wide_lab, wide_rgb = pf.case(rs, 40, 6, 0, 8)[0], pf.case(rs, 40, 6, 6, 8)[0]
    files = [lab, rgb, wide_lab, wide_rgb, damaged_crc(gpu, lab), damaged_crc(gpu, rgb), b"\x89PNG" + bytes(60)]
    for verify in (False, True):
        gpu.set_decode_verify(verify)
        try:
            _, st, _, _ = ragged_index(gpu, files, "uint8", max_w=16, max_h=16)
        finally:
            gpu.set_decode_verify(False)
        assert st[0] == 0 and st[1] == NOT_INDEXED and st[2] == SHAPE_MISMATCH and st[3] == NOT_INDEXED, st
        assert st[4] == (CRC if verify else 0) and st[5] == NOT_INDEXED and st[6] not in (0, NOT_INDEXED), st


# ---- 2. nearest resize ---------------------------------------------------------------------------------------------------------------
def random_boxes(rs, dims):
    out = []
    for w, h in dims:
        bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
        out.append((int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1)), bh, bw))
    return np.array(out, np.int32)


def bits(t):
    """the element bit patterns as numpy integers (a same-size view works at any strides)"""
    import torch
    es = t.element_size()
    return (t if es == 1 else t.view({2: torch.int16, 4: torch.int32}[es])).cpu().numpy()


def nearest_call(gpu, files, d, size, dtype, mode, boxes=None, nchw=False, scale=None, bias=None, flags=None):
    """the resized call and, from the same packed files, the ragged decode with the same flags; checks every file's slice against
    the model applied to the ragged output, and against torch's CUDA F.interpolate where torch has the dtype"""
    import torch
    import torch.nn.functional as F
    flags = flags or {}
    T = getattr(torch, dtype)
    H, W = size
    data, offsets, sizes = packed(files, 3)
    px, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, dtype=T, scale=scale, bias=bias, **flags)
    views = gpu.ragged_views(px, oo, info, st, d)
    assert (st.cpu().numpy() == 0).all(), st
    n = len(files)
    out = torch.empty((n, d, H, W) if nchw else (n, H, W, d), dtype=T, device="cuda")
    if T.itemsize == 1:
        out.fill_(GUARD)
    else:
        out.view(torch.int16 if T.itemsize == 2 else torch.int32).fill_(-3)
    if nchw:
        out = out.permute(0, 2, 3, 1)
    bt = None if boxes is None else torch.from_numpy(boxes).cuda()
    _, _, st2 = gpu.decode_packed_resized_device(data, offsets, sizes, size, d, boxes=bt, out=out, scale=scale, bias=bias,
                                                 interpolation=mode, **flags)
    torch.cuda.synchronize()
    assert (st2.cpu().numpy() == 0).all(), st2
    exact = mode == "nearest-exact"
    for i, v in enumerate(views):
        if T == torch.uint16:                                                  # torch's CUDA indexing has no uint16: same bytes
            v = v.view(torch.int16)
        top, left, bh, bw = (0, 0, v.shape[0], v.shape[1]) if boxes is None else (int(x) for x in boxes[i])
        crop = v[top:top + bh, left:left + bw]
        want = crop[torch.from_numpy(nearest_src(bh, H, exact)).cuda()][:, torch.from_numpy(nearest_src(bw, W, exact)).cuda()]
        assert np.array_equal(bits(out[i]), bits(want)), (i, d, dtype, mode, size, nchw)
        if (bh, bw) == (H, W):
            assert np.array_equal(bits(out[i]), bits(crop))
        if dtype != "uint16":
            ref = F.interpolate(crop.permute(2, 0, 1)[None].contiguous(), size=size, mode=mode)[0].permute(1, 2, 0)
            assert np.array_equal(bits(out[i]), bits(ref)), (i, "torch", d, dtype, mode)
    return out


def color_files(gpu, rs, n=6):
    files = [fpng_file(gpu, int(rs.randint(3, 90)), int(rs.randint(3, 60)), c, k)[0] for k, c in enumerate((3, 4, 3))]
    files += [pf.case(rs, int(rs.randint(3, 90)), int(rs.randint(3, 60)), ct, 8, 0, False, seed=k)[0] for k, ct in enumerate((2, 6, 0))]
    return files[:n]


def native_files(rs):
    out = []
    for k, (ct, dp, il, t) in enumerate([(0, 16, 0, False), (2, 16, 1, True), (6, 8, 0, False), (3, 4, 1, True), (4, 16, 0, False),
                                         (0, 2, 0, False), (6, 16, 1, False)]):
        out.append(pf.case(rs, int(rs.randint(2, 80)), int(rs.randint(2, 50)), ct, dp, il, t, seed=k)[0])
    return out


def label_files(rs, depths=(1, 2, 4, 8, 16)):
    out = []
    for k, (ct, dp) in enumerate([(3, d) for d in (1, 2, 4, 8)] + [(0, d) for d in depths]):
        out.append(pf.case(rs, int(rs.randint(2, 90)), int(rs.randint(2, 50)), ct, dp, k % 2, False, seed=k)[0])
    return out


def dims_of(gpu, files):
    return [gpu.get_png_info(f, all_formats=True)[1:3] for f in files]


SIZES = [(1, 1), (37, 300), (64, 53), (3, 1)]


@pytest.mark.parametrize("mode", ["nearest", "nearest-exact"])
def test_nearest_uint8_color(gpu, mode):
    rs = np.random.RandomState(31)
    files = color_files(gpu, rs)
    flags = dict(any_png=True, all_formats=True)
    for d in (3, 4):
        for size in SIZES:
            for nchw in (False, True):
                boxes = random_boxes(rs, dims_of(gpu, files))
                nearest_call(gpu, files, d, size, "uint8", mode, boxes, nchw, flags=flags)
        nearest_call(gpu, files, d, (29, 31), "bfloat16", mode, random_boxes(rs, dims_of(gpu, files)), True, scale=[0.5, 2.0, -1.0, 3.0][:d],
                     bias=[1.0, -2.0, 0.25, 0.0][:d], flags=flags)
        nearest_call(gpu, files, d, (29, 31), "float32", mode, None, False, scale=1 / 255.0, flags=flags)


@pytest.mark.parametrize("mode", ["nearest", "nearest-exact"])
def test_nearest_native(gpu, mode):
    rs = np.random.RandomState(32)
    files = native_files(rs)
    for d in (1, 2, 3, 4):
        for dtype in ("uint8", "uint16", "float32", "float16"):
            for size, nchw in (((1, 1), False), ((45, 130), True), ((17, 9), False)):
                kw = dict(scale=0.5, bias=-1.0) if dtype.startswith("float") else {}
                nearest_call(gpu, files, d, size, dtype, mode, random_boxes(rs, dims_of(gpu, files)), nchw, flags=dict(FULL), **kw)


@pytest.mark.parametrize("mode", ["nearest", "nearest-exact"])
def test_nearest_index(gpu, mode):
    rs = np.random.RandomState(33)
    for dtype, files in (("uint8", label_files(rs, (1, 2, 4, 8))), ("uint16", label_files(rs))):
        for size in SIZES + [(512, 512)]:
            nearest_call(gpu, files, 1, size, dtype, mode, random_boxes(rs, dims_of(gpu, files)), flags=dict(FULL, indices=True))


def test_nearest_identity_equals_ragged_crop(gpu):
    rs = np.random.RandomState(34)
    files = label_files(rs)
    dims = dims_of(gpu, files)
    h, w = min(d[1] for d in dims), min(d[0] for d in dims)
    boxes = np.array([(int(rs.randint(0, dh - h + 1)), int(rs.randint(0, dw - w + 1)), h, w) for dw, dh in dims], np.int32)
    for mode in ("nearest", "nearest-exact"):
        nearest_call(gpu, files, 1, (h, w), "uint16", mode, boxes, flags=dict(FULL, indices=True))
        nearest_call(gpu, files, 3, (h, w), "uint8", mode, boxes, True, flags=dict(FULL))


def test_resized_index_statuses(gpu):
    """105 before BAD_CROP; the slices of rejected files keep their guard; pixel_cap counts elem bytes per pixel"""
    import torch
    rs = np.random.RandomState(35)
    lab = [pf.case(rs, 12, 10, 3, 8, seed=k)[0] for k in range(3)]
    rgb = pf.case(rs, 12, 10, 2, 8)[0]
    files = [lab[0], rgb, lab[1], rgb, lab[2]]
    data, offsets, sizes = packed(files)
    boxes = torch.tensor([[0, 0, 10, 12], [0, 0, 10, 12], [5, 5, 10, 12], [5, 5, 10, 12], [1, 1, 2, 2]], dtype=torch.int32, device="cuda")
    out = torch.full((5, 4, 4, 1), GUARD, dtype=torch.uint8, device="cuda")
    cap = 2 * ((12 * 10 + 15) // 16 * 16)                  # two label files: the last fits only if 105 and 103 take no space
    _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (4, 4), 1, boxes=boxes, out=out, max_file_size=max(map(len, files)),
                                                max_w=12, max_h=10, pixel_cap=cap, interpolation="nearest", indices=True, **FULL)
    torch.cuda.synchronize()
    assert st.cpu().tolist() == [0, NOT_INDEXED, BAD_CROP, NOT_INDEXED, 0]
    o = out.cpu().numpy()
    assert (o[1:4] == GUARD).all() and not (o[0] == GUARD).all() and not (o[4] == GUARD).all()


def test_rejected_calls(gpu):
    import torch
    from fpng_b200._lib import lib
    from fpng_b200.api import PixelFormat
    rs = np.random.RandomState(36)
    files = [pf.case(rs, 8, 8, 3, 8)[0]]
    data, offsets, sizes = packed(files)
    out = torch.full((4096,), GUARD, dtype=torch.uint8, device="cuda")
    oo = torch.full((2,), -7, dtype=torch.int64, device="cuda"); info = torch.full((1, 6), -7, dtype=torch.int32, device="cuda")
    st = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    u16 = PixelFormat(); u16.dtype = 4
    f32 = PixelFormat(); f32.dtype = 1; f32.scale[0] = 1.0
    base = (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), 1, len(files[0]), 8, 8)
    rg = lambda d, flags, fmt: lib().fpngb_decode_packed_png_device_ex(  # noqa: E731
        *base, d, out.data_ptr(), 4096, oo.data_ptr(), info.data_ptr(), flags, fmt, st.data_ptr(), None)
    rz = lambda d, flags, fmt, es=1: lib().fpngb_decode_packed_resized_device(  # noqa: E731
        *base, 4096, None, 4, 4, d, flags, fmt, out.data_ptr(), 16 * d * es, 4 * d * es, d * es, es, info.data_ptr(), st.data_ptr(), None)
    torch.cuda.synchronize()
    before = gpu.launch_count()
    for d, flags, fmt in ((1, 8, None), (1, 8 | 1, None), (1, 8 | 4, None), (3, 8 | 5, None), (0, 8 | 5, None), (2, 8 | 5, None),
                          (1, 8 | 5, C.byref(f32)), (1, 8 | 5 | 2, None), (1, 8 | 5 | 0x100, None)):
        assert rg(d, flags, fmt) == 1, (d, flags)
    for d, flags, fmt in ((3, 4 | 32 | 64, None), (3, 4 | 32 | 1, None), (3, 4 | 64 | 1, None), (3, 32 | 2, None), (3, 32 | 8, None),
                          (1, 4 | 8 | 16 | 128, None), (1, 4 | 8 | 128 | 32, None), (1, 4 | 16 | 128 | 32, None), (1, 8 | 16 | 128 | 32, None),
                          (2, 4 | 8 | 16 | 128 | 32, None), (1, 4 | 8 | 16 | 128 | 32, C.byref(f32)), (3, 128 | 32, None),
                          (1, 4 | 8 | 16 | 128 | 32 | 64, None), (1, 256 | 32, None)):
        assert rz(d, flags, fmt, 4 if fmt is not None else 1) == 1, (d, flags)
    assert lib().fpngb_get_png_info_batch_device_ex(data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), 1, 8 | 1, info.data_ptr(), None) == 1
    w, h, c, io, il = (C.c_uint32() for _ in range(5))
    f0 = np.frombuffer(files[0], np.uint8)
    assert lib().fpngb_get_png_info_ex(f0.ctypes.data_as(C.c_void_p), f0.size, 8 | 1, *(C.byref(v) for v in (w, h, c, io, il))) == 2
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out.cpu().numpy() == GUARD).all() and (oo.cpu().numpy() == -7).all() and (st.cpu().numpy() == -7).all()
    # accepted as they are, with the launches of the calls without the new flags
    assert rg(1, 8 | 5, C.byref(u16)) == 0
    torch.cuda.synchronize()
    assert gpu.launch_count() - before == 15 and st.item() == 0
    assert rz(1, 4 | 8 | 16 | 128 | 64, None) == 0
    torch.cuda.synchronize()
    assert gpu.launch_count() - before == 15 + 16 and st.item() == 0


def test_profile_slot_8_reports_the_nearest_kernel(gpu):
    import torch
    from fpng_b200._lib import lib
    rs = np.random.RandomState(37)
    files = label_files(rs)
    data, offsets, sizes = packed(files)
    L = lib()
    L.fpngb_decode_profile_enable(1)
    try:
        gpu.decode_packed_resized_device(data, offsets, sizes, (256, 256), 1, dtype=torch.uint16, interpolation="nearest", indices=True,
                                         **FULL)
        ms = (C.c_float * 9)()
        assert L.fpngb_decode_profile_read(ms, 9) == 1
        assert ms[8] > 0 and ms[6] == 0 and ms[7] == 0, list(ms)
    finally:
        L.fpngb_decode_profile_enable(0)


def test_no_host_synchronisation(gpu):
    import torch
    rs = np.random.RandomState(38)
    files = label_files(rs)
    data, offsets, sizes = packed(files)
    dims = dims_of(gpu, files)
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims),
                  pixel_cap=sum((w * h * 2 + 15) // 16 * 16 for w, h in dims))
    kw = dict(interpolation="nearest-exact", indices=True, **FULL, **bounds)
    out = torch.empty((len(files), 48, 40, 1), dtype=torch.uint16, device="cuda")
    gpu.decode_packed_resized_device(data, offsets, sizes, (48, 40), 1, out=out, **kw)     # workspace reserved first
    torch.cuda.synchronize()
    want = as_np(out)
    out.zero_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)
        _, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (48, 40), 1, out=out, **kw)
        assert not s.query(), "the call waited for the stream"
    s.synchronize()
    assert (st.cpu().numpy() == 0).all() and np.array_equal(as_np(out), want)
