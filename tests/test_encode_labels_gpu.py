"""encode_labels_device (fpngb_encode_label_ragged_device) on the GPU: byte equality with the oracle over the corpus and at the
layout, width and height edges; byte identity with encode_png_device for gray 8 / 16; the per-image range check; round trips
through the index, colour and nearest-resized decodes; large inputs; call-level rejections."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from label_encode_cases import cases
from test_decode_labels_gpu import FULL, dims_of, nearest_call, ragged_index, random_boxes

pytestmark = pytest.mark.gpu

GUARD = 0xA5
INVALID_ARG = 2
CASES = cases()


@pytest.fixture(scope="module")
def penc():
    from label_oracle import LabelOracle
    return LabelOracle()


def dev(ids, dtype):
    import torch
    return torch.from_numpy(np.ascontiguousarray(ids).astype(dtype)).cuda()


def files_of(out, offsets, sizes):
    import torch
    torch.cuda.synchronize()
    o, s, raw = offsets.cpu().numpy(), sizes.cpu().numpy(), out.cpu().numpy()
    return [raw[o[i]:o[i] + s[i]].tobytes() if s[i] else None for i in range(len(s))], o, s


def encode(gpu, images, palette=None, depth=None, flags=0, guard=64):
    """one call into a guard-filled buffer; returns (files, offsets, sizes, guard bytes past the total)"""
    import torch
    total = int(gpu.label_slot_offsets([(t.shape[0], t.shape[1], d) for t, d in zip(images, depth_list(images, palette, depth))],
                                       pal_list(palette, len(images)))[-1])
    raw = torch.full((total + guard,), GUARD, dtype=torch.uint8, device="cuda")
    out, offsets, sizes = gpu.encode_labels_device(images, palette=palette, depth=depth, flags=flags, out=raw[:total])
    files, o, s = files_of(out, offsets, sizes)
    assert o[-1] == total
    return files, o, s, raw[total:].cpu().numpy()


def pal_list(palette, n):
    return palette if isinstance(palette, list) else [palette] * n


def depth_list(images, palette, depth):
    pals = pal_list(palette, len(images))
    ds = depth if isinstance(depth, list) else [depth] * len(images)
    return [d if d is not None else (1 if len(p) <= 2 else 2 if len(p) <= 4 else 4 if len(p) <= 16 else 8) for d, p in zip(ds, pals)]


# ---- oracle equality ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_equals_oracle(gpu, penc, case):
    want = penc.label_encode(case.ids, case.depth, case.palette, case.flags)
    for dtype in (np.uint8, np.int64) if case.depth <= 8 else (np.int64,):
        files, _, _, tail = encode(gpu, [dev(case.ids, dtype)], case.palette, case.depth, case.flags)
        assert files[0] == want, (case.name, dtype)
        assert (tail == GUARD).all()


def test_mixed_call_equals_oracle(gpu, penc):
    imgs = [dev(c.ids, np.int64) for c in CASES]
    pals = [c.palette for c in CASES]
    for flags in (0, 2):
        files, _, _, tail = encode(gpu, imgs, pals, [c.depth for c in CASES], flags)
        for c, f in zip(CASES, files):
            assert f == penc.label_encode(c.ids, c.depth, c.palette, flags), (c.name, flags)
        assert (tail == GUARD).all()


def test_views_equal_oracle(gpu, penc):
    rs = np.random.RandomState(7)
    canvas = rs.randint(0, 5, size=(61, 203)).astype(np.int64)
    for dtype in (np.uint8, np.int64):
        full = dev(canvas, dtype)
        crop = full[3:50, 7:190]                                          # odd pitch, odd origin
        views = [crop, full[5:6].expand(40, -1), full[1:40, 2:90].unsqueeze(-1), full[::3, 1:100]]   # stride-0 rows, [h, w, 1]
        pal = rs.randint(0, 256, (5, 3)).astype(np.uint8)
        files, _, _, _ = encode(gpu, views, pal, None)
        for v, f in zip(views, files):
            assert f == penc.label_encode(v.squeeze(-1).cpu().numpy().astype(np.int64), 4, pal), v.shape


@pytest.mark.parametrize("w", [1, 31, 32, 33, 1 << 24])
def test_widths_at_depth1(gpu, penc, w):
    rs = np.random.RandomState(w % 1000)
    h = 2 if w == 1 << 24 else 50                                         # 50 rows: seven 8-row CTAs of the row kernels
    ids = (rs.rand(h, w) < 0.02).astype(np.int64) if w > 64 else rs.randint(0, 2, size=(h, w)).astype(np.int64)
    files, _, _, _ = encode(gpu, [dev(ids, np.uint8), dev(ids, np.int64)], None, 1)
    want = penc.label_encode(ids, 1, None)
    assert files[0] == want and files[1] == want


def test_heights_across_ctas(gpu, penc):
    rs = np.random.RandomState(11)
    maps = [rs.randint(0, 3, size=(h, 45)).astype(np.int64) for h in (7, 8, 9, 16, 17, 63, 65, 257)]
    pal = rs.randint(0, 256, (3, 4)).astype(np.uint8)
    files, _, _, _ = encode(gpu, [dev(m, np.int64) for m in maps], pal, 2)
    for m, f in zip(maps, files):
        assert f == penc.label_encode(m, 2, pal)


# ---- byte identity with encode_png_device -------------------------------------------------------------------------------------------
def test_gray_equals_encode_png_device(gpu):
    import torch
    rs = np.random.RandomState(5)
    for flags in (0, 2):
        m8 = [rs.randint(0, k, size=(h, w)).astype(np.int64) for k, h, w in ((2, 31, 57), (21, 64, 64), (256, 9, 300))]
        m16 = [rs.randint(0, k, size=(h, w)).astype(np.int64) for k, h, w in ((3, 17, 33), (65536, 40, 21), (1000, 64, 129))]
        got8, _, _, _ = encode(gpu, [dev(m, np.uint8) for m in m8], None, 8, flags)
        got16, _, _, _ = encode(gpu, [dev(m, np.int64) for m in m16], None, 16, flags)
        ref = [dev(m, np.uint8)[..., None] for m in m8] + \
              [torch.from_numpy(m.astype(np.uint16).view(np.int16)).cuda().view(torch.uint16)[..., None] for m in m16]
        want, _, _ = files_of(*gpu.encode_png_device(ref, flags=flags))
        assert got8 + got16 == want


# ---- range check --------------------------------------------------------------------------------------------------------------------
def test_range_check(gpu, penc):
    import torch
    rs = np.random.RandomState(3)
    pal = rs.randint(0, 256, (5, 3)).astype(np.uint8)
    ok = [rs.randint(0, 5, size=(33, 70)).astype(np.int64) for _ in range(3)]
    first, last = ok[0].copy(), ok[0].copy()
    first[0, 0] = 5
    last[-1, -1] = 9
    neg = ok[1].copy()
    neg[10, 10] = -1
    for bad_map, dtypes in ((first, (np.uint8, np.int64)), (last, (np.uint8, np.int64)), (neg, (np.int64,))):
        for dtype in dtypes:
            imgs = [dev(ok[0], dtype), dev(bad_map, dtype), dev(ok[2], dtype)]
            files, o, s, tail = encode(gpu, imgs, pal, 4)
            assert s[1] == 0 and files[1] is None and (tail == GUARD).all()
            solo, _, _, _ = encode(gpu, [imgs[0], imgs[2]], pal, 4)
            assert [files[0], files[2]] == solo == [penc.label_encode(ok[0], 4, pal), penc.label_encode(ok[2], 4, pal)]
            # the decoders read the call's packed output as it is and take size 0 as an invalid argument
            data, offs, sizes = gpu.encode_labels_device(imgs, palette=pal, depth=4)
            _, _, _, st = gpu.decode_packed_ragged_device(data, offs, sizes, 1, indices=True, **FULL)
            assert st.cpu().numpy().tolist() == [0, INVALID_ARG, 0]
    # one id deep inside a 16384 x 8192 map
    big = torch.zeros((8192, 16384), dtype=torch.uint8, device="cuda")
    big[5000, 12345] = 2
    files, _, s, _ = encode(gpu, [big, big[:100]], None, 1)
    assert s[0] == 0 and s[1] > 0
    assert files[1] == penc.label_encode(np.zeros((100, 16384), np.int64), 1, None)


# ---- round trips --------------------------------------------------------------------------------------------------------------------
def test_round_trip_index_and_colour(gpu):
    import torch
    sel = [c for c in CASES if c.flags == 0]
    files = [encode(gpu, [dev(c.ids, np.int64)], c.palette, c.depth)[0][0] for c in sel]
    maps, pals = [c.ids for c in sel], [c.palette for c in sel]
    for dtype in ("uint8", "uint16"):
        idx = [k for k, c in enumerate(sel) if dtype == "uint16" or c.depth <= 8]
        views, st, _, _ = ragged_index(gpu, [files[k] for k in idx], dtype)
        assert (st == 0).all(), st
        for v, k in zip(views, idx):
            got = v.cpu().view(torch.int16).numpy().view(np.uint16) if dtype == "uint16" else v.cpu().numpy()
            assert np.array_equal(got[..., 0].astype(np.int64), sel[k].ids), sel[k].name
    # colour: a 4-channel decode gives the palette colours and tRNS alphas
    pf = [(f, m, p) for f, m, p in zip(files, maps, pals) if p is not None]
    data = np.frombuffer(b"".join(f + b"\0" * ((-len(f)) % 16) for f, _, _ in pf), np.uint8).copy()
    offs = np.cumsum([0] + [len(f) + (-len(f)) % 16 for f, _, _ in pf]).astype(np.int64)
    px, oo, info, st = gpu.decode_packed_ragged_device(torch.from_numpy(data).cuda(), torch.from_numpy(offs).cuda(),
                                                       torch.tensor([len(f) for f, _, _ in pf], dtype=torch.int32, device="cuda"), 4,
                                                       any_png=True, all_formats=True)
    assert (st.cpu().numpy() == 0).all()
    for v, (_, m, p) in zip(gpu.ragged_views(px, oo, info, st, 4), pf):
        rgba = np.concatenate([p[:, :3], p[:, 3:] if p.shape[1] == 4 else np.full((len(p), 1), 255, np.uint8)], 1)
        assert np.array_equal(v.cpu().numpy(), rgba[m])


@pytest.mark.parametrize("mode", ["nearest", "nearest-exact"])
def test_round_trip_nearest_resize(gpu, mode):
    rs = np.random.RandomState(17)
    sel = [c for c in CASES if c.flags == 0]
    files = [encode(gpu, [dev(c.ids, np.int64)], c.palette, c.depth)[0][0] for c in sel]
    for size in ((1, 1), (37, 300), (64, 53)):
        nearest_call(gpu, files, 1, size, "uint16", mode, random_boxes(rs, dims_of(gpu, files)), flags=dict(FULL, indices=True))
    lo = [f for f, c in zip(files, sel) if c.depth <= 8]
    nearest_call(gpu, lo, 1, (29, 31), "uint8", mode, None, flags=dict(FULL, indices=True))


# ---- large inputs -------------------------------------------------------------------------------------------------------------------
def test_int64_source_past_4gib(gpu, penc):
    import torch
    h, w = 16448, 32768                                                   # 4.02 GiB of int64 ids
    need = h * w * 8
    if torch.cuda.mem_get_info()[0] < 3 * need:
        pytest.skip("not enough free device memory")
    ids = torch.zeros((h, w), dtype=torch.int64, device="cuda")
    ids[-1, -5:] = 1                                                      # only reached past 4 GiB of source
    ids[-3, 7] = 1
    files, _, s, _ = encode(gpu, [ids], None, 1)
    assert s[0] > 0
    ids[-1, -1] = 2                                                       # the last id, out of range
    _, _, s2, _ = encode(gpu, [ids], None, 1)
    assert s2[0] == 0
    del ids
    data, offs = torch.from_numpy(np.frombuffer(files[0], np.uint8).copy()).cuda(), torch.zeros(2, dtype=torch.int64, device="cuda")
    px, oo, info, st = gpu.decode_packed_ragged_device(data, offs, torch.tensor([len(files[0])], dtype=torch.int32, device="cuda"), 1,
                                                       indices=True, **FULL)
    assert st.cpu().numpy().tolist() == [0]
    v = gpu.ragged_views(px, oo, info, st, 1)[0][..., 0]
    assert int(v[-1, -5:].sum()) == 5 and int(v[-3, 7]) == 1 and int(v.sum()) == 6


def test_many_masks_two_streams(gpu, penc):
    import torch
    rs = np.random.RandomState(21)
    maps = [rs.randint(0, 2, size=(int(rs.randint(1, 40)), int(rs.randint(1, 40)))).astype(np.int64) for _ in range(4096)]
    imgs = [dev(m, np.uint8) for m in maps]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    res = []
    for k, s in ((0, s1), (1, s2)):
        with torch.cuda.stream(s):
            res.append(gpu.encode_labels_device(imgs[k::2], depth=1))
    torch.cuda.synchronize()
    for k in (0, 1):
        files, _, _ = files_of(*res[k])
        for f, m in zip(files, maps[k::2]):
            assert f == penc.label_encode(m, 1, None)


# ---- rejections ---------------------------------------------------------------------------------------------------------------------
def test_rejections_enqueue_nothing(gpu):
    import torch
    from fpng_b200._lib import LabelPalette, lib
    L = lib()
    m = torch.zeros((10, 12), dtype=torch.int64, device="cuda")
    out = torch.full((1 << 16,), GUARD, dtype=torch.uint8, device="cuda")
    offs = torch.full((4,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    rgb = np.zeros((300, 4), np.uint8)

    def call(n=1, dims=(12, 10, 8, 8), strides=None, pal=None, flags=0, out_ptr=None, cap=1 << 16, ptr=None):
        ptrs = np.array([ptr if ptr is not None else m.data_ptr()] * n, np.uint64)
        d = np.array([dims] * n, np.uint32)
        st = None if strides is None else np.array([strides] * n, np.uint64)
        ps = None if pal is None else (LabelPalette * n)(*([pal] * n))
        before = gpu.launch_count()
        rc = L.fpngb_encode_label_ragged_device(n, ptrs.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p),
                                                None if st is None else st.ctypes.data_as(C.c_void_p),
                                                None if ps is None else C.cast(ps, C.c_void_p), flags,
                                                out_ptr if out_ptr is not None else out.data_ptr(), cap, offs.data_ptr(),
                                                sizes.data_ptr(), None)
        assert gpu.launch_count() == before
        return rc

    cases = [
        (1, dict(flags=1)), (1, dict(flags=4)), (1, dict(n=0)), (1, dict(n=65536)),
        (1, dict(dims=(12, 10, 3, 8))), (1, dict(dims=(12, 10, 8, 2))), (1, dict(dims=(12, 10, 16, 1))), (1, dict(dims=(0, 10, 8, 8))),
        (1, dict(dims=(12, 10, 1, 8), pal=LabelPalette(rgb.ctypes.data, 3, 3))),                    # K > 2^d
        (1, dict(dims=(12, 10, 8, 8), pal=LabelPalette(rgb.ctypes.data, 257, 3))),
        (1, dict(dims=(12, 10, 8, 8), pal=LabelPalette(rgb.ctypes.data, 4, 2))),                    # chans
        (1, dict(dims=(12, 10, 16, 8), pal=LabelPalette(rgb.ctypes.data, 4, 3))),                   # palette at depth 16
        (1, dict(dims=(12, 10, 8, 8), pal=LabelPalette(None, 4, 3))),
        (1, dict(ptr=0)),
        (2, dict(cap=16)),                                                                          # FPNGB_ERR_BUFFER_TOO_SMALL
        (5, dict(out_ptr=out.data_ptr() + 8)),                                                      # FPNGB_ERR_ALIGNMENT
        (5, dict(strides=(96, 4))),                                                                 # stride not a multiple of elem
    ]
    for want, kw in cases:
        assert call(**kw) == want, kw
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == GUARD).all() and (offs.cpu().numpy() == -7).all() and (sizes.cpu().numpy() == -7).all()
