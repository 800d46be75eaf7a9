"""GPU tests of the label-map decode at its grid-stride, fp32-index, layout, band and 4 GiB edges (cases: tests/label_edges.py).

Every comparison is exact.  A nearest output is compared with test_decode_labels_cpu's model applied to the ragged decode of the
same files with the same flags: the ragged view cropped to the box and gathered at nearest_src's rows and columns, on the device,
so every element of every output is checked.  Where torch's CUDA F.interpolate has the dtype it is a second check (uint16
values through float32, exact below 2^24).  Outputs are written into guard-filled buffers with spare room after them, and every
byte outside the view must keep its guard.  Index outputs are compared with the samples the test wrote (index_model).  Cases
that need several GB of device memory skip themselves unless three times their need is free."""
import numpy as np
import pytest

import decode_edges as de
import label_edges as le
import pngwrite_formats as pf
from test_decode_edges_gpu import _peak_memory, big_file, need_free, source  # noqa: F401  (fixtures used here)
from test_decode_labels_cpu import index_model, nearest_model, nearest_src
from test_decode_labels_gpu import color_files, label_files, native_files, random_boxes, ragged_index
from test_decode_native_gpu import as_np, packed

pytestmark = pytest.mark.gpu

GUARD = 0xA5
FULL = dict(any_png=True, all_formats=True, native=True)
INT = {1: "uint8", 2: "int16", 4: "int32"}


def ibits(t):
    """the element bit patterns as an integer tensor on the device (a same-size view works at any strides)"""
    import torch
    return t if t.element_size() == 1 and t.dtype == torch.uint8 else t.view(getattr(torch, INT[t.element_size()]))


def assert_same(got, want, what):
    import torch
    a, b = ibits(got), ibits(want)
    if not torch.equal(a, b):
        bad = (a != b).nonzero()[:4].cpu().numpy()
        pytest.fail(f"{what}: {int((a != b).sum())} elements differ, first at {bad.tolist()}")


def flags_of(native, indices):
    return dict(FULL, indices=True) if indices else dict(FULL) if native else dict(any_png=True, all_formats=True)


def ragged_views(gpu, data, offsets, sizes, d, T, flags, scale=None, bias=None):
    px, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, d, dtype=T, scale=scale, bias=bias, **flags)
    assert not st.any().item(), st.cpu().numpy()
    return gpu.ragged_views(px, oo, info, st, d)


def gathered(view, box, size, exact):
    """the model on the device: view [h, w, d] cropped to box and gathered at nearest_src's rows and columns"""
    import torch
    top, left, bh, bw = (int(v) for v in box)
    iy = torch.from_numpy(nearest_src(bh, size[0], exact) + top).cuda()
    ix = torch.from_numpy(nearest_src(bw, size[1], exact) + left).cuda()
    return ibits(view)[iy][:, ix]


def torch_nearest(view, box, size, mode):
    """torch's CUDA F.interpolate of the crop, [H, W, d] in view's dtype; uint16 through float32 (exact for 16-bit values)"""
    import torch
    import torch.nn.functional as F
    top, left, bh, bw = (int(v) for v in box)
    crop = view[top:top + bh, left:left + bw].permute(2, 0, 1)[None]
    if view.dtype == torch.uint16:
        crop = (ibits(crop).to(torch.int32) & 0xFFFF).float()
        return (F.interpolate(crop, size=size, mode=mode)[0].permute(1, 2, 0).to(torch.int32)).to(torch.int16)
    return F.interpolate(crop.contiguous(), size=size, mode=mode)[0].permute(1, 2, 0)


def guarded(T, n_elems):
    """a flat uint8 buffer of GUARD bytes and its view as n_elems elements of T"""
    import torch
    es = T.itemsize
    raw = torch.full((n_elems * es,), GUARD, dtype=torch.uint8, device="cuda")
    return raw, raw.view(T) if es > 1 else raw


def check_guard(raw, es, elem_offsets):
    """every byte of raw outside the elements at elem_offsets keeps its guard"""
    import torch
    keep = torch.ones(raw.numel(), dtype=torch.bool, device="cuda")
    e = torch.from_numpy(elem_offsets).cuda()
    for b in range(es):
        keep[e * es + b] = False
    bad = raw[keep] != GUARD
    assert not bad.any().item(), f"{int(bad.sum())} guard bytes overwritten"


def nearest_into(gpu, files_dev, size, d, T, mode, flags, out, boxes=None, scale=None, bias=None):
    _, _, st = gpu.decode_packed_resized_device(*files_dev, size, d, boxes=boxes, out=out, scale=scale, bias=bias, interpolation=mode,
                                                **flags)
    assert not st.any().item(), st.cpu().numpy()


def compare_batch(views, out, boxes, size, mode):
    """every file's slice of out against the model and against torch's CUDA F.interpolate"""
    exact = mode == "nearest-exact"
    for f, v in enumerate(views):
        box = (0, 0, v.shape[0], v.shape[1]) if boxes is None else boxes[f]
        assert_same(out[f], gathered(v, box, size, exact), f"file {f} against the model, box {tuple(box)}, {mode}")
        assert_same(out[f], torch_nearest(v, box, size, mode), f"file {f} against torch, {mode}")


# ---- 1. grid-stride loop -------------------------------------------------------------------------------------------------------
def grid_files(rs):
    return [pf.case(rs, w, h, ct, dp, seed=k)[0] for k, (w, h, ct, dp) in enumerate(le.GRID_SOURCES)]


GRID_VARIANTS = [(name, "index_uint8") for name, _ in le.GRID_CASES] + [(le.GRID_CASES[0][0], "native_uint16_d4")]


@pytest.mark.parametrize("case,variant", GRID_VARIANTS, ids=lambda v: v)
def test_grid_stride_loop(gpu, case, variant):
    """outputs of more than 65535 x 256 groups: every thread iterates, with the (row, group) carry, without it, and carrying on
    almost every step; three files with different boxes per call; one spare image after the batch"""
    import torch
    out_hw = dict(le.GRID_CASES)[case]
    rs = np.random.RandomState(70)
    files = grid_files(rs)
    dev = packed(files, 1)
    d, T, flags = (1, torch.uint8, flags_of(True, True)) if variant == "index_uint8" else (4, torch.uint16, flags_of(True, False))
    n, img = len(files), out_hw[0] * out_hw[1] * d
    need_free((n + 1) * img * T.itemsize * 2 / 1e9 + 0.5)
    views = ragged_views(gpu, *dev, d, T, flags)
    for k, mode in enumerate(le.MODES):
        boxes = le.grid_boxes(out_hw, k)
        raw, flat = guarded(T, (n + 1) * img)
        out = flat[:n * img].view(n, *out_hw, d)
        nearest_into(gpu, dev, out_hw, d, T, mode, flags, out, torch.from_numpy(boxes).cuda())
        compare_batch(views, out, boxes, out_hw, mode)
        assert (raw[n * img * T.itemsize:] == GUARD).all().item(), "the spare image was written"
        del raw, flat, out
        torch.cuda.empty_cache()


# ---- 2. fp32 source index past 2^23 ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def line_files(gpu):
    """{"wide": (data, offsets, sizes), "tall": ...}: 8-bit gray files 1 pixel high (wide) or 1 pixel wide (tall) of every FP32_LENGTHS
    length, line_pixel's samples, written by the GPU PNG encoder"""
    import torch
    out = {}
    for kind in ("wide", "tall"):
        imgs = []
        for n_in in le.FP32_LENGTHS:
            k = torch.arange(n_in, dtype=torch.int64, device="cuda")
            v = ((k * 7 + (k >> 8) * 3 + (k >> 16) * 5) & 255).to(torch.uint8)
            imgs.append(v.view(1, n_in, 1) if kind == "wide" else v.view(n_in, 1, 1))
        out[kind] = gpu.encode_png_device(imgs)
    return out


@pytest.mark.parametrize("mode", le.MODES)
def test_fp32_index_at_2_24(gpu, line_files, mode):
    """outputs 2^24 long along each axis from sources 2^24 - 1, 10,000,019 and 5,000 long: the fp32 index where it differs from
    exact arithmetic (all past 2^23 for 2^24 - 1) and the clamp at the last index"""
    import torch
    exact = mode == "nearest-exact"
    n = len(le.FP32_LENGTHS)
    for kind, size in (("wide", (1, le.FP32_OUT)), ("tall", (le.FP32_OUT, 1))):
        dev = line_files[kind]
        views = ragged_views(gpu, *dev, 1, torch.uint8, flags_of(True, True))
        for f, n_in in enumerate(le.FP32_LENGTHS):
            assert np.array_equal(views[f].cpu().numpy().ravel(), le.line_pixel(np.arange(n_in))), (kind, n_in)
        raw, flat = guarded(torch.uint8, (n + 1) * le.FP32_OUT)
        out = flat[:n * le.FP32_OUT].view(n, *size, 1)
        nearest_into(gpu, dev, size, 1, torch.uint8, mode, flags_of(True, True), out)
        got = out.cpu().numpy().reshape(n, -1)
        for f, n_in in enumerate(le.FP32_LENGTHS):
            want = le.line_pixel(nearest_src(n_in, le.FP32_OUT, exact))
            diff, clamp = le.fp32_report(n_in, le.FP32_OUT, exact)
            bad = np.nonzero(got[f] != want)[0]
            assert bad.size == 0, (kind, n_in, mode, bad[:4], np.isin(bad, diff).sum(), np.isin(bad, clamp).sum())
        compare_batch(views, out, None, size, mode)
        assert (raw[n * le.FP32_OUT:] == GUARD).all().item()


# ---- 3. output layouts --------------------------------------------------------------------------------------------------------
def layout_files(gpu, native, indices, dtype, rs):
    if indices:
        return label_files(rs, (1, 2, 4, 8) if dtype == "uint8" else (1, 2, 4, 8, 16))
    return native_files(rs) if native else color_files(gpu, rs)


def dims_of(gpu, files):
    return [gpu.get_png_info(f, all_formats=True)[1:3] for f in files]


@pytest.mark.parametrize("variant", le.layout_variants(), ids=lambda v: "%s_d%d%s" % (v[0], v[1], "_index" if v[3] else "_native" if v[2] else ""))
def test_layouts_and_row_ends(gpu, variant):
    """a canvas crop at an odd element offset, NCHW planes padded in H and W, and HCW rows, at out_w % 4 = 0 .. 3: every element of
    the view against the model and torch, every other byte of the buffer its guard"""
    import torch
    dtype, d, native, indices = variant
    T = getattr(torch, dtype)
    rs = np.random.RandomState(100 + le.layout_variants().index(variant))
    files = layout_files(gpu, native, indices, dtype, rs)
    dev = packed(files, 2)
    flags = flags_of(native, indices)
    sb = {}
    if T.is_floating_point:
        sb = dict(scale=[0.5, 2.0, -1.0, 0.25][:d], bias=[1.0, -3.0, 0.5, 0.0][:d])
    views = ragged_views(gpu, *dev, d, T, flags, **sb)
    dims = dims_of(gpu, files)
    n = len(files)
    for j, w in enumerate(le.LAYOUT_WIDTHS):
        size = (le.LAYOUT_OUT_H, w)
        for k, layout in enumerate(le.LAYOUTS):
            mode = le.MODES[(j + k) % 2]
            shape, strides, offset, total = le.layout_strides(layout, n, *size, d)
            raw, flat = guarded(T, total)
            out = flat.as_strided(shape, strides, offset)
            boxes = random_boxes(rs, dims)
            nearest_into(gpu, dev, size, d, T, mode, flags, out, torch.from_numpy(boxes).cuda(), **sb)
            compare_batch(views, out, boxes, size, mode)
            check_guard(raw, T.itemsize, le.element_offsets(strides, offset, shape))


# ---- 4. index store at band, pass and sub-byte edges -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def index_cases():
    rs = np.random.RandomState(80)
    return [(spec,) + le.index_file(rs, spec, k) for k, spec in enumerate(le.index_specs())]


@pytest.mark.parametrize("dtype", ["uint8", "uint16"])
def test_index_ragged_edges(gpu, index_cases, dtype):
    """every label format at widths 8k - 1 .. 8k + 1 over one to four bands, Adam7 files of 271 and 280 rows, palettes shorter than
    their indices, 8-bit gray with and without a tRNS key, in one indices=True call"""
    cases = [c for c in index_cases if not (dtype == "uint8" and c[0][1] == 16)]
    views, st, oo, raw = ragged_index(gpu, [c[1] for c in cases], dtype)
    assert (st == 0).all(), st
    for k, (spec, png, s) in enumerate(cases):
        assert np.array_equal(index_model(png), s)
        assert np.array_equal(as_np(views[k])[..., 0].astype(np.int64), s), (dtype, spec, le.unfilter_kernel(spec))
    keep = np.ones(raw.size, bool)
    for i in range(len(cases)):
        keep[oo[i]:oo[i + 1]] = False
    assert (raw[keep] == GUARD).all()


@pytest.mark.parametrize("dtype", ["uint8", "uint16"])
def test_index_resized_identity_edges(gpu, index_cases, dtype):
    """the same files resized at identity, one call per shape and mode: the index store read back through the nearest kernel"""
    import torch
    T = getattr(torch, dtype)
    groups = {}
    for spec, png, s in index_cases:
        if not (dtype == "uint8" and spec[1] == 16):
            groups.setdefault(s.shape, []).append((spec, png, s))
    for (h, w), cases in groups.items():
        dev = packed([c[1] for c in cases], 3)
        for mode in le.MODES:
            raw, flat = guarded(T, (len(cases) + 1) * h * w)
            out = flat[:len(cases) * h * w].view(len(cases), h, w, 1)
            nearest_into(gpu, dev, (h, w), 1, T, mode, flags_of(True, True), out)
            got = as_np(out)
            for k, (spec, _, s) in enumerate(cases):
                assert np.array_equal(got[k, ..., 0].astype(np.int64), s), (dtype, mode, spec)
            assert (raw[len(cases) * h * w * T.itemsize:] == GUARD).all().item()


# ---- 5. pairing: one box tensor, a color call and an index call ---------------------------------------------------------------
PAIR_TABLE = np.array([[(37 * k) % 256, (91 * k + 11) % 256, (53 * k + 200) % 256] for k in range(16)], np.uint8)


def test_color_and_label_calls_agree(gpu):
    """RGB images and their 4-bit palette label maps (labels a function of the color), cropped by one shared box tensor and resized
    in two stream-ordered calls: the color output is the table entry of the label output at every pixel"""
    import torch
    rs = np.random.RandomState(90)
    assert len({tuple(c) for c in PAIR_TABLE}) == 16
    dims = [(int(rs.randint(5, 90)), int(rs.randint(5, 70))) for _ in range(6)]
    labels = [rs.randint(0, 16, (h, w, 1)).astype(np.uint32) for w, h in dims]
    color = [pf.make_png(PAIR_TABLE[s[..., 0]].astype(np.uint32), 2, 8, seed=k) for k, s in enumerate(labels)]
    index = [pf.make_png(s, 3, 4, k % 2, plte=PAIR_TABLE, seed=k) for k, s in enumerate(labels)]
    cdev, idev = packed(color, 4), packed(index, 5)
    table = torch.from_numpy(PAIR_TABLE).cuda()
    bounds = lambda files, es: dict(max_file_size=max(map(len, files)), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims),  # noqa: E731
                                     pixel_cap=sum((w * h * es + 15) // 16 * 16 for w, h in dims))
    for size in ((1, 1), (37, 53), (128, 96)):
        for mode in le.MODES:
            boxes = torch.from_numpy(random_boxes(rs, dims)).cuda()
            cout = torch.full((len(dims),) + size + (3,), GUARD, dtype=torch.uint8, device="cuda")
            iout = torch.full((len(dims),) + size + (1,), GUARD, dtype=torch.uint8, device="cuda")
            _, _, cst = gpu.decode_packed_resized_device(*cdev, size, 3, boxes=boxes, out=cout, interpolation=mode, any_png=True,
                                                         all_formats=True, **bounds(color, 3))
            _, _, ist = gpu.decode_packed_resized_device(*idev, size, 1, boxes=boxes, out=iout, interpolation=mode, indices=True, **FULL,
                                                         **bounds(index, 1))
            torch.cuda.synchronize()
            assert not cst.any().item() and not ist.any().item()
            assert torch.equal(table[iout[..., 0].long()], cout), (size, mode)
            b = boxes.cpu().numpy()
            for f, s in enumerate(labels):
                want = nearest_model(s[..., 0].astype(np.uint8), *size, mode == "nearest-exact", b[f])
                assert np.array_equal(iout[f, ..., 0].cpu().numpy(), want), (f, size, mode)


# ---- 6. past 4 GiB ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", le.MODES)
def test_big_nearest_rows_past_4_gib(gpu, big_file, mode):
    """crops of the 24000 x 23000 file decoded natively to RGBA uint16: the bottom-right crop starts 4.4 GB into the intermediate,
    the full-height strip's source rows reach 4.3 GB past its base, the top-left crop is the control"""
    import torch
    exact = mode == "nearest-exact"
    for name, box in le.BIG_BOXES:
        raw, flat = guarded(torch.uint16, 2 * le.BIG_OUT[0] * le.BIG_OUT[1] * 4)
        out = flat[:le.BIG_OUT[0] * le.BIG_OUT[1] * 4].view(1, *le.BIG_OUT, 4)
        nearest_into(gpu, big_file, le.BIG_OUT, 4, torch.uint16, mode, dict(any_png=True, native=True), out,
                     torch.tensor([box], dtype=torch.int32, device="cuda"))
        top, left, bh, bw = box
        iy, ix = nearest_src(bh, le.BIG_OUT[0], exact), nearest_src(bw, le.BIG_OUT[1], exact)
        rows = [de.big_fetch((top + int(r), left))(0, 1, 0, bw)[0] for r in iy]
        want = np.stack(rows)[:, ix]
        assert np.array_equal(as_np(out[0]).astype(np.int64), want), (name, mode)
        assert (raw[out.numel() * 2:] == GUARD).all().item()
        del raw, flat, out
        torch.cuda.empty_cache()


def test_nearest_batch_past_4_gib(gpu):
    """9 files resized by nearest to 8192 x 8192 RGBA uint16, 512 MiB each: the last starts at byte 2^32 of the output"""
    import torch
    need_free((de.BATCH_N + 1) * le.BATCH_IMAGE / 1e9 + 1.0)
    files = [source(11 + k, 13 + 2 * k, 4, True, 40 + k)[0] for k in range(le.BATCH_N)]
    dev = packed(files, 6)
    views = ragged_views(gpu, *dev, 4, torch.uint16, flags_of(True, False))
    img = le.BATCH_IMAGE // 2
    raw, flat = guarded(torch.uint16, (le.BATCH_N + 1) * img)
    out = flat[:le.BATCH_N * img].view(le.BATCH_N, *le.BATCH_OUT, 4)
    nearest_into(gpu, dev, le.BATCH_OUT, 4, torch.uint16, "nearest-exact", flags_of(True, False), out)
    for f in (0, 1, le.BATCH_N - 2, le.BATCH_N - 1):
        v = views[f]
        assert_same(out[f], gathered(v, (0, 0, v.shape[0], v.shape[1]), le.BATCH_OUT, True), f"file {f}")
    assert (raw[le.BATCH_N * le.BATCH_IMAGE:] == GUARD).all().item()
    del raw, flat, out, views
    torch.cuda.empty_cache()


def test_index_batch_past_4_gib(gpu):
    """eight 16384 x 16384 8-bit gray id maps decoded to uint16 (512 MiB each), then an Adam7 4-bit palette file and a 16-bit gray
    file, placed at output bytes >= 2^32: the index stores of both unfilter kernels there"""
    import torch
    need_free(10)
    S = le.INDEX_BIG_SIDE
    parts = []
    y = torch.arange(S, dtype=torch.int64, device="cuda")[:, None]
    x = torch.arange(S, dtype=torch.int64, device="cuda")[None, :]
    for k in range(le.INDEX_BIG_N):
        img = (((y >> 3) * 7 + (x >> 5) * 13 + k * 29 + ((x ^ y) & 1)) & 255).to(torch.uint8)[..., None]
        data, offsets, sizes = gpu.encode_png_device([img])
        o, n = int(offsets[0].item()), int(sizes[0].item())
        parts.append(data[o:o + n].clone())
        del img, data
    del x, y
    torch.cuda.empty_cache()
    rs = np.random.RandomState(95)
    tail = []
    for k, (ct, dp, il, t, w, h) in enumerate(le.INDEX_BIG_TAIL):
        png, s, _, _ = pf.case(rs, w, h, ct, dp, il, t, seed=k)
        tail.append((png, s[..., 0].astype(np.int64)))
        parts.append(torch.from_numpy(np.frombuffer(png, np.uint8).copy()).cuda())
    offs, at = [], 0
    for p in parts:
        offs.append(at)
        at += (p.numel() + 15) // 16 * 16
    data = torch.zeros(at, dtype=torch.uint8, device="cuda")
    for o, p in zip(offs, parts):
        data[o:o + p.numel()] = p
    offsets = torch.tensor(offs, dtype=torch.int64, device="cuda")
    sizes = torch.tensor([p.numel() for p in parts], dtype=torch.int32, device="cuda")
    del parts
    out, oo, info, st = gpu.decode_packed_ragged_device(data, offsets, sizes, 1, dtype=torch.uint16, indices=True, **FULL)
    assert not st.any().item(), st.cpu().numpy()
    place = oo.cpu().numpy()
    assert np.array_equal(place, le.index_big_placement()), place
    views = gpu.ragged_views(out, oo, info, st, 1)
    rows = de.sample_rows(S, 4, 9)
    for k in range(le.INDEX_BIG_N):
        got = ibits(views[k])[torch.as_tensor(rows, device="cuda"), :, 0].cpu().numpy().view(np.uint16).astype(np.int64)
        assert np.array_equal(got, le.index_big_id(k, rows[:, None], np.arange(S)[None, :])), k
    for k, (png, s) in enumerate(tail):
        assert place[le.INDEX_BIG_N + k] >= le.FOUR_GIB
        assert np.array_equal(as_np(views[le.INDEX_BIG_N + k])[..., 0].astype(np.int64), s), k
        assert np.array_equal(index_model(png), s)
    del out, views, data
    torch.cuda.empty_cache()
