"""GPU tests of fpngb_decode_packed_views_device (decode_packed_views_device): any number of output images ("views") per call, each
a crop of a file resized to its own size, flipped and placed on a filled canvas.  The expected value of every view is built from
the existing call: decode_packed_resized_device at the view's size and box, then torch.flip, then a paste onto a canvas of the
fill, compared with torch.equal.  Also: the identity table against the resized call, torchvision's eval transform and ten-crop,
image and mask alignment, view statuses and their order, rejected calls, launches, profiling, stream ordering, and the m, 4 GiB
and offset edges."""
import ctypes as C

import numpy as np
import pytest

import imagegen
import pngwrite_formats as pf
from test_decode_device_gpu import to_device
from test_decode_ragged_gpu import pack_at
from test_decode_resized_gpu import TOL_CUDA_AA, corpus, damaged, decoded

pytestmark = pytest.mark.gpu

INVALID_ARG, CRC, OUT_OF_SPACE, ADLER, BAD_CROP, BAD_VIEW = 2, 4, 101, 102, 103, 106
HFLIP, VFLIP = 1, 2
LIM = 1 << 24
FULL = dict(any_png=True, all_formats=True, native=True)


def packed(files, seed=0):
    buf, offs = pack_at(files, np.random.RandomState(seed), True)
    return to_device(buf, offs, [len(f) for f in files])


def table(rows):
    import torch
    return torch.tensor(np.asarray(rows, np.int64).reshape(-1, 10), dtype=torch.int32, device="cuda")


def sentinel_out(m, H, W, d, T, layout):
    """an output of m images in NHWC, NCHW or a strided window of a larger canvas, every element a sentinel bit pattern"""
    import torch
    if layout == "nchw":
        base = torch.empty((m, d, H, W), dtype=T, device="cuda")
    elif layout == "strided":
        base = torch.empty((m, H + 3, W + 5, d), dtype=T, device="cuda")
    else:
        base = torch.empty((m, H, W, d), dtype=T, device="cuda")
    if T.itemsize == 1:
        base.fill_(0xA5)
    else:
        base.view({2: torch.int16, 4: torch.int32}[T.itemsize]).fill_(-3)
    if layout == "nchw":
        return base.permute(0, 2, 3, 1)
    if layout == "strided":
        return base[:, 2:2 + H, 1:1 + W, :]
    return base


def fill_value(fill, d, T, scale, bias, native=False):
    """the stored fill of a call: a source value stored as the call stores one (float: fp32 fill * scale + bias, each operation
    rounded; native float: the value / 257 first; uint8 / uint16 / index: the value itself)"""
    import torch
    f = np.broadcast_to(np.asarray(fill if fill is not None else 0, np.float32), (d,)).astype(np.float32)
    if T in (torch.uint8, torch.uint16):
        return torch.tensor(f.astype(np.int64)).to(T)
    if native:
        f = (f / np.float32(257)).astype(np.float32)
    s = np.broadcast_to(np.asarray(1.0 if scale is None else scale, np.float32), (d,))
    b = np.broadcast_to(np.asarray(0.0 if bias is None else bias, np.float32), (d,))
    return torch.from_numpy(((f * s).astype(np.float32) + b).astype(np.float32)).to(T)


def expected_views(gpu, data, offsets, sizes, rows, canvas, d, T, fill, kw):
    """[m, H, W, d] on the device: per view row, the resized call at (rh, rw) with the view's box, flipped, pasted onto the fill"""
    import torch
    n = sizes.shape[0]
    H, W = canvas
    fv = fill_value(fill, d, T, kw.get("scale"), kw.get("bias"), kw.get("native", False)).cuda()
    out = fv.view(1, 1, 1, d).expand(len(rows), H, W, d).clone()
    for v, row in enumerate(rows):
        f, top, left, bh, bw, rh, rw, oy, ox, flags = (int(x) for x in row)
        boxes = torch.tensor([[0, 0, 1, 1]] * n, dtype=torch.int32)
        boxes[f] = torch.tensor([top, left, bh, bw])
        r, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, (rh, rw), d, boxes=boxes.cuda(), dtype=T, **kw)
        assert int(st[f]) == 0, (row, int(st[f]))
        r = r[f]
        if flags & HFLIP:
            r = r.flip(1)
        if flags & VFLIP:
            r = r.flip(0)
        y0, y1, x0, x1 = max(oy, 0), min(oy + rh, H), max(ox, 0), min(ox + rw, W)
        if y0 < y1 and x0 < x1:
            out[v, y0:y1, x0:x1] = r[y0 - oy:y1 - oy, x0 - ox:x1 - ox]
    return out


def same(a, b):
    """bit-for-bit equality of two tensors of one dtype (any strides)"""
    import torch
    if a.dtype.is_floating_point:
        it = {2: torch.int16, 4: torch.int32}[a.element_size()]
        return torch.equal(a.contiguous().view(it), b.contiguous().view(it))
    return torch.equal(a.contiguous(), b.contiguous())


def random_views(rs, dims, canvas, per_file=(0, 1, 2, 3)):
    """several views per file (none for some), boxes inside the image, resize sizes below and above the box (1 included),
    offsets negative, zero, positive and off the canvas, every flag value"""
    H, W = canvas
    rows, k = [], 0
    for f, (w, h) in enumerate(dims):
        for _ in range(per_file[f % len(per_file)]):
            bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
            top, left = int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1))
            rh = (1, max(1, bh // 3), bh, 2 * bh + 1, int(rs.randint(1, 150)))[k % 5]
            rw = (int(rs.randint(1, 150)), 1, 3 * bw, max(1, bw // 2), bw)[k % 5]
            rh, rw = min(rh, 300), min(rw, 300)
            oy = (0, -int(rs.randint(1, rh + 1)), int(rs.randint(0, H)), H + 2, -rh)[(k // 2) % 5]
            ox = (int(rs.randint(-rw, W)), 0, -int(rs.randint(0, rw)), int(rs.randint(0, W)), W)[(k // 3) % 5]
            rows.append((f, top, left, bh, bw, rh, rw, oy, ox, k % 4))
            k += 1
    return rows


def run_views(gpu, files, rows, canvas, d, T, layout, fill, seed=0, **kw):
    import torch
    data, offsets, sizes = packed(files, seed)
    out = sentinel_out(len(rows), canvas[0], canvas[1], d, T, layout)
    got, info, st, vst = gpu.decode_packed_views_device(data, offsets, sizes, table(rows), canvas, d, fill=fill, out=out, dtype=T, **kw)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    return (data, offsets, sizes), got, st, vst


# ---- 1. bit-exact against the resized call --------------------------------------------------------------------------------------
INTERPS = [("bilinear", True), ("bilinear", False), ("nearest", False), ("nearest-exact", False)]


@pytest.mark.parametrize("dtype", ["uint8", "float16", "bfloat16", "float32"])
def test_views_equal_resized_flip_paste(gpu, oracle, dtype):
    import torch
    T = getattr(torch, dtype)
    files = corpus(oracle, 40)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(41)
    k = 0
    for d in (3, 4):
        for interp, aa in INTERPS:
            layout = ("nhwc", "nchw", "strided")[k % 3]
            canvas = ((64, 80), (33, 17), (1, 1), (96, 96))[k % 4]
            k += 1
            rows = random_views(rs, dims, canvas)
            fill = [int(v) for v in rs.randint(0, 256, d)]
            kw = dict(antialias=aa, interpolation=interp)
            if T != torch.uint8:
                kw.update(scale=[0.5, -2.0, 1.0 / 255, 3.0][:d], bias=[1.0, 0.25, -0.5, 0.0][:d])
            pk, got, st, vst = run_views(gpu, files, rows, canvas, d, T, layout, fill, **kw)
            assert (st.cpu() == 0).all() and (vst.cpu() == 0).all(), (st, vst)
            want = expected_views(gpu, *pk, rows, canvas, d, T, fill, kw)
            for v in range(len(rows)):
                assert same(got[v], want[v]), (dtype, d, interp, aa, layout, rows[v])


def test_resize_to_one_pixel_and_offsets_at_the_limit(gpu, oracle):
    """resize_w = 1 and resize_h = 1 with antialias; offsets of +-2^24 (views entirely off the canvas hold the fill)"""
    import torch
    files = corpus(oracle, 42)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rows = []
    for f, (w, h) in enumerate(dims):
        rows += [(f, 0, 0, h, w, 1, 37, 3, -2, f % 4), (f, 0, 0, h, w, 29, 1, -1, 5, (f + 1) % 4), (f, 0, 0, h, w, 1, 1, 4, 4, 0)]
    edge = [(0, 0, 0, 1, 1, 5, 5, LIM, 0, 0), (1, 0, 0, 3, 5, 5, 5, -LIM, 0, 1), (2, 0, 0, 9, 9, 9, 9, 0, LIM, 2),
            (3, 0, 0, 9, 9, 9, 9, 0, -LIM, 3), (4, 0, 0, 9, 9, LIM, LIM, -LIM + 3, -LIM + 2, 3)]
    rows += edge
    for T, kw in ((torch.uint8, {}), (torch.float32, dict(scale=2.0, bias=-1.0))):
        pk, got, st, vst = run_views(gpu, files, rows, (8, 40), 3, T, "nhwc", [7, 8, 9], antialias=True, **kw)
        assert (vst.cpu() == 0).all()
        want = expected_views(gpu, *pk, rows[:-1], (8, 40), 3, T, [7, 8, 9], dict(antialias=True, **kw))
        for v in range(len(rows) - 1):
            assert same(got[v], want[v]), rows[v]
        fv = fill_value([7, 8, 9], 3, T, kw.get("scale"), kw.get("bias")).cuda()
        for v in range(len(rows) - 5, len(rows) - 1):                          # entirely off the canvas
            assert same(got[v], fv.expand_as(got[v]))
        # the last view: a 9 x 9 box resized to 2^24 x 2^24, flipped both ways and placed so that the canvas shows its bottom-right
        # corner, which is R's top-left: resized rows and columns 0..2 and 0..1, whose only tap is the box's pixel (0, 0)
        px, _, _ = gpu.decode_packed_resized_device(*pk, (1, 1), 3, boxes=table([(0, 0, 0, 1, 1, 0, 0, 0, 0, 0)] * len(files))[:, 1:5].contiguous(),
                                                    dtype=T, antialias=True, **kw)
        last = got[len(rows) - 1]
        assert same(last[:3, :2], px[4].expand(3, 2, 3))
        mask = torch.ones((8, 40), dtype=torch.bool, device="cuda")
        mask[:3, :2] = False
        assert same(last[mask], fv.expand(int(mask.sum()), 3))


def test_native_and_index_views(gpu):
    import torch
    rs = np.random.RandomState(43)
    files = [pf.case(rs, int(rs.randint(2, 80)), int(rs.randint(2, 50)), ct, dp, il, t, seed=k)[0]
             for k, (ct, dp, il, t) in enumerate([(0, 16, 0, False), (2, 16, 1, True), (6, 8, 0, False), (3, 4, 1, True), (4, 16, 0, False),
                                                  (0, 2, 0, False), (6, 16, 1, False)])]
    dims = [gpu.get_png_info(f, all_formats=True)[1:3] for f in files]
    for d in (1, 2, 3, 4):
        for T, fill, kw in ((torch.uint16, 40000, {}), (torch.float32, 1000, dict(scale=0.5, bias=-1.0))):
            for interp, aa in INTERPS:
                rows = random_views(rs, dims, (23, 31))
                kw2 = dict(FULL, antialias=aa, interpolation=interp, **kw)
                pk, got, st, vst = run_views(gpu, files, rows, (23, 31), d, T, ("nchw", "nhwc")[d % 2], fill, **kw2)
                assert (vst.cpu() == 0).all(), vst
                want = expected_views(gpu, *pk, rows, (23, 31), d, T, fill, kw2)
                for v in range(len(rows)):
                    assert same(got[v], want[v]), (d, T, interp, aa, rows[v])
    labels = [pf.case(rs, int(rs.randint(2, 90)), int(rs.randint(2, 50)), ct, dp, k % 2, False, seed=k)[0]
              for k, (ct, dp) in enumerate([(3, 1), (3, 2), (3, 4), (3, 8), (0, 1), (0, 4), (0, 8), (0, 16)])]
    for T, fill, fl in ((torch.uint8, 255, labels[:7]), (torch.uint16, 255, labels), (torch.uint16, 65535, labels)):
        ldims = [gpu.get_png_info(f, all_formats=True)[1:3] for f in fl]
        for interp in ("nearest", "nearest-exact"):
            rows = random_views(rs, ldims, (40, 24))
            kw2 = dict(FULL, indices=True, interpolation=interp)
            pk, got, st, vst = run_views(gpu, fl, rows, (40, 24), 1, T, "strided", fill, **kw2)
            assert (vst.cpu() == 0).all(), vst
            want = expected_views(gpu, *pk, rows, (40, 24), 1, T, fill, kw2)
            for v in range(len(rows)):
                assert same(got[v], want[v]), (T, fill, interp, rows[v])


def test_identity_table_equals_resized_call(gpu, oracle):
    import torch
    files = corpus(oracle, 44)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    rs = np.random.RandomState(45)
    data, offsets, sizes = packed(files)
    for d in (3, 4):
        for T, kw in ((torch.uint8, {}), (torch.bfloat16, dict(scale=[0.1, 0.2, 0.3, 0.4][:d], bias=-0.5))):
            for interp, aa in INTERPS:
                for canvas in ((224, 224), (31, 67)):
                    boxes = []
                    for (w, h) in dims:
                        bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
                        boxes.append((int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1)), bh, bw))
                    rows = [(i, *b, canvas[0], canvas[1], 0, 0, 0) for i, b in enumerate(boxes)]
                    a, _, st = gpu.decode_packed_resized_device(data, offsets, sizes, canvas, d, boxes=table(rows)[:, 1:5].contiguous(),
                                                                dtype=T, antialias=aa, interpolation=interp, **kw)
                    b, _, st2, vst = gpu.decode_packed_views_device(data, offsets, sizes, table(rows), canvas, d, dtype=T, antialias=aa,
                                                                    interpolation=interp, **kw)
                    assert (st.cpu() == 0).all() and (st2.cpu() == 0).all() and (vst.cpu() == 0).all()
                    assert same(a, b), (d, T, interp, aa, canvas)


# ---- 2. torchvision parity -----------------------------------------------------------------------------------------------------
def test_eval_resize_center_crop_matches_torchvision(gpu, oracle):
    import torch
    import torchvision.transforms.v2.functional as F
    files = corpus(oracle, 46)
    data, offsets, sizes = packed(files)
    info = gpu.get_info_batch_device(data, offsets, sizes)
    views = gpu.resize_crop_views(info, 256, 224)
    got, _, st, vst = gpu.decode_packed_views_device(data, offsets, sizes, views, (224, 224), 3, dtype=torch.float32)
    assert (vst.cpu() == 0).all()
    compared = 0
    for i, f in enumerate(files):
        x = torch.from_numpy(decoded(oracle, f, 3)).cuda().permute(2, 0, 1).float()
        try:
            ref = F.center_crop(F.resize(x, 256, antialias=True), [224, 224]).permute(1, 2, 0)
        except RuntimeError as e:                               # torch's CUDA antialias kernel refuses large downscales
            assert "shared memory" in str(e), e
            continue
        compared += 1
        dmax = float((ref - got[i]).abs().max())
        assert dmax <= TOL_CUDA_AA, (i, dmax)
    assert compared >= len(files) - 1


def test_ten_crop_equals_torchvision(gpu, oracle):
    import torch
    import torchvision.transforms.v2.functional as F
    files = corpus(oracle, 47)
    data, offsets, sizes = packed(files)
    info = gpu.get_info_batch_device(data, offsets, sizes)
    base = gpu.resize_crop_views(info, 256, 224).cpu().numpy()
    rows = []
    for i in range(len(files)):
        rh, rw = int(base[i, 5]), int(base[i, 6])
        h, w = int(base[i, 3]), int(base[i, 4])
        c = (int(round((rh - 224) / 2)), int(round((rw - 224) / 2)))
        anchors = [(0, 0), (0, rw - 224), (rh - 224, 0), (rh - 224, rw - 224), c]
        for flip in (0, HFLIP):
            rows += [(i, 0, 0, h, w, rh, rw, -t, -l, flip) for (t, l) in anchors]
    got, _, st, vst = gpu.decode_packed_views_device(data, offsets, sizes, table(rows), (224, 224), 3)
    assert (vst.cpu() == 0).all() and len(rows) == 10 * len(files)
    for i in range(len(files)):
        rh, rw = int(base[i, 5]), int(base[i, 6])
        r, _, _ = gpu.decode_packed_resized_device(data, offsets, sizes, (rh, rw), 3)
        crops = F.ten_crop(r[i].permute(2, 0, 1), [224, 224])
        for k in range(10):
            assert torch.equal(got[10 * i + k], crops[k].permute(1, 2, 0)), (i, k)


# ---- 3. image and mask alignment ---------------------------------------------------------------------------------------------------
def test_image_and_mask_with_one_table(gpu):
    import torch
    rs = np.random.RandomState(48)
    files_rgb, files_idx, plts = [], [], []
    for k, (w, h) in enumerate(((61, 47), (128, 9), (3, 90), (200, 150))):
        plte = rs.randint(0, 256, (21, 3)).astype(np.uint8)
        idx = rs.randint(0, 21, (h, w, 1)).astype(np.uint8)
        files_idx.append(pf.make_png(idx, 3, 8, k % 2, plte=plte, seed=k))
        files_rgb.append(pf.make_png(plte[idx[:, :, 0]], 2, 8, 0, seed=k))
        plts.append(torch.from_numpy(plte).cuda())
    dims = [gpu.get_png_info(f, all_formats=True)[1:3] for f in files_idx]
    rows = random_views(rs, dims, (50, 70), per_file=(3, 4))
    canvas = (50, 70)
    for interp in ("nearest", "nearest-exact"):
        _, rgb, _, v1 = run_views(gpu, files_rgb, rows, canvas, 3, torch.uint8, "nchw", 0, any_png=True, interpolation=interp)
        _, ids, _, v2 = run_views(gpu, files_idx, rows, canvas, 1, torch.uint8, "nhwc", 255, interpolation=interp, indices=True, **FULL)
        assert (v1.cpu() == 0).all() and (v2.cpu() == 0).all()
        for v, row in enumerate(rows):
            f, _, _, _, _, rh, rw, oy, ox, _ = row
            inside = torch.zeros(canvas, dtype=torch.bool, device="cuda")
            inside[max(oy, 0):max(min(oy + rh, canvas[0]), 0), max(ox, 0):max(min(ox + rw, canvas[1]), 0)] = True
            lab = ids[v, :, :, 0].long()
            assert torch.equal(rgb[v][inside], plts[f][lab[inside]]), row
            assert (rgb[v][~inside] == 0).all() and (lab[~inside] == 255).all(), row


# ---- 4. statuses ----------------------------------------------------------------------------------------------------------------------
def test_view_statuses_and_precedence(gpu, oracle):
    import torch
    enc = lambda k, w, h, c, s: oracle.encode(imagegen.make(k, w, h, c, s), w, h, c, 0)  # noqa: E731
    good = [enc("g1", 64, 16, 4, 1), enc("g0", 33, 7, 3, 2), enc("g2", 48, 48, 4, 4)]
    files = [good[0], good[1], good[0][:40], good[2], b""]
    walk = gpu.get_info_ex(files[2])[0]
    ok = lambda f, w, h: (f, 0, 0, h, w, 9, 13, 0, 0, 0)  # noqa: E731
    rows, want = [], []

    def add(row, st):
        rows.append(row)
        want.append(st)

    add(ok(0, 64, 16), 0)
    for bad in (-1, 5, 1 << 30):                                                # file out of range wins over everything
        add((bad, -1, -1, 0, 0, 0, 0, LIM + 1, 0, 8), BAD_VIEW)
    add((2, -1, 0, 0, 0, 0, 0, 0, 0, 8), walk)                                  # the file's status before the box and the view
    add((4, 0, 0, 1, 1, 0, 0, 0, 0, 0), INVALID_ARG)
    for box in ((-1, 0, 3, 3), (0, -1, 3, 3), (0, 0, 0, 5), (0, 0, 5, 0), (10, 0, 7, 5), (0, 60, 5, 5), (0, 0, 17, 64), (1 << 30, 0, 1 << 30, 1)):
        add((0, *box, 0, 0, LIM + 1, 0, 4), BAD_CROP)                           # the box before the view's own fields
    for f in ((0, 0, 0, 16, 64, 0, 5, 0, 0, 0), (0, 0, 0, 16, 64, 5, 0, 0, 0, 0), (0, 0, 0, 16, 64, LIM + 1, 5, 0, 0, 0),
              (0, 0, 0, 16, 64, 5, -3, 0, 0, 0), (0, 0, 0, 16, 64, 5, 5, LIM + 1, 0, 0), (0, 0, 0, 16, 64, 5, 5, -LIM - 1, 0, 0),
              (0, 0, 0, 16, 64, 5, 5, 0, LIM + 1, 0), (0, 0, 0, 16, 64, 5, 5, 0, -LIM - 1, 0), (0, 0, 0, 16, 64, 5, 5, 0, 0, 4),
              (0, 0, 0, 16, 64, 5, 5, 0, 0, -1)):
        add(f, BAD_VIEW)
    add(ok(1, 33, 7), 0)
    add((3, 5, 6, 20, 30, 11, 4, 2, -1, 3), 0)
    add(ok(3, 48, 48), 0)
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=64, max_h=48)
    cap = sum((w * h * 4 + 15) // 16 * 16 for (w, h) in ((64, 16), (33, 7), (48, 48)))
    pk, got, st, vst = run_views(gpu, files, rows, (9, 13), 4, torch.float32, "nhwc", [1, 2, 3, 4], pixel_cap=cap, **bounds)
    assert st.cpu().tolist() == [0, 0, walk, 0, INVALID_ARG]
    assert vst.cpu().tolist() == want, list(zip(vst.cpu().tolist(), want))
    oks = [v for v in range(len(rows)) if want[v] == 0]
    exp = expected_views(gpu, *pk, [rows[v] for v in oks], (9, 13), 4, torch.float32, [1, 2, 3, 4], {})
    sentinel = sentinel_out(1, 9, 13, 4, torch.float32, "nhwc")[0]
    for v in range(len(rows)):
        if want[v]:
            assert same(got[v], sentinel), v
        else:
            assert same(got[v], exp[oks.index(v)]), v
    # one byte less: the last file (index 3) gets OUT_OF_SPACE, and so do its views; the others are unaffected
    pk, got2, st, vst = run_views(gpu, files, rows, (9, 13), 4, torch.float32, "nhwc", [1, 2, 3, 4], pixel_cap=cap - 1, **bounds)
    assert st.cpu().tolist() == [0, 0, walk, OUT_OF_SPACE, INVALID_ARG]
    want2 = [OUT_OF_SPACE if (w == 0 and rows[v][0] == 3) else w for v, w in enumerate(want)]
    assert vst.cpu().tolist() == want2
    for v in range(len(rows)):
        assert same(got2[v], got[v] if want2[v] == 0 else sentinel), v


def test_verify_statuses_reach_the_views(gpu, oracle):
    import torch
    good = [oracle.encode(imagegen.make("g1", w, h, c, w), w, h, c, 0) for (w, h, c) in ((40, 20, 3), (64, 33, 4), (17, 9, 3))]
    files = [good[0], damaged(good[1], gpu, "crc"), damaged(good[2], gpu, "adler")]
    rows = [(f, 0, 0, 5, 5, 8, 8, 1, 1, f % 4) for f in (0, 1, 2, 2, 1, 0)]
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=64, max_h=33, pixel_cap=1 << 20)
    before = gpu.launch_count()
    gpu.set_decode_verify(True)
    try:
        _, got, st, vst = run_views(gpu, files, rows, (8, 8), 3, torch.float16, "nhwc", 9, **bounds)
    finally:
        gpu.set_decode_verify(False)
    assert gpu.launch_count() - before == 14
    assert st.cpu().tolist() == [0, CRC, ADLER] and vst.cpu().tolist() == [0, CRC, ADLER, ADLER, CRC, 0]
    sentinel = sentinel_out(1, 8, 8, 3, torch.float16, "nhwc")[0]
    for v in (1, 2, 3, 4):
        assert same(got[v], sentinel)


# ---- 5. rejected calls, launches, profiling, streams ------------------------------------------------------------------------------
def test_rejected_calls(gpu, oracle):
    import torch
    from fpng_b200._lib import PixelFormat, lib
    files = corpus(oracle)[:3]
    data, offsets, sizes = packed(files)
    views = table([(i, 0, 0, 1, 1, 8, 8, 0, 0, 0) for i in range(3)] * 2)
    out = torch.full((6, 8, 8, 4), -5.0, dtype=torch.float32, device="cuda")
    st = torch.full((3,), -7, dtype=torch.int32, device="cuda")
    vst = torch.full((6,), -7, dtype=torch.int32, device="cuda")
    info = torch.full((3, 6), -7, dtype=torch.int32, device="cuda")
    fmt = PixelFormat(); fmt.dtype = 1; fmt.scale[:] = [1.0] * 4
    u16 = PixelFormat(); u16.dtype = 4
    fill_ok = (C.c_uint32 * 4)(1, 2, 3, 255)
    fill_wide = (C.c_uint32 * 4)(1, 2, 3, 256)
    fill_16 = (C.c_uint32 * 4)(65535, 2, 3, 4)
    fill_17 = (C.c_uint32 * 4)(65536, 2, 3, 4)

    def args(**kw):
        a = dict(n=3, views=views.data_ptr(), m=6, flags=1, fmt=C.byref(fmt), fill=fill_ok, out=out.data_ptr(), d=4, vst=vst.data_ptr(),
                 strides=(8 * 8 * 16, 8 * 16, 16, 4))
        a.update(kw)
        return (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), a["n"], 1 << 20, 1 << 12, 1 << 12, 1 << 24, a["views"],
                a["m"], 8, 8, a["d"], a["flags"], a["fmt"], a["fill"], a["out"], *a["strides"], info.data_ptr(), st.data_ptr(), a["vst"], None)

    native = 4 | 16
    cases = [dict(m=0), dict(m=65536), dict(views=None), dict(vst=None), dict(fill=fill_wide), dict(n=0), dict(flags=2),
             dict(out=None), dict(d=2), dict(strides=(8 * 16, 8 * 16, 16, 4)),
             dict(flags=native, fmt=C.byref(u16), fill=fill_17), dict(flags=native | 1, fmt=None, fill=fill_17)]
    before = gpu.launch_count()
    for kw in cases:
        assert lib().fpngb_decode_packed_views_device(*args(**kw)) == 1, kw
    assert lib().fpngb_decode_packed_views_device(*args(strides=(8 * 8 * 16, 8 * 16 + 2, 16, 4))) == 5
    torch.cuda.synchronize()
    assert gpu.launch_count() == before
    assert (out.cpu() == -5).all() and (st.cpu() == -7).all() and (vst.cpu() == -7).all() and (info.cpu() == -7).all()
    # accepted as they are: 12 launches; a 16-bit fill in a native call; a NULL fill
    for kw in ({}, dict(flags=native, fmt=C.byref(u16), fill=fill_16, strides=(8 * 8 * 8, 8 * 8, 8, 2)), dict(fill=None)):
        before = gpu.launch_count()
        assert lib().fpngb_decode_packed_views_device(*args(**kw)) == 0, kw
        torch.cuda.synchronize()
        assert (st.cpu() == 0).all() and (vst.cpu() == 0).all()
        assert gpu.launch_count() - before == (12 if not kw.get("flags") else 15), kw


def test_launches_and_profile_slot_8(gpu, oracle):
    import torch
    from fpng_b200._lib import lib
    files = corpus(oracle)
    data, offsets, sizes = packed(files)
    rows = [(i, 0, 0, 1, 1, 30, 30, 2, 2, 0) for i in range(len(files))] * 3
    for interp in ("bilinear", "nearest"):
        for kw in ({}, dict(any_png=True)):
            b = gpu.launch_count()
            gpu.decode_packed_resized_device(data, offsets, sizes, (32, 32), 3, interpolation=interp, antialias=False, pixel_cap=1 << 24,
                                             max_file_size=1 << 20, max_w=1024, max_h=1024, **kw)
            n_resized = gpu.launch_count() - b
            b = gpu.launch_count()
            gpu.decode_packed_views_device(data, offsets, sizes, table(rows), (32, 32), 3, interpolation=interp, antialias=False,
                                           pixel_cap=1 << 24, max_file_size=1 << 20, max_w=1024, max_h=1024, **kw)
            torch.cuda.synchronize()
            assert gpu.launch_count() - b == n_resized == (12 if not kw else 15)
    L = lib()
    L.fpngb_decode_profile_enable(1)
    try:
        gpu.decode_packed_views_device(data, offsets, sizes, table(rows), (224, 224), 3, dtype=torch.bfloat16)
        ms = (C.c_float * 9)()
        assert L.fpngb_decode_profile_read(ms, 9) == 1
        assert ms[8] > 0 and ms[6] == 0 and ms[7] == 0 and ms[0] > 0, list(ms)
    finally:
        L.fpngb_decode_profile_enable(0)


def test_no_host_synchronisation(gpu, oracle):
    import torch
    files = corpus(oracle)
    data, offsets, sizes = packed(files, 1)
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    bounds = dict(max_file_size=max(len(f) for f in files), max_w=max(w for w, _ in dims), max_h=max(h for _, h in dims),
                  pixel_cap=sum((w * h * 3 + 15) // 16 * 16 for w, h in dims))
    views = table(random_views(np.random.RandomState(50), dims, (64, 64)))
    m = views.shape[0]
    out = torch.empty((m, 3, 64, 64), dtype=torch.bfloat16, device="cuda").permute(0, 2, 3, 1)
    gpu.decode_packed_views_device(data, offsets, sizes, views, (64, 64), 3, fill=[1, 2, 3], out=out, **bounds)   # workspace first
    torch.cuda.synchronize()
    want = out.float().cpu()
    out.fill_(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 30)
        _, _, st, vst = gpu.decode_packed_views_device(data, offsets, sizes, views, (64, 64), 3, fill=[1, 2, 3], out=out, **bounds)
        assert not s.query(), "the call waited for the stream"
    s.synchronize()
    assert (st.cpu() == 0).all() and (vst.cpu() == 0).all() and torch.equal(out.float().cpu(), want)


def test_two_streams_with_workspace_growth(gpu, oracle):
    import torch
    small = corpus(oracle)[:4]
    big = [oracle.encode(imagegen.make("g1", 1920, 1080, 3, k), 1920, 1080, 3, 0) for k in range(3)] + corpus(oracle, 20)
    A, B = packed(small, 2), packed(big, 2)
    dims_a = [gpu.get_info_ex(f)[1:3] for f in small]
    dims_b = [gpu.get_info_ex(f)[1:3] for f in big]
    va = table(random_views(np.random.RandomState(51), dims_a, (96, 80)))
    vb = table(random_views(np.random.RandomState(52), dims_b, (224, 224)))
    kw_a = dict(max_file_size=max(len(f) for f in small), max_w=640, max_h=448, pixel_cap=1 << 20)
    kw_b = dict(max_file_size=max(len(f) for f in big), max_w=1920, max_h=1080, pixel_cap=sum((w * h * 3 + 15) // 16 * 16 for w, h in dims_b))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for st_ in (s1, s2):
        st_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        torch.cuda._sleep(1 << 28)
        oa, _, sa, vsa = gpu.decode_packed_views_device(*A, va, (96, 80), 4, fill=9, dtype=torch.float32, scale=0.5, **kw_a)
    with torch.cuda.stream(s2):
        torch.cuda._sleep(1 << 26)
        ob, _, sb, vsb = gpu.decode_packed_views_device(*B, vb, (224, 224), 3, fill=[114, 114, 114], antialias=False, **kw_b)
    torch.cuda.synchronize()
    alone_a = gpu.decode_packed_views_device(*A, va, (96, 80), 4, fill=9, dtype=torch.float32, scale=0.5, **kw_a)[0].cpu()
    alone_b = gpu.decode_packed_views_device(*B, vb, (224, 224), 3, fill=[114, 114, 114], antialias=False, **kw_b)[0].cpu()
    assert (sa.cpu() == 0).all() and (sb.cpu() == 0).all() and (vsa.cpu() == 0).all() and (vsb.cpu() == 0).all()
    assert torch.equal(oa.cpu(), alone_a) and torch.equal(ob.cpu(), alone_b)


# ---- 6. edges ---------------------------------------------------------------------------------------------------------------------------
def test_65535_views(gpu, oracle):
    import torch
    files = corpus(oracle, 53)[:4]
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    distinct = random_views(np.random.RandomState(54), dims, (6, 5), per_file=(4, 5))
    m = 65535
    pick = np.random.RandomState(55).randint(0, len(distinct), m)
    data, offsets, sizes = packed(files)
    few, _, _, vf = gpu.decode_packed_views_device(data, offsets, sizes, table(distinct), (6, 5), 4, fill=[5, 6, 7, 8])
    many, _, _, vm = gpu.decode_packed_views_device(data, offsets, sizes, table([distinct[k] for k in pick]), (6, 5), 4, fill=[5, 6, 7, 8])
    assert (vf.cpu() == 0).all() and (vm.cpu() == 0).all() and many.shape[0] == m
    assert torch.equal(many, few[torch.from_numpy(pick).cuda()])
    want = expected_views(gpu, data, offsets, sizes, distinct, (6, 5), 4, torch.uint8, [5, 6, 7, 8], {})
    assert torch.equal(few, want)


def test_output_past_4_gib(gpu, oracle):
    """m * H * W * C past 2^32 bytes: the last view's last row, against the resized call, flip and paste"""
    import torch
    files = corpus(oracle, 56)[:5]
    dims = [gpu.get_info_ex(f)[1:3] for f in files]
    H, W, d = 1024, 1024, 4
    m = (1 << 32) // (H * W * d) + 1
    last = (4, 0, 0, dims[4][1], dims[4][0], 700, 1100, 400, -30, HFLIP | VFLIP)
    rows = [(k % 5, 0, 0, 1, 1, 3, 3, 0, 0, 0) for k in range(m - 1)] + [last]
    data, offsets, sizes = packed(files)
    out = torch.empty((m, H, W, d), dtype=torch.uint8, device="cuda")
    got, _, st, vst = gpu.decode_packed_views_device(data, offsets, sizes, table(rows), (H, W), d, fill=[1, 2, 3, 4], out=out)
    torch.cuda.synchronize()
    assert (vst.cpu() == 0).all() and m * H * W * d > 1 << 32
    want = expected_views(gpu, data, offsets, sizes, [last], (H, W), d, torch.uint8, [1, 2, 3, 4], {})[0]
    assert torch.equal(got[m - 1, H - 1], want[H - 1]) and torch.equal(got[m - 1, 400], want[400])
    assert (got[m - 2, 3:] == torch.tensor([1, 2, 3, 4], dtype=torch.uint8, device="cuda")).all()
    del out, got
    torch.cuda.empty_cache()
