"""CPU tests of the views decode (include/fpng_b200.h, fpngb_decode_packed_views_device): a numpy model of one view (the resized
model of test_decode_resized_cpu.py or the nearest model of test_decode_labels_cpu.py, then a flip and a paste onto a filled
canvas) checked against torchvision v2 on CPU tensors; the geometry helpers resize_crop_views and letterbox_views against
torchvision's public functions and a plain statement of the letterbox rule; and the Python argument rules that fail before the
library is called."""
import numpy as np
import pytest

from test_decode_labels_cpu import nearest_model
from test_decode_resized_cpu import TOL_AA, TOL_PLAIN, resize_model

HFLIP, VFLIP = 1, 2


def view_model(px, row, canvas, fill, interpolation="bilinear", aa=True):
    """float64 [H, W, C] of one view row (file, top, left, height, width, rh, rw, oy, ox, flags) of the uint8 image px [h, w, C]:
    the resize model at (rh, rw), the flips, and a paste at (oy, ox) onto a canvas of fill"""
    _, top, left, bh, bw, rh, rw, oy, ox, flags = (int(v) for v in row)
    box = (top, left, bh, bw)
    if interpolation == "bilinear":
        r = resize_model(px, rh, rw, aa, box)
    else:
        r = nearest_model(px, rh, rw, interpolation == "nearest-exact", box).astype(np.float64)
    if flags & HFLIP:
        r = r[:, ::-1]
    if flags & VFLIP:
        r = r[::-1]
    H, W = canvas
    out = np.empty((H, W, px.shape[2]))
    out[:] = np.asarray(fill, np.float64)
    y0, y1, x0, x1 = max(oy, 0), min(oy + rh, H), max(ox, 0), min(ox + rw, W)
    if y0 < y1 and x0 < x1:
        out[y0:y1, x0:x1] = r[y0 - oy:y1 - oy, x0 - ox:x1 - ox]
    return out


def tv_view(px, row, canvas, fill, aa):
    """the same view by torchvision v2 functionals on a CPU tensor: crop, resize, flips, then pad or crop onto the canvas"""
    import torch
    import torchvision.transforms.v2.functional as F
    _, top, left, bh, bw, rh, rw, oy, ox, flags = (int(v) for v in row)
    x = torch.from_numpy(np.ascontiguousarray(px)).permute(2, 0, 1).float()
    x = F.crop(x, top, left, bh, bw)
    x = F.resize(x, [rh, rw], antialias=aa)
    if flags & HFLIP:
        x = F.hflip(x)
    if flags & VFLIP:
        x = F.vflip(x)
    H, W = canvas
    # place: pad (left, top, right, bottom) where positive, crop where negative
    l, t, r, b = ox, oy, W - ox - rw, H - oy - rh
    x = F.pad(x, [max(l, 0), max(t, 0), max(r, 0), max(b, 0)], fill=list(map(float, fill)))
    x = x[:, max(-t, 0):x.shape[1] - max(-b, 0), max(-l, 0):x.shape[2] - max(-r, 0)]
    return x.permute(1, 2, 0).double().numpy()


def test_view_model_matches_torchvision_cpu():
    rs = np.random.RandomState(3)
    checked = 0
    for (h, w) in ((37, 53), (120, 90), (9, 200), (64, 64)):
        px = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        for _ in range(12):
            bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
            top, left = int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1))
            rh, rw = int(rs.randint(2, 90)), int(rs.randint(2, 90))
            canvas = (int(rs.randint(1, 80)), int(rs.randint(1, 80)))
            oy, ox = int(rs.randint(-rh, canvas[0] + 1)), int(rs.randint(-rw, canvas[1] + 1))
            row = (0, top, left, bh, bw, rh, rw, oy, ox, int(rs.randint(0, 4)))
            fill = [int(v) for v in rs.randint(0, 256, 3)]
            for aa in (True, False):
                got = view_model(px, row, canvas, fill, aa=aa)
                want = tv_view(px, row, canvas, fill, aa)
                assert got.shape == want.shape
                assert np.abs(got - want).max() <= (TOL_AA if aa else TOL_PLAIN), (row, canvas, aa)
                checked += 1
    assert checked == 96


def test_view_model_identity_and_off_canvas():
    px = np.arange(5 * 7 * 3, dtype=np.uint8).reshape(5, 7, 3)
    full = (0, 0, 0, 5, 7, 5, 7, 0, 0, 0)
    for interp in ("bilinear", "nearest", "nearest-exact"):
        assert np.array_equal(view_model(px, full, (5, 7), (0, 0, 0), interp), px)
        flipped = view_model(px, full[:9] + (HFLIP | VFLIP,), (5, 7), (0, 0, 0), interp)
        assert np.array_equal(flipped, px[::-1, ::-1])
        assert (view_model(px, (0, 0, 0, 5, 7, 5, 7, 5, -7, 0), (5, 7), (9, 8, 7), interp) == [9, 8, 7]).all()


# ---- geometry helpers ----------------------------------------------------------------------------------------------------------
def grid():
    """(h, w) from 1 to about 2000: small sides, both orientations, squares, and sides around the crop and resize values"""
    sides = sorted({1, 2, 3, 7, 100, 111, 223, 224, 225, 255, 256, 257, 299, 300, 333, 375, 480, 500, 511, 640, 801, 1080, 1333, 1999})
    return [(h, w) for h in sides for w in sides]


def info_of(dims):
    import torch
    info = torch.zeros((len(dims), 6), dtype=torch.int32)
    info[:, 1] = torch.tensor([w for _, w in dims])
    info[:, 2] = torch.tensor([h for h, _ in dims])
    return info


RESIZE_CROP = [(256, 224, None), (224, 224, None), (232, 224, None), (256, 224, 300), (300, 299, None), (64, 100, None),
               ((240, 320), 224, None), ((100, 200), (300, 150), None), (256, (224, 300), None), (255, 224, 400)]


@pytest.mark.parametrize("resize,crop,max_size", RESIZE_CROP)
def test_resize_crop_views_match_torchvision(resize, crop, max_size):
    import torch
    import torchvision.transforms.v2.functional as F
    from fpng_b200 import resize_crop_views
    dims = grid()
    table = resize_crop_views(info_of(dims), resize, crop, max_size=max_size).numpy()
    assert table.dtype == np.int32 and table.shape == (len(dims), 10)
    ch, cw = (crop, crop) if isinstance(crop, int) else crop
    for i, (h, w) in enumerate(dims):
        row = table[i]
        assert tuple(row[:5]) == (i, 0, 0, h, w) and row[9] == 0
        size = resize if isinstance(resize, int) else list(resize)
        try:
            rh, rw = F.resize(torch.zeros(1, h, w, dtype=torch.uint8), size, interpolation=F.InterpolationMode.NEAREST,
                              max_size=max_size).shape[-2:]
        except RuntimeError:        # max_size squeezes the shorter side of a thin image to 0: torchvision refuses, the call gives BAD_VIEW
            assert max_size is not None and min(row[5], row[6]) == 0, (h, w, tuple(row))
            continue
        assert (row[5], row[6]) == (rh, rw), (h, w, tuple(row), (rh, rw))
        # offsets: where centre_crop takes its first pixel from (values are 1 + the resized index; 0 is torchvision's padding)
        cc = F.center_crop(torch.arange(1, rh * rw + 1, dtype=torch.float64).view(1, rh, rw), [ch, cw])[0].numpy()
        got = np.zeros((ch, cw))
        oy, ox = int(row[7]), int(row[8])
        ys, xs = np.arange(ch)[:, None] - oy, np.arange(cw)[None, :] - ox
        inside = (ys >= 0) & (ys < rh) & (xs >= 0) & (xs < rw)
        got[inside] = (ys * rw + xs + 1)[inside]
        assert np.array_equal(got, cc), (h, w, tuple(row))


def test_resize_crop_views_cover_padding_and_ties():
    """the grid reaches a crop that pads on each axis, and .5 ties of both parities, at torchvision's eval setting"""
    from fpng_b200 import resize_crop_views
    dims = grid()
    t = resize_crop_views(info_of(dims), 256, 300).numpy()
    assert (t[:, 5] < 300).any() and (t[:, 6] < 300).any() and (t[:, 7] > 0).any() and (t[:, 8] > 0).any()
    t = resize_crop_views(info_of(dims), 256, 224).numpy()
    half = (t[:, 6] - 224) / 2
    odd = t[:, 6] % 2 == 1
    assert odd.any() and set(np.floor(half[odd]).astype(int) % 2) == {0, 1}      # .5 ties rounding down and up


def letterbox_rule(h, w, H, W):
    r = min(H / h, W / w)
    rw, rh = max(round(w * r), 1), max(round(h * r), 1)
    return rh, rw, round((H - rh) / 2 - 0.1), round((W - rw) / 2 - 0.1)


@pytest.mark.parametrize("canvas", [(640, 640), (384, 640), (512, 320), (1, 1), (7, 1000)])
def test_letterbox_views_match_the_rule(canvas):
    from fpng_b200 import letterbox_views
    dims = grid()
    t = letterbox_views(info_of(dims), canvas).numpy()
    H, W = canvas
    for i, (h, w) in enumerate(dims):
        assert tuple(t[i, :5]) == (i, 0, 0, h, w) and t[i, 9] == 0
        rh, rw, oy, ox = letterbox_rule(h, w, H, W)
        assert tuple(t[i, 5:9]) == (rh, rw, oy, ox), (h, w, canvas, tuple(t[i]))
        assert 0 <= oy and oy + rh <= H and 0 <= ox and ox + rw <= W, (h, w, canvas, tuple(t[i]))


# ---- Python argument rules (no device call) -------------------------------------------------------------------------------------
def test_python_argument_rules():
    import torch
    from fpng_b200 import decode_packed_views_device as f
    good = torch.zeros((2, 10), dtype=torch.int32)
    bad_tables = [torch.zeros((2, 10), dtype=torch.int64), torch.zeros((2, 9), dtype=torch.int32), torch.zeros(20, dtype=torch.int32),
                  torch.zeros((10, 2), dtype=torch.int32).t(), torch.zeros((0, 10), dtype=torch.int32),
                  torch.zeros((65536, 10), dtype=torch.int32), [[0] * 10]]
    for t in bad_tables:
        with pytest.raises(ValueError, match="views"):
            f(None, None, None, t, (8, 8), 3)
    for fill, kw in (([1, 2], {}), ([1, 2, 3, 4], {}), (256, {}), (-1, {}), ([0, 0, 300], {}), (1.5, {}),
                     (65536, dict(any_png=True, native=True)), (256, dict(any_png=True, all_formats=True, native=True, indices=True,
                                                                          interpolation="nearest", desired_channels=1))):
        args = dict(desired_channels=3)
        args.update(kw)
        d = args.pop("desired_channels")
        with pytest.raises(ValueError, match="fill"):
            f(None, None, None, good, (8, 8), d, fill=fill, **args)
    with pytest.raises(ValueError, match="nearest"):
        f(None, None, None, good, (8, 8), 1, any_png=True, all_formats=True, native=True, indices=True)     # bilinear on ids
    for kw in (dict(desired_channels=2), dict(size=(0, 4)), dict(dtype=torch.int16), dict(dtype=torch.uint8, scale=2.0),
               dict(interpolation="bicubic")):
        args = dict(size=(8, 8), desired_channels=3)
        args.update(kw)
        with pytest.raises(ValueError):
            f(None, None, None, good, **args)
    with pytest.raises(ValueError, match="CUDA"):            # a valid CPU table
        f(None, None, None, good, (8, 8), 3, fill=[1, 2, 3])


def test_constants():
    import os
    import re
    import fpng_b200 as fb
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "fpng_b200.h")).read()
    values = {k: int(v) for k, v in re.findall(r"(FPNGB_[A-Z0-9_]+) = (\d+)", header)}
    for name in ("FPNGB_VIEW_HFLIP", "FPNGB_VIEW_VFLIP", "FPNGB_DECODE_BAD_VIEW"):
        assert getattr(fb, name) == values[name], name
    assert (fb.FPNGB_VIEW_HFLIP, fb.FPNGB_VIEW_VFLIP, fb.FPNGB_DECODE_BAD_VIEW) == (1, 2, 106)
