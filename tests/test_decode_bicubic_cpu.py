"""CPU tests of the bicubic rule of the resized and views decodes (include/fpng_b200.h, FPNGB_RESIZE_BICUBIC): a numpy model of the
per-axis taps and weights, checked against torch's F.interpolate(mode="bicubic", align_corners=False) on the CPU with and without
antialiasing, the places where the rule differs from the bilinear one, and the Python argument rules that fail before any device
call.

As test_decode_resized_cpu.py does for bilinear, the model computes taps and raw weights in float32, operation by operation as the
header writes them, and normalises (antialiased only) and sums in float64.  Over every in, out in 1..9 it agrees with torch's CPU
kernel to 2.6e-4 (TOL_SMALL); on larger shapes to TOL_AA with antialiasing and to TOL_PLAIN without.  The plain gap grows with the
source index, as for bilinear: torch's CPU kernel derives the tap fraction t with other roundings (0.017 at 1920 -> 224).
Antialiased output of width 1 and height above 1 is compared on a channels_last input, for the torch CPU finding recorded in
test_decode_resized_cpu.py."""
import numpy as np
import pytest

from test_decode_resized_cpu import TOL_AA, TOL_PLAIN, axis_weights

F32 = np.float32
TOL_SMALL = 3e-4
A_PLAIN, A_AA = F32(-0.75), F32(-0.5)


def cubic(d, a):
    """torch's cubic convolution kernel at float32 distances d >= 0, each operation rounded to float32"""
    d = d.astype(F32)
    c1 = ((a + F32(2)) * d - (a + F32(3))) * d * d + F32(1)
    c2 = ((a * d - F32(5) * a) * d + F32(8) * a) * d - F32(4) * a
    return np.where(d < 1, c1, np.where(d < 2, c2, F32(0))).astype(F32)


def bicubic_weights(inp, out, aa):
    """[out, inp] float64 matrix of one axis: antialiased, the span rule with support 2 * max(scale, 1) and normalised cubic(-0.5)
    weights; plain, 4 taps at floorf(real) - 1 .. + 2 clamped to the crop, cubic(-0.75) weights, not normalised"""
    scale = F32(inp) / F32(out)
    i = np.arange(out, dtype=F32)
    m = np.zeros((out, inp))
    rows = np.arange(out)
    if aa:
        sup = F32(2) * scale if scale >= 1 else F32(2)
        inv = F32(1) / scale if scale >= 1 else F32(1)
        c = scale * (i + F32(0.5))
        xmin = np.maximum((c - sup + F32(0.5)).astype(np.int64), 0)         # astype truncates toward 0, as (int) does
        xmax = np.minimum((c + sup + F32(0.5)).astype(np.int64), inp)
        xs = xmax - xmin
        j = np.arange(int(xs.max()))
        t = ((j[None, :] + xmin[:, None]).astype(F32) - c[:, None] + F32(0.5)) * inv
        w = cubic(np.abs(t), A_AA).astype(np.float64)
        w[j[None, :] >= xs[:, None]] = 0
        s = w.sum(1, keepdims=True)
        w = np.where(s != 0, w / np.where(s != 0, s, 1), w)
        for q in range(len(j)):
            ok = q < xs
            m[rows[ok], xmin[ok] + q] += w[ok, q]
        return m
    real = scale * (i + F32(0.5)) - F32(0.5)
    x0 = np.floor(real)
    t = real - x0
    d = [t + F32(1), t, F32(1) - t, F32(2) - t]
    for k in range(4):
        col = np.clip(x0.astype(np.int64) - 1 + k, 0, inp - 1)
        np.add.at(m, (rows, col), cubic(d[k], A_PLAIN).astype(np.float64))
    return m


def bicubic_model(px, out_h, out_w, aa, box=None):
    """float64 [out_h, out_w, C] resampled values of px [h, w, C] cropped to box (top, left, height, width)"""
    if box is not None:
        top, left, bh, bw = (int(v) for v in box)
        px = px[top:top + bh, left:left + bw]
    x = px.astype(np.float64)
    wy, wx = bicubic_weights(x.shape[0], out_h, aa), bicubic_weights(x.shape[1], out_w, aa)
    return np.einsum("yh,hwc,xw->yxc", wy, x, wx, optimize=True)


def torch_bicubic(x_hwc, out_h, out_w, aa):
    """torch CPU F.interpolate(mode="bicubic") of a float32 [h, w, C] image, as float64 [out_h, out_w, C]"""
    import torch
    import torch.nn.functional as F
    t = torch.from_numpy(np.ascontiguousarray(x_hwc.transpose(2, 0, 1))).float()[None]
    if aa and out_w == 1 and out_h > 1:
        t = t.contiguous(memory_format=torch.channels_last)
    r = F.interpolate(t, size=(out_h, out_w), mode="bicubic", align_corners=False, antialias=aa)
    return r[0].permute(1, 2, 0).double().numpy()


@pytest.mark.parametrize("aa", [False, True])
def test_model_matches_torch_cpu_small(aa):
    """every in, out in 1..9 on both axes"""
    rs = np.random.RandomState(3)
    for a in range(1, 10):
        for b in range(1, 10):
            x = rs.randint(0, 256, (a, b, 3)).astype(np.uint8)
            d = np.abs(bicubic_model(x, b, a, aa) - torch_bicubic(x, b, a, aa)).max()
            assert d <= TOL_SMALL, (a, b, aa, d)


CASES = [(17, 23, 40, 50), (23, 17, 11, 7), (37, 53, 224, 224), (333, 517, 224, 160), (224, 224, 37, 53), (100, 61, 13, 211),
         (1080, 1920, 224, 224), (7, 90, 3, 1), (3, 5, 1000, 1), (1, 3840, 1, 3), (2, 3840, 5, 3), (224, 224, 224, 224)]


@pytest.mark.parametrize("aa", [False, True])
def test_model_matches_torch_cpu(aa):
    """odd ratios up and down, a 1080p crop to 224, and 3840 -> 3"""
    rs = np.random.RandomState(4)
    for (h, w, H, W) in CASES:
        x = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        d = np.abs(bicubic_model(x, H, W, aa) - torch_bicubic(x, H, W, aa)).max()
        assert d <= (TOL_AA if aa else TOL_PLAIN), (h, w, H, W, aa, d)


def test_identity_weights():
    """at identity size both filters weigh the source pixel 1 and its neighbours 0, exactly"""
    for n in (1, 2, 7, 224, 3840):
        assert np.array_equal(bicubic_weights(n, n, True), np.eye(n)) and np.array_equal(bicubic_weights(n, n, False), np.eye(n))


def test_antialias_applies_when_upscaling():
    """unlike bilinear, the antialiased bicubic filter differs from the plain one below scale 1; torch agrees with each model"""
    rs = np.random.RandomState(5)
    x = rs.randint(0, 256, (17, 23, 3)).astype(np.uint8)
    aa, plain = bicubic_model(x, 40, 50, True), bicubic_model(x, 40, 50, False)
    assert np.abs(aa - plain).max() > 10
    assert np.abs(aa - torch_bicubic(x, 40, 50, True)).max() <= TOL_AA
    assert np.abs(plain - torch_bicubic(x, 40, 50, False)).max() <= TOL_AA
    # bilinear: the two coincide when upscaling
    assert np.array_equal(axis_weights(17, 40, True), axis_weights(17, 40, False))


def test_plain_taps_clamp_to_the_crop():
    """a crop is interpolated as the cropped tensor: taps left of the box read the box's first column, not the file's column
    left - 1.  A model that reads the file's neighbours differs from torch, the crop model does not."""
    rs = np.random.RandomState(6)
    px = rs.randint(0, 256, (40, 50, 3)).astype(np.uint8)
    px[:, :10] = 255
    px[:, 30:] = 0
    px[:5] = 255
    px[25:] = 0
    top, left, bh, bw = 5, 10, 20, 20
    crop = px[top:top + bh, left:left + bw]
    m = bicubic_model(px, 9, 31, False, (top, left, bh, bw))
    assert np.array_equal(m, bicubic_model(crop, 9, 31, False))
    assert np.abs(m - torch_bicubic(crop, 9, 31, False)).max() <= TOL_AA
    # the same taps read from the file (clamped to the file instead of the box) give other values at the box's edges
    wy, wx = file_edge_weights(40, top, bh, 9), file_edge_weights(50, left, bw, 31)
    edge = np.einsum("yh,hwc,xw->yxc", wy, px.astype(np.float64), wx)
    assert np.abs(edge - m).max() > 20


def file_edge_weights(size, start, length, out):
    """plain weights of a box [start, start + length) of an axis of the file, with the taps clamped to the file, not the box"""
    scale = F32(length) / F32(out)
    real = scale * (np.arange(out, dtype=F32) + F32(0.5)) - F32(0.5)
    x0 = np.floor(real).astype(np.int64)
    t = real - np.floor(real)
    d = [t + F32(1), t, F32(1) - t, F32(2) - t]
    m = np.zeros((out, size))
    for k in range(4):
        np.add.at(m, (np.arange(out), np.clip(start + x0 - 1 + k, 0, size - 1)), cubic(d[k], A_PLAIN).astype(np.float64))
    return m


@pytest.mark.parametrize("aa", [False, True])
def test_model_overshoots(aa):
    """bicubic leaves [0, 255] on a step: below 0 and above 255, as torch's float result does"""
    x = np.zeros((8, 16, 3), np.uint8)
    x[:, 8:] = 255
    m = bicubic_model(x, 8, 45, aa)
    t = torch_bicubic(x, 8, 45, aa)
    assert m.min() < -5 and m.max() > 260 and t.min() < -5 and t.max() > 260
    assert np.abs(m - t).max() <= TOL_AA


def test_python_argument_rules():
    import torch
    from fpng_b200 import FPNGB_RESIZE_BICUBIC, decode_packed_resized_device, decode_packed_views_device
    assert FPNGB_RESIZE_BICUBIC == 256
    data = torch.zeros(64, dtype=torch.uint8)
    offsets = torch.zeros(2, dtype=torch.int64)
    sizes = torch.full((2,), 16, dtype=torch.int32)
    views = torch.zeros(2, 10, dtype=torch.int32)
    idx = dict(any_png=True, all_formats=True, native=True, indices=True, desired_channels=1, interpolation="bicubic")
    for kw in (dict(interpolation="cubic"), dict(interpolation="BICUBIC"), idx, dict(idx, antialias=False),
               dict(interpolation="bicubic", antialias=True, desired_channels=2), dict(interpolation="bicubic", antialias=False, all_formats=True)):
        args = dict(size=(8, 8), desired_channels=3)
        args.update(kw)
        with pytest.raises(ValueError) as e:
            decode_packed_resized_device(data, offsets, sizes, **args)
        if kw.get("interpolation") in ("cubic", "BICUBIC"):
            assert "'bicubic'" in str(e.value)
        if kw.get("indices"):
            assert "nearest" in str(e.value)
        with pytest.raises(ValueError):
            decode_packed_views_device(data, offsets, sizes, views, **args)
    # bicubic has no default antialias (torch's F.interpolate and torchvision's resize default differently, and the two rules
    # differ at every scale); given either way, the call passes the argument checks and stops at the CPU tensors
    for f, extra in ((decode_packed_resized_device, ()), (decode_packed_views_device, (views,))):
        with pytest.raises(ValueError, match="antialias"):
            f(data, offsets, sizes, *extra, (8, 8), 3, interpolation="bicubic")
        for aa in (True, False):
            with pytest.raises((AssertionError, ValueError)) as e:
                f(data, offsets, sizes, *extra, (8, 8), 3, interpolation="bicubic", antialias=aa)
            assert "antialias" not in str(e.value) and "CUDA" in str(e.value)
