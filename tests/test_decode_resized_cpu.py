"""CPU tests of the resized decode's rule (include/fpng_b200.h, fpngb_decode_packed_resized_device): a numpy model of the per-axis
spans and weights, checked against torch's F.interpolate(mode="bilinear", align_corners=False) on the CPU, and the Python
argument rules that fail before any device call.

The model computes spans and raw weights in float32, operation by operation as the header writes them, and normalises and sums
in float64.  It agrees with torch's CPU kernel to TOL_AA with antialiasing and to TOL_PLAIN without; the larger gap without
antialiasing comes from torch's float32 `src - x0` interpolation weight at large source indices, which the tap rule computes
differently (it grows with the index: 0.014 at 1920 -> 224).

One finding: for antialiased output of width 1 and height above 1 (7x90 -> 3x1, 3x5 -> 1000x1, 8x1 -> 4x1), torch's CPU kernel on
a contiguous NCHW tensor returns the first output row for every row, so it differs from the model by tens of levels.  The same
call on the transposed input, or on a channels_last input, agrees with the model to TOL_AA, and so does torch's CUDA kernel
(tests/test_decode_resized_gpu.py, test_torch_cuda_parity).  The model is right; the comparison below uses a channels_last input
for those shapes and test_torch_cpu_width_one_rows records the failure mode."""
import numpy as np
import pytest

F32 = np.float32
TOL_AA, TOL_PLAIN = 1e-3, 0.05


def axis_weights(inp, out, aa):
    """[out, inp] float64 matrix of the normalised weights of one axis: row i holds w_j at column xmin + j"""
    scale = F32(inp) / F32(out)
    a = bool(aa) and scale >= 1
    sup = scale if a else F32(1)
    inv = F32(1) / scale if a else F32(1)
    i = np.arange(out, dtype=F32)
    c = scale * (i + F32(0.5))
    xmin = np.maximum((c - sup + F32(0.5)).astype(np.int64), 0)             # astype truncates toward 0, as (int) does
    xmax = np.minimum((c + sup + F32(0.5)).astype(np.int64), inp)
    xs = xmax - xmin
    k = int(xs.max())
    j = np.arange(k)
    t = ((j[None, :] + xmin[:, None]).astype(F32) - c[:, None] + F32(0.5)) * inv
    w = np.maximum(F32(0), F32(1) - np.abs(t)).astype(np.float64)
    w[j[None, :] >= xs[:, None]] = 0
    s = w.sum(1, keepdims=True)
    w = np.where(s != 0, w / np.where(s != 0, s, 1), w)
    m = np.zeros((out, inp))
    rows = np.arange(out)
    for q in range(k):
        ok = q < xs
        m[rows[ok], xmin[ok] + q] += w[ok, q]
    return m


def resize_model(px, out_h, out_w, aa, box=None):
    """float64 [out_h, out_w, C] resampled values of the uint8 image px [h, w, C] cropped to box (top, left, height, width)"""
    if box is not None:
        top, left, bh, bw = (int(v) for v in box)
        px = px[top:top + bh, left:left + bw]
    x = px.astype(np.float64)
    wy, wx = axis_weights(x.shape[0], out_h, aa), axis_weights(x.shape[1], out_w, aa)
    return np.einsum("yh,hwc,xw->yxc", wy, x, wx, optimize=True)


def torch_resize(x_chw, out_h, out_w, aa, channels_last=False):
    import torch
    import torch.nn.functional as F
    t = torch.from_numpy(np.ascontiguousarray(x_chw)).float()[None]
    if channels_last:
        t = t.contiguous(memory_format=torch.channels_last)
    return F.interpolate(t, size=(out_h, out_w), mode="bilinear", align_corners=False, antialias=aa)[0].double().numpy()


CASES = [(37, 53, 224, 224), (1080, 1920, 224, 224), (480, 640, 480, 640), (100, 200, 50, 100), (7, 90, 3, 1), (7, 90, 3, 2),
         (3, 5, 1000, 1), (3, 5, 1000, 2), (1, 1, 5, 9), (1, 1000, 1, 1000), (1, 1, 1000, 1), (2160, 3840, 1, 1), (1, 3840, 1, 1),
         (333, 517, 224, 160), (17, 250, 160, 7), (224, 224, 224, 224), (8, 1, 4, 1)]


@pytest.mark.parametrize("aa", [False, True])
def test_model_matches_torch_cpu(aa):
    rs = np.random.RandomState(1)
    for (h, w, H, W) in CASES:
        x = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        m = resize_model(x, H, W, aa)
        # torch's CPU antialias kernel mishandles a contiguous output of width 1 (module docstring): channels_last there
        t = torch_resize(x.transpose(2, 0, 1), H, W, aa, channels_last=aa and W == 1 and H > 1).transpose(1, 2, 0)
        d = np.abs(m - t).max()
        assert d <= (TOL_AA if aa else TOL_PLAIN), (h, w, H, W, aa, d)


def test_torch_cpu_width_one_rows():
    """the torch CPU discrepancy of the module docstring: where the contiguous NCHW result differs from the model, every output
    row equals the first one, while the transposed call agrees with the model"""
    rs = np.random.RandomState(2)
    for (h, w, H) in ((7, 90, 3), (3, 5, 1000), (8, 1, 4), (90, 7, 3)):
        x = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        m = resize_model(x, H, 1, True)
        t = torch_resize(x.transpose(2, 0, 1), H, 1, True).transpose(1, 2, 0)
        tt = torch_resize(x.transpose(2, 1, 0), 1, H, True).transpose(2, 1, 0)
        assert np.abs(m - tt).max() <= TOL_AA
        if np.abs(m - t).max() > TOL_AA:
            assert np.array_equal(t, np.broadcast_to(t[:1], t.shape)), (h, w, H)


def test_model_edges_and_identity():
    # identity: one tap of weight 1 per output; exact 2x downscale without antialiasing: two taps of 0.5
    for n in (1, 7, 224, 3840):
        assert np.array_equal(axis_weights(n, n, True), np.eye(n)) and np.array_equal(axis_weights(n, n, False), np.eye(n))
    m = axis_weights(10, 5, False)
    assert np.array_equal(m, np.kron(np.eye(5), [[0.5, 0.5]]))
    # 3840 -> 1 with antialiasing: every column, weights summing to 1; without: the two centre taps
    m = axis_weights(3840, 1, True)
    assert (m > 0).sum() == 3840 and abs(m.sum() - 1) < 1e-12
    assert np.flatnonzero(axis_weights(3840, 1, False)[0]).tolist() == [1919, 1920]
    # 1 -> 1000: every output is the single input
    assert np.array_equal(axis_weights(1, 1000, True), np.ones((1000, 1)))


def test_python_argument_rules():
    import torch
    from fpng_b200 import decode_packed_resized_device as f
    data = torch.zeros(64, dtype=torch.uint8)
    offsets = torch.zeros(2, dtype=torch.int64)
    sizes = torch.full((2,), 16, dtype=torch.int32)
    for kw in (dict(desired_channels=2), dict(desired_channels=5), dict(size=(0, 4)), dict(size=(4, (1 << 24) + 1)),
               dict(dtype=torch.int16), dict(dtype=torch.uint8, scale=2.0), dict(dtype=torch.float32, scale=[1.0, 2.0]),
               dict(boxes=torch.zeros(2, 4, dtype=torch.int64)), dict(boxes=torch.zeros(3, 4, dtype=torch.int32)),
               dict(boxes=torch.zeros(2, 4, dtype=torch.int32)), dict(boxes=[[0, 0, 1, 1]] * 2)):
        args = dict(size=(8, 8), desired_channels=3)
        args.update(kw)
        with pytest.raises(ValueError):
            f(data, offsets, sizes, **args)
