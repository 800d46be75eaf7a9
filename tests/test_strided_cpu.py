"""The stride helper of the strided device calls (fpng_b200.layout_strides): byte strides of an [n, h, w, chans] uint8 view ->
the four strides of the C ABI, with size-1 dimensions canonicalised and everything but the interleaved and planar layouts
rejected.  The C side (csrc/layout.h) applies the same rules; tests/test_strided_gpu.py checks its rejections."""
import numpy as np
import pytest
import torch

from fpng_b200 import layout_strides


def strides_of(t):
    return layout_strides(t.shape, t.stride())


@pytest.mark.parametrize("c", [3, 4])
def test_contiguous_nhwc_is_tight_interleaved(c):
    t = torch.empty(5, 7, 9, c, dtype=torch.uint8)
    assert strides_of(t) == (7 * 9 * c, 9 * c, c, 1)


@pytest.mark.parametrize("c", [3, 4])
def test_interleaved_crops_and_pitches(c):
    canvas = torch.empty(3, 40, 100, c, dtype=torch.uint8)
    assert strides_of(canvas[:, 5:25, 13:60, :]) == (40 * 100 * c, 100 * c, c, 1)
    rows = torch.empty(2, 10, 33 * c + 7, dtype=torch.uint8)[:, :, : 33 * c].view(2, 10, 33, c)   # padded rows
    assert strides_of(rows) == (10 * (33 * c + 7), 33 * c + 7, c, 1)


@pytest.mark.parametrize("c", [3, 4])
def test_planar_nchw_and_hcw(c):
    x = torch.empty(4, c, 6, 11, dtype=torch.uint8)
    assert strides_of(x.permute(0, 2, 3, 1)) == (c * 6 * 11, 11, 1, 6 * 11)
    hcw = torch.empty(4, 6, c, 11, dtype=torch.uint8)
    assert strides_of(hcw.permute(0, 1, 3, 2)) == (6 * c * 11, c * 11, 1, 11)
    four = torch.empty(2, 4, 6, 11, dtype=torch.uint8)                          # RGB / RGBA planes sliced out of 4 planes
    assert strides_of(four[:, 1:1 + 3].permute(0, 2, 3, 1) if c == 3 else four.permute(0, 2, 3, 1)) == (4 * 66, 11, 1, 66)


def test_planar_with_odd_plane_stride():
    big = torch.empty(3 * 101 + 5, dtype=torch.uint8)
    v = big.as_strided((1, 10, 10, 3), (0, 10, 1, 101))
    assert strides_of(v) == (100, 10, 1, 101)


@pytest.mark.parametrize("c", [3, 4])
def test_size_one_dimensions_in_every_position(c):
    # n == 1: the image stride is ignored (tight value)
    assert layout_strides((1, 5, 6, c), (12345, 6 * c, c, 1)) == (5 * 6 * c, 6 * c, c, 1)
    assert layout_strides((1, 5, 6, c), (7, 6, 1, 30)) == (5 * 6, 6, 1, 30)
    # h == 1: the row pitch is ignored
    assert layout_strides((2, 1, 6, c), (999, 3, c, 1)) == (999, 6 * c, c, 1)
    assert layout_strides((2, 1, 6, c), (999, 3, 1, 6)) == (999, 6, 1, 6)
    # w == 1: interleaved when chan_stride == 1, planar otherwise (torch reports any pixel stride for it)
    assert layout_strides((2, 5, 1, c), (5 * c, c, 77, 1)) == (5 * c, c, c, 1)
    assert layout_strides((2, 5, 1, c), (5 * c, 1, 77, 5)) == (5 * c, 1, 1, 5)
    # all of them at once
    assert layout_strides((1, 1, 1, c), (0, 0, 0, 1)) == (c, c, c, 1)
    assert layout_strides((1, 1, 1, c), (0, 0, 0, 9)) == (1, 1, 1, 9)
    # what torch reports for real size-1 views
    x = torch.empty(1, c, 1, 1, dtype=torch.uint8).permute(0, 2, 3, 1)
    assert strides_of(x) == (c, c, c, 1)
    y = torch.empty(3, c, 8, 1, dtype=torch.uint8).permute(0, 2, 3, 1)
    assert strides_of(y) == (c * 8, 1, 1, 8)


@pytest.mark.parametrize("c", [3, 4])
def test_stride_zero_batches(c):
    img = torch.empty(1, 9, 13, c, dtype=torch.uint8)
    assert strides_of(img.expand(6, -1, -1, -1)) == (0, 13 * c, c, 1)
    planes = torch.empty(1, c, 9, 13, dtype=torch.uint8).expand(6, -1, -1, -1).permute(0, 2, 3, 1)
    assert strides_of(planes) == (0, 13, 1, 9 * 13)
    rows = torch.empty(1, 1, 13, c, dtype=torch.uint8).expand(2, 9, -1, -1)      # every row the same: row pitch 0 (read-only input)
    assert strides_of(rows) == (0, 0, c, 1)


def test_rejections():
    rgba = torch.empty(2, 5, 6, 4, dtype=torch.uint8)
    with pytest.raises(ValueError, match="interleaved.*planar"):
        strides_of(rgba[..., :3])                                               # RGB view of RGBA pixels
    with pytest.raises(ValueError):
        layout_strides((2, 5, 6, 3), (90, 18, 3, 0))                            # interleaved pixels, channel stride 0
    with pytest.raises(ValueError):
        layout_strides((2, 5, 6, 3), (90, 18, 1, 0))                            # planar, channel stride 0
    with pytest.raises(ValueError):
        layout_strides((2, 5, 6, 3), (90, 18, 2, 1))                            # neither pixel stride
    with pytest.raises(ValueError):
        layout_strides((2, 5, 6, 3), (90, 18, 6, 2))                            # every other byte
    with pytest.raises(ValueError):
        layout_strides((2, 5, 6, 3), (90, -18, 3, 1))                           # negative strides
    with pytest.raises(ValueError):
        layout_strides((2, 5, 6, 2), (60, 12, 2, 1))                            # 2 channels
    with pytest.raises(ValueError):
        strides_of(torch.empty(2, 6, 5, 3, dtype=torch.uint8).transpose(1, 2))  # columns as rows: pixel stride 15


def test_numpy_views_map_the_same_way():
    a = np.empty((3, 4, 5, 6), np.uint8)
    v = a.transpose(0, 2, 3, 1)[..., 1:4]                                       # NCHW -> [n, h, w, 3] planes 1..3
    assert layout_strides(v.shape, v.strides) == (120, 6, 1, 30)
