"""CPU tests of the typed decode's Python layer: normalize_scale_bias, the element-to-byte stride mapping of float views and
the argument rules that need no device."""
import numpy as np
import pytest


def test_normalize_scale_bias_values():
    from fpng_b200 import normalize_scale_bias
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    s, b = normalize_scale_bias(mean, std)
    assert s.dtype == np.float32 and b.dtype == np.float32 and s.shape == (3,)
    m, sd = np.array(mean, np.float64), np.array(std, np.float64)
    assert np.array_equal(s, (1.0 / (255.0 * sd)).astype(np.float32))
    assert np.array_equal(b, (-m / sd).astype(np.float32))
    s1, b1 = normalize_scale_bias((0.5,), (0.5,), max_value=1.0)
    assert s1[0] == np.float32(2.0) and b1[0] == np.float32(-1.0)
    # close to torchvision's Normalize(mean, std)(x / 255), not necessarily equal in the last bits
    x = np.arange(256, dtype=np.float32)[:, None]
    tv = (x / np.float32(255) - np.float32(mean)) / np.float32(std)
    assert np.allclose(x * s + b, tv, rtol=0, atol=1e-5)


def test_typed_layout_maps_element_strides_to_bytes():
    import torch
    from fpng_b200 import typed_layout
    for dtype, es in ((torch.float32, 4), (torch.float16, 2), (torch.bfloat16, 2)):
        n, c, h, w = 2, 3, 5, 7
        nchw = torch.empty(n, c, h, w, dtype=dtype).permute(0, 2, 3, 1)
        assert typed_layout(nchw.shape, nchw.stride(), nchw.element_size()) == (c * h * w * es, w * es, es, h * w * es)
        nhwc = torch.empty(n, h, w, c, dtype=dtype)
        assert typed_layout(nhwc.shape, nhwc.stride(), es) == (h * w * c * es, w * c * es, c * es, es)
        crop = torch.empty(n, h + 2, w + 3, 4, dtype=dtype)[:, 1:1 + h, 2:2 + w, :]
        assert typed_layout(crop.shape, crop.stride(), es) == ((h + 2) * (w + 3) * 4 * es, (w + 3) * 4 * es, 4 * es, es)
        plane_crop = torch.empty(n, 4, h + 1, w + 2, dtype=dtype)[:, :3, :h, 1:1 + w].permute(0, 2, 3, 1)
        assert typed_layout(plane_crop.shape, plane_crop.stride(), es) == (4 * (h + 1) * (w + 2) * es, (w + 2) * es, es, (h + 1) * (w + 2) * es)
        # size-1 dimensions get the strides of a tightly packed batch, in bytes
        one = torch.empty(1, 3, 1, 1, dtype=dtype).permute(0, 2, 3, 1)
        assert typed_layout(one.shape, one.stride(), es) == (3 * es, 3 * es, 3 * es, es)
        col = torch.empty(1, 3, h, 1, dtype=dtype).permute(0, 2, 3, 1)
        assert typed_layout(col.shape, col.stride(), es) == (h * es, es, es, h * es)
    with pytest.raises(ValueError):
        typed_layout((1, 2, 2, 3), (12, 8, 4, 1), 4)                         # RGB view of RGBA pixels


def test_uint8_output_takes_no_scale_or_bias():
    import torch
    from fpng_b200.api import _out_dtype, _pixel_format
    with pytest.raises(ValueError):
        _pixel_format(torch.uint8, [1.0, 1.0, 1.0], None, 3)
    with pytest.raises(ValueError):
        _pixel_format(torch.uint8, None, 0.0, 3)
    assert _pixel_format(torch.uint8, None, None, 3) is None
    with pytest.raises(ValueError):
        _pixel_format(torch.int32, None, None, 3)
    with pytest.raises(ValueError):
        _out_dtype(torch.empty(1, dtype=torch.float16), torch.float32)
    assert _out_dtype(None, None) == torch.uint8
    f = _pixel_format(torch.bfloat16, None, [0.5, -1.0, 2.0], 3)
    assert f.dtype == 3 and list(f.scale)[:3] == [1.0, 1.0, 1.0] and list(f.bias)[:3] == [0.5, -1.0, 2.0]
    f = _pixel_format(torch.float32, 0.25, None, 4)
    assert f.dtype == 1 and list(f.scale) == [0.25] * 4 and list(f.bias) == [0.0] * 4
    with pytest.raises(ValueError):
        _pixel_format(torch.float16, [1.0, 2.0], None, 3)
