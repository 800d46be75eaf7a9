"""CPU tests of the typed encode's Python layer and of its quantisation rule: denormalize_scale_bias, the decode -> encode round
trip over all 256 values of every channel, the rule on ties, signed zeros, infinities, NaN, subnormals and float16 overflow, and
the argument rules that need no device."""
import numpy as np
import pytest

IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
CLIP = ((0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711))
UNIT = ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
PM1 = ((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))


def quantize(x, scale, bias):
    """the typed encode's rule (include/fpng_b200.h) in torch: x [..., c] of any float dtype -> uint8"""
    import torch
    s = torch.as_tensor(np.asarray(scale, np.float32))
    b = torch.as_tensor(np.asarray(bias, np.float32))
    return torch.nan_to_num(x.float() * s + b, nan=0.0).round().clamp(0, 255).to(torch.uint8)


def round_trip(dtype, mean, std):
    """[256, 3] uint8: every value of every channel decoded with normalize_scale_bias(mean, std) into dtype (the typed decode's
    T(v * s + b)) and encoded back with denormalize_scale_bias(mean, std)"""
    import torch
    from fpng_b200 import denormalize_scale_bias, normalize_scale_bias
    v = torch.arange(256, dtype=torch.float32)[:, None].expand(256, 3)
    sn, bn = normalize_scale_bias(mean, std)
    x = (v * torch.from_numpy(sn) + torch.from_numpy(bn)).to(dtype)
    sd, bd = denormalize_scale_bias(mean, std)
    return quantize(x, sd, bd)


def test_denormalize_scale_bias_values():
    from fpng_b200 import denormalize_scale_bias
    for mean, std in (IMAGENET, CLIP, UNIT, PM1):
        s, b = denormalize_scale_bias(mean, std)
        assert s.dtype == np.float32 and b.dtype == np.float32 and s.shape == (3,)
        assert np.array_equal(s, (255.0 * np.array(std, np.float64)).astype(np.float32))
        assert np.array_equal(b, (255.0 * np.array(mean, np.float64)).astype(np.float32))
    s, b = denormalize_scale_bias((0.5,), (0.5,))
    assert s[0] == np.float32(127.5) and b[0] == np.float32(127.5)
    s, b = denormalize_scale_bias((0.25,), (2.0,), max_value=1.0)
    assert s[0] == np.float32(2.0) and b[0] == np.float32(0.25)


@pytest.mark.parametrize("dtype_name,config,mismatches", [
    ("float32", "unit", 0), ("float32", "pm1", 0), ("float32", "imagenet", 0), ("float32", "clip", 0),
    ("float16", "unit", 0), ("float16", "pm1", 0), ("float16", "imagenet", 0), ("float16", "clip", 0),
    ("bfloat16", "unit", 0), ("bfloat16", "pm1", 0), ("bfloat16", "imagenet", 0), ("bfloat16", "clip", 1),
])
def test_round_trip_model_exhaustive(dtype_name, config, mismatches):
    """decode with normalize_scale_bias, encode with denormalize_scale_bias: every byte comes back, except one value of 768 for
    bfloat16 under CLIP's mean and std (bfloat16 keeps 8 significant bits)"""
    import torch
    mean, std = {"unit": UNIT, "pm1": PM1, "imagenet": IMAGENET, "clip": CLIP}[config]
    got = round_trip(getattr(torch, dtype_name), mean, std)
    want = torch.arange(256, dtype=torch.uint8)[:, None].expand(256, 3)
    assert int((got != want).sum()) == mismatches


def test_quantisation_rule():
    import torch
    vals = [0.5, 1.5, 2.5, 254.5, 255.5, -0.5, 1e30, -1e30, float("nan"), float("inf"), float("-inf"), 0.0, -0.0, 1e-45, -1e-45,
            0.49999997, 253.50002, 3.4e38]
    want = [0, 2, 2, 254, 255, 0, 255, 0, 0, 255, 0, 0, 0, 0, 0, 0, 254, 255]
    x = torch.tensor(vals, dtype=torch.float32)[:, None]
    assert quantize(x, [1.0], [0.0])[:, 0].tolist() == want
    # half-to-even on every tie of the range, never torchvision's add-0.5-and-truncate
    ties = torch.arange(256, dtype=torch.float32)[:, None] + 0.5
    assert quantize(ties, [1.0], [0.0])[:, 0].tolist() == [min(255, k + (k & 1)) for k in range(256)]
    # float16: the multiply runs in float32, so a product past float16's range still saturates instead of overflowing to inf first
    h = torch.tensor([65504.0, -65504.0, 60000.0, 0.0], dtype=torch.float16)[:, None]
    assert quantize(h, [2.0], [0.0])[:, 0].tolist() == [255, 0, 255, 0]
    # subnormal float16 / bfloat16 inputs are exact in float32
    sub = torch.tensor([2.0 ** -24, -(2.0 ** -24)], dtype=torch.float16)[:, None]
    assert quantize(sub, [2.0 ** 24 * 3.0], [0.0])[:, 0].tolist() == [3, 0]
    bsub = torch.tensor([2.0 ** -130], dtype=torch.bfloat16)[:, None]
    assert quantize(bsub, [2.0 ** 127], [1.4])[:, 0].tolist() == [2]                  # 1.4 + 0.125, not 1.4 (flushed to zero)
    # the multiply and the add round separately: x * s + b here differs from a fused multiply-add
    x = torch.tensor([[1.0 + 2.0 ** -23]], dtype=torch.float32)
    s, b = np.float32(1.0 + 2.0 ** -23), np.float32(-1.0)
    fused = float(np.float64(x.item()) * np.float64(s) + np.float64(b))
    assert (x * torch.tensor([s]) + torch.tensor([b])).item() != fused


def test_python_argument_rules():
    import torch
    from fpng_b200 import encode_batch_device, encode_ragged_device, typed_layout
    u8 = torch.zeros(1, 4, 4, 3, dtype=torch.uint8)
    with pytest.raises(ValueError):
        encode_batch_device(u8, scale=2.0)
    with pytest.raises(ValueError):
        encode_batch_device(u8, bias=[0.0, 1.0, 2.0])
    for dt in (torch.int32, torch.int16, torch.float64, torch.bool):
        with pytest.raises(ValueError):
            encode_batch_device(torch.zeros(1, 4, 4, 3, dtype=dt))
    with pytest.raises(ValueError):
        encode_batch_device(torch.zeros(1, 4, 4, 3), scale=[1.0, 2.0])                    # neither one value nor one per channel
    with pytest.raises(ValueError):
        encode_ragged_device([torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(4, 4, 3)])
    with pytest.raises(ValueError):
        encode_ragged_device([torch.zeros(4, 4, 3, dtype=torch.float16), torch.zeros(4, 4, 3, dtype=torch.bfloat16)])
    # byte strides of float views: NCHW, a pitched crop, HCW, a broadcast
    for dtype, es in ((torch.float32, 4), (torch.float16, 2), (torch.bfloat16, 2)):
        n, c, h, w = 2, 3, 5, 7
        nchw = torch.empty(n, c, h, w, dtype=dtype).permute(0, 2, 3, 1)
        assert typed_layout(nchw.shape, nchw.stride(), es) == (c * h * w * es, w * es, es, h * w * es)
        crop = torch.empty(n, h + 2, w + 3, c, dtype=dtype)[:, 1:1 + h, 2:2 + w]
        assert typed_layout(crop.shape, crop.stride(), es) == ((h + 2) * (w + 3) * c * es, (w + 3) * c * es, c * es, es)
        hcw = torch.empty(n, h, c, w, dtype=dtype).permute(0, 1, 3, 2)
        assert typed_layout(hcw.shape, hcw.stride(), es) == (h * c * w * es, c * w * es, es, w * es)
        bc = torch.empty(1, h, w, c, dtype=dtype).expand(n, -1, -1, -1)
        assert typed_layout(bc.shape, bc.stride(), es) == (0, w * c * es, c * es, es)
        with pytest.raises(ValueError):
            rgb_of_rgba = torch.empty(n, h, w, 4, dtype=dtype)[..., :3]
            typed_layout(rgb_of_rgba.shape, rgb_of_rgba.stride(), es)
