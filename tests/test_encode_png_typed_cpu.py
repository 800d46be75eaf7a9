"""CPU tests of the typed PNG encode's quantisation rule at 16 bits (include/fpng_b200.h, fpngb_encode_png_ragged_device_typed), of
the exhaustive native-decode -> encode round trip of every 16-bit sample, and of the Python argument rules that need no device."""
import numpy as np
import pytest


def quantize(x, scale, bias, depth):
    """the typed PNG encode's rule in torch: x [..., c] of any float dtype -> uint8 (depth 8) or uint16 (depth 16)"""
    import torch
    s = torch.as_tensor(np.asarray(scale, np.float32))
    b = torch.as_tensor(np.asarray(bias, np.float32))
    m = (1 << depth) - 1
    return torch.nan_to_num(x.float() * s + b, nan=0.0).round().clamp(0, m).to(torch.uint8 if depth == 8 else torch.uint16)


def q16(vals, dtype=None, scale=1.0, bias=0.0):
    import torch
    x = torch.tensor(vals, dtype=dtype or torch.float32)[:, None]
    return quantize(x, [scale], [bias], 16)[:, 0].to(torch.int64).tolist()


def test_rule_ties_half_to_even():
    import torch
    k = torch.arange(65536, dtype=torch.float64)
    ties = (k + 0.5).to(torch.float32)                       # every k + 0.5 is exact in float32 below 2^23
    got = quantize(ties[:, None], [1.0], [0.0], 16)[:, 0].to(torch.int64)
    want = torch.clamp(k.to(torch.int64) + (k.to(torch.int64) & 1), max=65535)
    assert torch.equal(got, want)
    assert q16([65534.5, 65535.5, 65536.5]) == [65534, 65535, 65535]


def test_rule_special_values():
    vals = [-0.5, -0.0, 0.0, float("nan"), float("inf"), float("-inf"), 1e30, -1e30, 3.4e38, 0.49999997, 65535.0, 65535.49]
    assert q16(vals) == [0, 0, 0, 0, 65535, 0, 65535, 0, 65535, 0, 65535, 65535]
    # a NaN produced by the arithmetic (inf * 0) becomes 0 as well
    assert q16([float("inf")], scale=0.0) == [0]


def test_rule_float16_saturates_in_fp32():
    import torch
    # 65504 * 2 overflows float16 but not the fp32 multiply, so it saturates to 65535 rather than going through inf
    assert q16([65504.0, -65504.0, 30000.0, 0.0], dtype=torch.float16, scale=2.0) == [65535, 0, 60000, 0]
    assert q16([65504.0], dtype=torch.float16, scale=2.0, bias=-70000.0) == [61008]


def test_rule_subnormals():
    import torch
    # subnormal float16 / bfloat16 inputs are exact in float32 and are not flushed to zero
    assert q16([2.0 ** -24, -(2.0 ** -24), 3 * 2.0 ** -24], dtype=torch.float16, scale=2.0 ** 24 * 1000.0) == [1000, 0, 3000]
    assert q16([2.0 ** -130], dtype=torch.bfloat16, scale=2.0 ** 127, bias=1.4) == [2]          # 1.4 + 0.125, not 1.4


def test_rule_multiply_and_add_round_separately():
    import torch
    # x * s rounds to a tie of the output grid that an FMA would not see: fl(x * s) = 2.5 exactly -> 2, the exact product
    # 2.5 + 2^-22 + 2^-46 would round to 3
    x = np.float32(1.0 + 2.0 ** -23)
    s = np.float32(2.5 - 2.0 ** -22)
    exact = float(np.float64(x) * np.float64(s))
    assert np.float32(x * s) == np.float32(2.5) and exact != 2.5
    assert q16([float(x)], scale=float(s)) == [2]
    # the same with the add: fl(fl(x * s) + b) against fma(x, s, b)
    b = np.float32(1000.0)
    fused = round(np.float64(x) * np.float64(s) + np.float64(b))
    got = q16([float(x)], scale=float(s), bias=float(b))[0]
    assert got == 1002 and fused == 1003


def decoded(k, dtype):
    """the native float decode of every 16-bit sample s with scale k (bias 0): T(fl(fl(s / 257) * k))"""
    import torch
    s = torch.arange(65536, dtype=torch.float32)
    return (s / torch.tensor(257.0) * torch.tensor(np.float32(k))).to(dtype)


# (decode scale k, encode scale): 16-bit values, depth in metres stored as millimetres, and the [0, 1] range
PAIRS = {"u16": (257.0, 1.0), "mm": (0.257, 1000.0), "unit": (257.0 / 65535.0, 65535.0)}


@pytest.mark.parametrize("pair,dtype_name,mismatches", [
    ("u16", "float32", 0), ("mm", "float32", 0), ("unit", "float32", 0),
    # float16 keeps 11 significant bits: 2049 samples up to 2048, 1024 per octave above (minus the shared 2048), and 65535,
    # which rounds to inf and saturates back, come back; bfloat16 keeps 8: 257 + 1023 and 65535.  The "mm" pair's products
    # land on slightly different float16 / bfloat16 values.
    ("u16", "float16", 58367), ("mm", "float16", 58390), ("unit", "float16", 58367),
    ("u16", "bfloat16", 64255), ("mm", "bfloat16", 64258), ("unit", "bfloat16", 64255),
])
def test_round_trip_exhaustive(pair, dtype_name, mismatches):
    """decode every 16-bit sample natively into a float with scale k, encode with the inverse scale at depth 16: lossless in
    float32 only"""
    import torch
    k, sc = PAIRS[pair]
    got = quantize(decoded(k, getattr(torch, dtype_name))[:, None], [sc], [0.0], 16)[:, 0].to(torch.int64)
    assert int((got != torch.arange(65536)).sum()) == mismatches


def test_depth8_is_the_typed_encode_rule():
    """at depth 8 the rule is the fpng typed encode's (tests/test_encode_typed_cpu.py), bit for bit"""
    import torch
    x = torch.tensor([0.5, 1.5, 254.5, 255.5, -0.5, float("nan"), float("inf"), 1e30, 2.0 ** -149], dtype=torch.float32)[:, None]
    want = torch.nan_to_num(x * 1.0 + 0.0, nan=0.0).round().clamp(0, 255).to(torch.uint8)
    assert torch.equal(quantize(x, [1.0], [0.0], 8), want)
    assert quantize(x, [1.0], [0.0], 8)[:, 0].tolist() == [0, 2, 254, 255, 0, 0, 255, 255, 0]


def test_python_argument_rules():
    """checked before anything touches the device, so CPU tensors are enough"""
    import torch
    from fpng_b200 import encode_png_device
    f32 = torch.zeros((4, 4, 1), dtype=torch.float32)
    u8 = torch.zeros((4, 4, 1), dtype=torch.uint8)
    u16 = torch.zeros((4, 4, 3), dtype=torch.uint16)
    bad = [
        dict(images=[f32]),                                                   # a float list needs a depth
        dict(images=[f32], depth=12),
        dict(images=[f32, f32], depth=[8]),                                  # one depth per image
        dict(images=[f32, f32], depth=[8, 16, 16]),
        dict(images=[f32], depth=[32]),
        dict(images=[f32, u8], depth=8),                                     # float mixed with uint
        dict(images=[u16, f32], depth=16),
        dict(images=[f32, torch.zeros((4, 4, 1), dtype=torch.float16)], depth=16),   # two float dtypes
        dict(images=[torch.zeros((4, 4, 1), dtype=torch.bfloat16), torch.zeros((4, 4, 1), dtype=torch.float16)], depth=8),
        dict(images=[u8], depth=8),                                          # uint lists take no depth, scale or bias
        dict(images=[u16], scale=2.0),
        dict(images=[u8, u16], bias=1.0),
        dict(images=[torch.zeros((4, 4, 1), dtype=torch.int32)]),
        dict(images=[torch.zeros((4, 4, 1), dtype=torch.float64)], depth=16),
        dict(images=[torch.zeros((4, 4, 3))], depth=8, scale=[1.0, 2.0]),   # neither one value nor one per channel
        dict(images=[torch.zeros((4, 4, 1)), torch.zeros((4, 4, 2))], depth=16, bias=[1.0, 2.0, 3.0]),
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            encode_png_device(**kw)
