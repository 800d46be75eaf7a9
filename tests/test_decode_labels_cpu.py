"""CPU tests of the label-map decode (include/fpng_b200.h, "label maps"): the numpy models of the nearest and nearest-exact resize
rules against torch's F.interpolate on the CPU, the index rule (each pixel's raw sample) against PIL on the committed PIL-written
fixtures, and the Python argument rules that fail before any device call.  tests/test_decode_labels_gpu.py checks the decoder
against these models."""
import io
import os
import re

import numpy as np
import pytest

import pngwrite_formats as pf

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMATS = os.path.join(ROOT, "tests", "golden", "anypng_formats")
ANYPNG = os.path.join(ROOT, "tests", "golden", "anypng")


def nearest_src(n_in, n_out, exact):
    """source index of every output index along one axis: the header's rule, each float32 operation rounded on its own"""
    scale = F32(n_in) / F32(n_out)
    i = np.arange(n_out, dtype=F32)
    x = i + F32(0.5) if exact else i
    return np.minimum(np.floor(x * scale).astype(np.int64), n_in - 1)


def nearest_model(px, out_h, out_w, exact, box=None):
    """px [h, w, ...] cropped to box (top, left, height, width) and resized by nearest neighbour to out_h x out_w"""
    if box is not None:
        top, left, bh, bw = (int(v) for v in box)
        px = px[top:top + bh, left:left + bw]
    return px[nearest_src(px.shape[0], out_h, exact)][:, nearest_src(px.shape[1], out_w, exact)]


def index_model(data: bytes) -> np.ndarray:
    """[h, w] raw samples of a palette or gray PNG: the index decode's pixel rule"""
    return pf.parse(data)["samples"][..., 0].astype(np.int64)


# ---- the nearest rules against torch ------------------------------------------------------------------------------------------------
def axis_pairs():
    pairs = [(n, n) for n in (1, 2, 3, 7, 100)]                                     # identity
    pairs += [(n, 2 * n) for n in (1, 2, 3, 5, 37, 250)] + [(2 * n, n) for n in (1, 2, 3, 5, 37, 250)]   # 2x up and down
    pairs += [(a, b) for a in (1, 2) for b in (1, 2, 3, 17)] + [(a, b) for a in (3, 17) for b in (1, 2)]     # lengths 1 and 2
    pairs += [(a, b) for a in (7, 13, 101, 499) for b in (11, 97, 331)]             # primes
    rs = np.random.RandomState(11)
    pairs += [(int(rs.randint(1, 5000)), int(rs.randint(1, 5000))) for _ in range(200)]
    return pairs


@pytest.mark.parametrize("mode", ["nearest", "nearest-exact"])
def test_nearest_model_matches_torch_cpu(mode):
    import torch
    import torch.nn.functional as F
    exact = mode == "nearest-exact"
    for n_in, n_out in axis_pairs():
        x = torch.arange(n_in, dtype=torch.int64).remainder(251).to(torch.uint8)
        # along each axis separately: a 1-row and a 1-column image
        got_w = F.interpolate(x.view(1, 1, 1, n_in), size=(1, n_out), mode=mode).view(-1).numpy()
        got_h = F.interpolate(x.view(1, 1, n_in, 1), size=(n_out, 1), mode=mode).view(-1).numpy()
        want = x.numpy()[nearest_src(n_in, n_out, exact)]
        assert np.array_equal(got_w, want) and np.array_equal(got_h, want), (mode, n_in, n_out)
    rs = np.random.RandomState(3)
    for _ in range(20):                                                             # both axes at once, with channels
        h, w, oh, ow, c = (int(v) for v in rs.randint(1, 90, 5) % np.array([90, 90, 90, 90, 4]) + 1)
        img = rs.randint(0, 256, (h, w, c)).astype(np.uint8)
        got = F.interpolate(torch.from_numpy(img).permute(2, 0, 1)[None], size=(oh, ow), mode=mode)[0].permute(1, 2, 0).numpy()
        assert np.array_equal(got, nearest_model(img, oh, ow, exact)), (mode, h, w, oh, ow, c)


def test_nearest_model_identity_and_crop():
    rs = np.random.RandomState(4)
    img = rs.randint(0, 65536, (23, 31)).astype(np.uint16)
    for exact in (False, True):
        assert np.array_equal(nearest_model(img, 23, 31, exact), img)
        assert np.array_equal(nearest_model(img, 5, 7, exact, (3, 4, 5, 7)), img[3:8, 4:11])
        assert nearest_model(img, 1, 1, exact, (2, 3, 4, 4)).shape == (1, 1)


# ---- the index rule against PIL -----------------------------------------------------------------------------------------------------
def golden_label_files():
    names = sorted(f for f in os.listdir(FORMATS) if f.startswith("pil_p") or f == "pil_mode1.png")
    out = [os.path.join(FORMATS, f) for f in names]
    out += [os.path.join(ANYPNG, f) for f in ("pil_L_g0.png", "pil_L_g1.png")]
    return out


def test_index_model_matches_pil_on_golden_files():
    from PIL import Image
    files = golden_label_files()
    assert len(files) == 11
    for path in files:
        data = open(path, "rb").read()
        im = Image.open(io.BytesIO(data))
        assert im.mode in ("P", "1", "L"), (path, im.mode)
        want = np.asarray(im).astype(np.int64)                                       # mode "1": the bool array as 0 / 1
        assert np.array_equal(index_model(data), want), path


def test_index_model_sub_byte_gray_is_unscaled():
    """2- and 4-bit gray: PIL scales the samples to 0..255, the index rule keeps them"""
    rs = np.random.RandomState(6)
    for depth in (1, 2, 4):
        png, s, _, _ = pf.case(rs, 13, 7, 0, depth, 0, False)
        got = index_model(png)
        assert got.max() <= (1 << depth) - 1 and np.array_equal(got, s[..., 0])


# ---- Python argument rules (no device call) -------------------------------------------------------------------------------------------
def test_python_argument_rules():
    import torch
    import fpng_b200 as fb
    ragged = fb.decode_packed_ragged_device
    full = dict(any_png=True, all_formats=True, native=True)
    for kw in (dict(any_png=True, all_formats=True), dict(any_png=True, native=True), dict(all_formats=True, native=True)):
        with pytest.raises(ValueError):
            ragged(None, None, None, 1, indices=True, **kw)
    for d in (0, None, 2, 3, 4):
        with pytest.raises(ValueError, match="desired_channels"):
            ragged(None, None, None, d, indices=True, **full)
    for dt in (torch.float32, torch.float16, torch.bfloat16, torch.int32):
        with pytest.raises(ValueError, match="uint8 or torch.uint16"):
            ragged(None, None, None, 1, indices=True, dtype=dt, **full)
    resized = fb.decode_packed_resized_device
    with pytest.raises(ValueError, match="interpolation"):
        resized(None, None, None, (4, 4), 3, interpolation="bicubic")
    with pytest.raises(ValueError, match="nearest"):
        resized(None, None, None, (4, 4), 1, indices=True, **full)                  # bilinear on ids
    for kw in (dict(any_png=True, all_formats=True), dict(any_png=True, native=True)):
        with pytest.raises(ValueError):
            resized(None, None, None, (4, 4), 1, interpolation="nearest", indices=True, **kw)
    with pytest.raises(ValueError, match="desired_channels"):
        resized(None, None, None, (4, 4), 2, interpolation="nearest", indices=True, **full)
    for dt in (torch.float32, torch.bfloat16):
        with pytest.raises(ValueError, match="uint8 or torch.uint16"):
            resized(None, None, None, (4, 4), 1, interpolation="nearest-exact", indices=True, dtype=dt, **full)


def test_constants_keep_unknown_bits_unknown():
    import fpng_b200 as fb
    header = open(os.path.join(ROOT, "include", "fpng_b200.h")).read()
    values = {k: int(v) for k, v in re.findall(r"(FPNGB_[A-Z0-9_]+) = (\d+)", header)}
    for name in ("FPNGB_PNG_INDEX", "FPNGB_RESIZE_NEAREST", "FPNGB_RESIZE_NEAREST_EXACT", "FPNGB_RESIZE_INDEX", "FPNGB_DECODE_NOT_INDEXED"):
        assert getattr(fb, name) == values[name], name
    png_bits = [fb.FPNGB_PNG_ALL_FORMATS, fb.FPNGB_PNG_NATIVE, fb.FPNGB_PNG_INDEX]
    assert fb.FPNGB_PNG_INDEX & (2 | 0x100) == 0 and len(set(png_bits)) == 3 and all(b & (b - 1) == 0 for b in png_bits)
    resize_bits = [fb.FPNGB_RESIZE_ANTIALIAS, fb.FPNGB_RESIZE_ANY_PNG, fb.FPNGB_RESIZE_ALL_PNG_FORMATS, fb.FPNGB_RESIZE_NATIVE,
                   fb.FPNGB_RESIZE_NEAREST, fb.FPNGB_RESIZE_NEAREST_EXACT, fb.FPNGB_RESIZE_INDEX]
    assert all(b & (b - 1) == 0 and b & 2 == 0 for b in resize_bits) and len(set(resize_bits)) == len(resize_bits)
    statuses = [fb.FPNGB_DECODE_SHAPE_MISMATCH, fb.FPNGB_DECODE_OUT_OF_SPACE, fb.FPNGB_DECODE_ADLER_MISMATCH, fb.FPNGB_DECODE_BAD_CROP,
                fb.FPNGB_DECODE_UNSUPPORTED_PNG, fb.FPNGB_DECODE_NOT_INDEXED]
    assert len(set(statuses)) == len(statuses)
