"""CPU tests of the native-output rules of the any-PNG ragged decode (FPNGB_PNG_NATIVE, native=True): a numpy model of the rules in
include/fpng_b200.h, built on pngwrite_formats.model16 and pinned against Pillow's convert("L") / ("LA") for 8-bit files and against
OpenCV and torchvision for 16-bit files, the 32-bit luma bound, and the Python argument rules, which raise before any device work."""
import io

import numpy as np
import pytest

import pngwrite_formats as pf


def luma(r, g, b):
    return (19595 * np.asarray(r, np.int64) + 38470 * np.asarray(g, np.int64) + 7471 * np.asarray(b, np.int64) + 0x8000) >> 16


def native16(s, ctype, depth, desired, plte=None, trns=None):
    """[h, w, c] int64 output values in the 16-bit domain (8-bit values v as v * 257); desired 0: the info row's channels"""
    m = pf.model16(s, ctype, depth, plte, trns)
    d = desired or pf.info_chans(ctype, trns)
    if d >= 3:
        return m[..., :d]
    if depth == 16:
        lum = luma(m[..., 0], m[..., 1], m[..., 2])
    else:
        lum = luma(m[..., 0] >> 8, m[..., 1] >> 8, m[..., 2] >> 8) * 257
    return lum[..., None] if d == 1 else np.stack([lum, m[..., 3]], -1)


def native_out(m16, depth, dtype, scale=None, bias=None):
    """the stored elements: uint8 the high byte, uint16 the value, float T(x * scale + bias) with x = s / 257 or v"""
    if dtype == "uint8":
        return (m16 >> 8).astype(np.uint8)
    if dtype == "uint16":
        return m16.astype(np.uint16)
    x = m16.astype(np.float32) / np.float32(257.0) if depth == 16 else (m16 >> 8).astype(np.float32)
    if scale is not None:
        x = x * np.float32(scale) + np.float32(bias)
    return x.astype(dtype)


def fpng_native16(img, desired):
    """native model of an 8-bit RGB / RGBA image (fpng files): the 8-bit RGB / RGBA rule"""
    return native16(img.astype(np.uint32), 2 if img.shape[2] == 3 else 6, 8, desired)


# ---- the model against Pillow for 8-bit files -------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctype", [2, 6, 4, 3, 0])
@pytest.mark.parametrize("trns", [False, True])
def test_model_matches_pillow_l_la(ctype, trns):
    Image = pytest.importorskip("PIL.Image")
    if trns and ctype not in (0, 2, 3):
        pytest.skip("tRNS only in types 0 / 2 / 3")
    rs = np.random.RandomState(10 * ctype + trns)
    for k, (w, h) in enumerate([(1, 1), (7, 5), (33, 17), (64, 48)]):
        png, s, plte, tr = pf.case(rs, w, h, ctype, 8, 0, trns, seed=k, n_plte=200 if ctype == 3 else None)
        im = Image.open(io.BytesIO(png))
        im.load()
        want_l = np.asarray(im.convert("L"))[..., None].astype(np.int64) * 257
        assert np.array_equal(native16(s, ctype, 8, 1, plte, tr), want_l), (ctype, trns, w, h)
        if ctype in (2, 0) and trns:
            continue                     # Pillow's LA of a color-keyed file: its own keying rules; the model's alpha is checked below
        want_la = np.asarray(im.convert("LA")).astype(np.int64) * 257
        assert np.array_equal(native16(s, ctype, 8, 2, plte, tr), want_la), (ctype, trns, w, h)


def test_model_color_key_alpha():
    """desired 2 of a color-keyed file: (L, 0) on the key, (L, max) elsewhere; desired 0 of keyed gray is (Y, A)"""
    s = np.array([[[5], [9], [5]]], np.uint32)
    m = native16(s, 0, 8, 0, trns=pf.key_trns(0, 5))
    assert m.tolist() == [[[5 * 257, 0], [9 * 257, 65535], [5 * 257, 0]]]
    s16 = np.array([[[1000], [1001]]], np.uint32)
    assert native16(s16, 0, 16, 2, trns=pf.key_trns(0, 1001)).tolist() == [[[1000, 65535], [1001, 0]]]


@pytest.mark.parametrize("combo", pf.combos(), ids=lambda c: "t%d_d%d_i%d_%s" % (c[0], c[1], c[2], "trns" if c[3] else "plain"))
def test_model_shapes_and_domains(combo):
    """desired 0 gives the info row's channels; gray's luma is Y itself; every value stays in 0..65535; uint8 and float of the
    native model agree with the all-formats model at desired 3 / 4"""
    ctype, depth, il, t = combo
    rs = np.random.RandomState(ctype * 31 + depth)
    png, s, plte, trns = pf.case(rs, 9, 7, ctype, depth, il, t, seed=3)
    m0 = native16(s, ctype, depth, 0, plte, trns)
    assert m0.shape[2] == pf.info_chans(ctype, trns)
    for d in (1, 2, 3, 4):
        m = native16(s, ctype, depth, d, plte, trns)
        assert m.shape[2] == d and m.min() >= 0 and m.max() <= 0xFFFF
    if ctype in (0, 4):
        assert np.array_equal(native16(s, ctype, depth, 1, plte, trns)[..., 0], pf.model16(s, ctype, depth, plte, trns)[..., 0])
    for d in (3, 4):
        assert np.array_equal(native_out(native16(s, ctype, depth, d, plte, trns), depth, "uint8"), pf.model_u8(s, ctype, depth, d, plte, trns))
        assert np.array_equal(native_out(native16(s, ctype, depth, d, plte, trns), depth, "float32"),
                              pf.model_values(s, ctype, depth, d, plte, trns))


# ---- 16-bit files against OpenCV and torchvision -----------------------------------------------------------------------------------
def _cases16():
    rs = np.random.RandomState(16)
    out = []
    for ctype in (0, 4, 2, 6):
        for il in (0, 1):
            out.append((ctype,) + pf.case(rs, 23, 11, ctype, 16, il, False, seed=ctype + il))
    return out


def test_uint16_matches_opencv():
    cv2 = pytest.importorskip("cv2")
    for ctype, png, s, plte, trns in _cases16():
        got = cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)
        assert got.dtype == np.uint16
        got = got.reshape(got.shape[0], got.shape[1], -1)
        if got.shape[2] >= 3:
            got = got[..., [2, 1, 0] + ([3] if got.shape[2] == 4 else [])]       # BGR(A) -> RGB(A)
        want = native_out(native16(s, ctype, 16, 0, plte, trns), 16, "uint16")
        if ctype == 4:                   # OpenCV has no gray+alpha: it returns BGRA with gray replicated
            want = native_out(native16(s, ctype, 16, 4, plte, trns), 16, "uint16")
        assert np.array_equal(got, want), ctype


def test_uint16_matches_torchvision():
    torch = pytest.importorskip("torch")
    io_ = pytest.importorskip("torchvision.io")
    for ctype, png, s, plte, trns in _cases16():
        try:
            got = io_.decode_png(torch.frombuffer(bytearray(png), dtype=torch.uint8), io_.ImageReadMode.UNCHANGED)
        except RuntimeError as e:                                                   # a build without 16-bit PNG support
            pytest.skip(str(e))
        got = got.permute(1, 2, 0).numpy()
        want = native_out(native16(s, ctype, 16, 0, plte, trns), 16, "uint16")
        assert np.array_equal(got.astype(np.int64), want.astype(np.int64)), ctype


def test_luma_fits_in_32_bits():
    """the largest luma sum, at 16-bit white, stays below 2^32 and gives 65535; gray (R = G = B) gives itself in both domains"""
    top = 19595 * 65535 + 38470 * 65535 + 7471 * 65535 + 0x8000
    assert 19595 + 38470 + 7471 == 65536 and top < 1 << 32
    assert int(luma(65535, 65535, 65535)) == 65535
    v = np.arange(65536)
    assert np.array_equal(luma(v, v, v), v)


# ---- argument rules (raised before the device is touched) -------------------------------------------------------------------------
def _call(**kw):
    import torch
    import fpng_b200
    data = torch.zeros(16, dtype=torch.uint8)
    offsets = torch.zeros(1, dtype=torch.int64)
    sizes = torch.zeros(1, dtype=torch.int32)
    args = dict(desired_channels=3)
    args.update(kw)
    d = args.pop("desired_channels")
    return fpng_b200.decode_packed_ragged_device(data, offsets, sizes, d, **args)


@pytest.mark.parametrize("kw", [
    dict(native=True),                                                  # native without any_png
    dict(native=True, all_formats=True),
    dict(desired_channels=1, any_png=True),                             # 1 / 2 / 0 without native
    dict(desired_channels=2, any_png=True, all_formats=True),
    dict(desired_channels=0, any_png=True),
    dict(desired_channels=None, any_png=True),
    dict(dtype="uint16", any_png=True),                                 # uint16 without native
    dict(dtype="uint16", any_png=True, native=True, scale=2.0),         # uint16 takes no scale or bias
    dict(dtype="uint16", any_png=True, native=True, bias=1.0),
    dict(dtype="uint8", any_png=True, native=True, scale=2.0),
    dict(desired_channels=5, any_png=True, native=True),
], ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_python_argument_rules(kw):
    import torch
    if isinstance(kw.get("dtype"), str):
        kw = dict(kw, dtype=getattr(torch, kw["dtype"]))
    with pytest.raises(ValueError):
        _call(**kw)


def test_resized_call_keeps_its_channel_rule():
    import torch
    import fpng_b200
    data = torch.zeros(16, dtype=torch.uint8)
    for d in (0, 1, 2):
        with pytest.raises(ValueError):
            fpng_b200.decode_packed_resized_device(data, torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int32), (4, 4), d,
                                                   any_png=True)


@pytest.mark.parametrize("kw", [
    dict(desired_channels=1, native=True),                              # native without any_png
    dict(desired_channels=0, native=True, any_png=True),                # one batch shape: no desired 0
    dict(desired_channels=None, native=True, any_png=True),
    dict(desired_channels=3, dtype="uint16", any_png=True),             # uint16 without native
    dict(desired_channels=1, dtype="uint16", native=True, any_png=True, scale=2.0),
], ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_resized_native_argument_rules(kw):
    import torch
    import fpng_b200
    if isinstance(kw.get("dtype"), str):
        kw = dict(kw, dtype=getattr(torch, kw["dtype"]))
    d = kw.pop("desired_channels")
    with pytest.raises(ValueError):
        fpng_b200.decode_packed_resized_device(torch.zeros(16, dtype=torch.uint8), torch.zeros(1, dtype=torch.int64),
                                               torch.zeros(1, dtype=torch.int32), (4, 4), d, **kw)


def test_exports():
    import fpng_b200
    assert fpng_b200.FPNGB_PNG_NATIVE == 4 and fpng_b200.FPNGB_DTYPE_UINT16 == 4 and fpng_b200.FPNGB_RESIZE_NATIVE == 16
    assert fpng_b200.FPNGB_PNG_NATIVE & (fpng_b200.FPNGB_PNG_ALL_FORMATS | 2 | 0x100) == 0
