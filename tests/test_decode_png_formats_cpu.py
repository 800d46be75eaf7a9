"""CPU tests of the all-formats walk (FPNGB_PNG_ALL_FORMATS, fpngb_get_png_info_ex): one status per walk rule, the inflated-size
formula against the test writer, flag-off statuses, the Python argument rules, and the numpy pixel model of
tests/pngwrite_formats.py pinned against PIL, torchvision's decode_png (libpng) and, where oracle/_ref is built, lodepng and wuffs."""
import ctypes as C
import io
import struct
import zlib

import numpy as np
import pytest

import pngwrite_formats as pf
from pngwrite import IEND, SIG, chunk, ihdr

OK, CHUNK_PARSING, INVALID_IDAT, UNSUPPORTED = 0, 7, 8, 104


@pytest.fixture(scope="module")
def fb():
    import fpng_b200
    return fpng_b200


def z(n=64):
    return chunk(b"IDAT", zlib.compress(b"\0" * n))


def png(ctype, depth=8, interlace=0, pre=(), post=()):
    return SIG + ihdr(8, 8, depth, ctype, interlace=interlace) + b"".join(pre) + z() + b"".join(post) + IEND


PLTE4 = chunk(b"PLTE", bytes(range(12)))
TRNS2, TRNS6 = chunk(b"tRNS", b"\0\1"), chunk(b"tRNS", b"\0\1\0\2\0\3")


def walk_cases():
    c = []
    for ctype, depths in pf.DEPTHS.items():
        for d in depths:
            for il in (0, 1):
                c.append((f"ok_{ctype}_{d}_{il}", png(ctype, d, il, [PLTE4] if ctype == 3 else []), OK))
    for ctype, d in [(0, 3), (0, 32), (2, 4), (3, 16), (4, 4), (6, 1), (1, 8), (5, 8), (7, 8)]:
        c.append((f"bad_ihdr_{ctype}_{d}", png(ctype, d), UNSUPPORTED))
    c.append(("interlace_2", png(2, 8, 2), UNSUPPORTED))
    c.append(("compression_1", SIG + ihdr(8, 8, 8, 2, comp=1) + z() + IEND, UNSUPPORTED))
    c.append(("filter_method_1", SIG + ihdr(8, 8, 8, 2, filt=1) + z() + IEND, UNSUPPORTED))
    c.append(("plte_missing", png(3), CHUNK_PARSING))
    c.append(("plte_empty", png(3, pre=[chunk(b"PLTE", b"")]), CHUNK_PARSING))
    c.append(("plte_len_not_3n", png(3, pre=[chunk(b"PLTE", b"\0" * 7)]), CHUNK_PARSING))
    c.append(("plte_too_long", png(3, pre=[chunk(b"PLTE", b"\0" * 771)]), CHUNK_PARSING))
    c.append(("plte_768", png(3, pre=[chunk(b"PLTE", b"\0" * 768)]), OK))
    c.append(("plte_second", png(3, pre=[PLTE4, PLTE4]), CHUNK_PARSING))
    c.append(("plte_after_idat", png(3, post=[PLTE4]), CHUNK_PARSING))
    c.append(("plte_in_gray", png(0, pre=[PLTE4]), UNSUPPORTED))
    c.append(("plte_in_gray_alpha", png(4, pre=[PLTE4]), UNSUPPORTED))
    c.append(("plte_in_rgb_ignored", png(2, pre=[PLTE4]), OK))
    c.append(("plte_in_rgba_ignored", png(6, 16, pre=[PLTE4]), OK))
    c.append(("trns_gray", png(0, pre=[TRNS2]), OK))
    c.append(("trns_gray_len", png(0, pre=[TRNS6]), CHUNK_PARSING))
    c.append(("trns_rgb", png(2, pre=[TRNS6]), OK))
    c.append(("trns_rgb_len", png(2, pre=[TRNS2]), CHUNK_PARSING))
    c.append(("trns_second", png(0, pre=[TRNS2, TRNS2]), CHUNK_PARSING))
    c.append(("trns_after_idat", png(2, post=[TRNS6]), CHUNK_PARSING))
    c.append(("trns_palette", png(3, pre=[PLTE4, chunk(b"tRNS", b"\1\2\3\4")]), OK))
    c.append(("trns_palette_empty", png(3, pre=[PLTE4, chunk(b"tRNS", b"")]), OK))
    c.append(("trns_palette_long", png(3, pre=[PLTE4, chunk(b"tRNS", b"\1" * 5)]), CHUNK_PARSING))
    c.append(("trns_before_plte", png(3, pre=[chunk(b"tRNS", b"\1"), PLTE4]), CHUNK_PARSING))
    c.append(("trns_gray_alpha_ignored", png(4, pre=[chunk(b"tRNS", b"\1\2\3")]), OK))
    c.append(("trns_rgba_ignored", png(6, pre=[chunk(b"tRNS", b"")]), OK))
    c.append(("unknown_critical", png(2, pre=[chunk(b"ABCD", b"")]), UNSUPPORTED))
    c.append(("second_ihdr", png(0, 16, pre=[ihdr(8, 8)]), UNSUPPORTED))
    c.append(("no_idat", SIG + ihdr(8, 8, 16, 0) + chunk(b"tEXt", b"k\0" + b"v" * 32) + IEND, INVALID_IDAT))
    c.append(("idat_run_broken", SIG + ihdr(8, 8, 1, 0) + z() + chunk(b"tEXt", b"a\0b") + z() + IEND, CHUNK_PARSING))
    return c


@pytest.mark.parametrize("name,data,want", walk_cases(), ids=[c[0] for c in walk_cases()])
def test_walk_rules(fb, name, data, want):
    st = fb.get_png_info(data, all_formats=True)
    assert st[0] == want, (name, st)
    if want == OK:
        assert st[1:3] == (8, 8)


@pytest.mark.parametrize("ctype,trns,want", [(0, None, 1), (0, TRNS2, 2), (4, None, 2), (2, None, 3), (2, TRNS6, 4), (6, None, 4),
                                             (3, None, 3), (3, chunk(b"tRNS", b"\1"), 4)])
def test_info_chans(fb, ctype, trns, want):
    pre = ([PLTE4] if ctype == 3 else []) + ([trns] if trns else [])
    data = png(ctype, 8 if ctype != 0 else 2, 1, pre)
    st = fb.get_png_info(data, all_formats=True)
    assert st[0] == 0 and st[3] == want
    assert st[4] == len(SIG) + 25 + sum(len(p) for p in pre) and st[5] == len(z()) - 12


def test_raw_len_formula(fb):
    f = fb._lib.lib().fpngb_debug_png_raw_len
    for bits in (1, 2, 4, 8, 16, 24, 32, 48, 64):
        for w in range(1, 18):
            for h in range(1, 18):
                for il in (0, 1):
                    assert f(w, h, bits, il) == pf.raw_len(w, h, bits, il), (w, h, bits, il)
    assert f(1 << 15, 1 << 15, 64, 0) == (1 << 15) * (1 + 8 * (1 << 15)) > 1 << 32   # 64 bits: 16-bit RGBA at 2^30 pixels
    assert f(1 << 15, 1 << 15, 64, 1) > 1 << 33


def test_raw_len_matches_writer():
    rs = np.random.RandomState(3)
    for ctype, depth, il, t in pf.combos():
        for (w, h) in [(1, 1), (3, 5), (9, 2), (17, 17)]:
            s = pf.random_samples(rs, w, h, ctype, depth, 4)
            raw = pf.raw_stream(s, ctype, depth, il)
            assert len(raw) == pf.raw_len(w, h, depth * pf.SAMPLES[ctype], il)


def corpus():
    rs = np.random.RandomState(11)
    out = []
    for k, (ctype, depth, il, t) in enumerate(pf.combos()):
        for (w, h) in [(1, 1), (5, 3), (13, 17), (33, 9)]:
            out.append((ctype, depth, il, t) + pf.case(rs, w, h, ctype, depth, il, t, seed=k))
    return out


def test_flag_off_statuses(fb):
    for ctype, depth, il, t, data, s, plte, trns in corpus():
        ext = depth != 8 or il or ctype == 3 or t
        off = fb.get_png_info(data)
        assert off[0] == (UNSUPPORTED if ext else OK), (ctype, depth, il, t, off)
        assert fb.get_png_info(data, all_formats=False) == off
        on = fb.get_png_info(data, all_formats=True)
        assert on[0] == OK and on[1:3] == (s.shape[1], s.shape[0]) and on[3] == pf.info_chans(ctype, trns)
        if not ext:
            assert on == off


def test_unknown_flag_bits(fb):
    L = fb._lib.lib()
    data = np.frombuffer(png(2), np.uint8)
    v = [C.c_uint32() for _ in range(5)]
    for flags in (2, 4, 0x80000000):
        assert L.fpngb_get_png_info_ex(data.ctypes.data_as(C.c_void_p), data.size, flags, *[C.byref(x) for x in v]) == 2


def test_python_argument_rules(fb):
    import torch
    data = torch.zeros(64, dtype=torch.uint8)
    offs = torch.zeros(1, dtype=torch.int64)
    sizes = torch.ones(1, dtype=torch.int32)
    with pytest.raises(ValueError, match="any_png"):
        fb.get_info_batch_device(data, offs, sizes, all_formats=True)
    with pytest.raises(ValueError, match="any_png"):
        fb.decode_packed_ragged_device(data, offs, sizes, 3, all_formats=True)
    with pytest.raises(ValueError, match="any_png"):
        fb.decode_packed_resized_device(data, offs, sizes, (4, 4), 3, all_formats=True)
    assert fb.FPNGB_PNG_ALL_FORMATS == 1 and fb.FPNGB_RESIZE_ALL_PNG_FORMATS == 8


# ---- the model against other decoders ---------------------------------------------------------------------------------------------
def test_model_against_pil():
    from PIL import Image
    for ctype, depth, il, t, data, s, plte, trns in corpus():
        im = Image.open(io.BytesIO(data))
        want = pf.model_u8(s, ctype, depth, 4, plte, trns)
        if ctype == 0 and depth == 16:                       # I;16: the full samples
            np.testing.assert_array_equal(np.array(im).astype(np.int64), pf.model16(s, ctype, depth)[..., 0])
            continue
        got = np.array(im.convert("RGBA"))
        np.testing.assert_array_equal(got[..., :3], want[..., :3], err_msg=str((ctype, depth, il, t)))
        if depth == 8 or ctype == 3 or (depth < 8 and trns is None):   # PIL's key compare works on 8-bit values
            np.testing.assert_array_equal(got[..., 3], want[..., 3], err_msg=str((ctype, depth, il, t)))


def test_model_pil_writers():
    """files PIL writes (palette at 1/2/4/8 bits with transparency, mode 1, I;16) decode in the model to what PIL reads back"""
    from PIL import Image
    rs = np.random.RandomState(5)
    for bits in (1, 2, 4, 8):
        idx = rs.randint(0, 1 << bits, (7, 13)).astype(np.uint8)
        im = Image.fromarray(idx, "P")
        im.putpalette(rs.randint(0, 256, 3 * (1 << bits)).astype(np.uint8).tobytes())
        for tr in (None, bytes(rs.randint(0, 256, 1 << bits).astype(np.uint8))):
            b = io.BytesIO()
            im.save(b, "PNG", bits=bits, **({} if tr is None else {"transparency": tr}))
            f = pf.parse(b.getvalue())
            want = pf.model_u8(f["samples"], f["ctype"], f["depth"], 4, f["plte"], f["trns"])
            np.testing.assert_array_equal(np.array(Image.open(io.BytesIO(b.getvalue())).convert("RGBA")), want)
    for mode, arr in [("1", rs.randint(0, 2, (9, 11)).astype(bool)), ("I;16", rs.randint(0, 65536, (9, 11)).astype(np.uint16))]:
        b = io.BytesIO()
        (Image.fromarray(arr.astype(np.uint8) * 255).convert("1") if mode == "1" else Image.fromarray(arr)).save(b, "PNG")
        f = pf.parse(b.getvalue())
        want = pf.model16(f["samples"], f["ctype"], f["depth"])[..., 0]
        np.testing.assert_array_equal(want, arr.astype(np.int64) * 65535 if mode == "1" else arr.astype(np.int64))


def test_model_against_libpng():
    """torchvision's decode_png in RGB mode (libpng's expand, palette lookup and de-interlacing; 16-bit files as uint16); the
    alpha channel is pinned by PIL and lodepng"""
    import torch
    from torchvision.io import ImageReadMode, decode_png
    for ctype, depth, il, t, data, s, plte, trns in corpus():
        got = decode_png(torch.frombuffer(bytearray(data), dtype=torch.uint8), ImageReadMode.RGB).permute(1, 2, 0)
        if got.dtype == torch.uint16:
            np.testing.assert_array_equal(got.numpy().astype(np.int64), pf.model16(s, ctype, depth, plte, trns)[..., :3],
                                          err_msg=str((ctype, depth, il, t)))
        else:
            np.testing.assert_array_equal(got.numpy(), pf.model_u8(s, ctype, depth, 3, plte, trns), err_msg=str((ctype, depth, il, t)))


def test_model_against_lodepng_and_wuffs():
    from oracle.pyoracle import Ref, Verifiers
    if not Ref.available() and not Verifiers.available():
        pytest.skip("oracle/_ref is not built")
    ref = Ref() if Ref.available() else None
    ver = Verifiers() if Verifiers.available() else None
    for ctype, depth, il, t, data, s, plte, trns in corpus():
        h, w = s.shape[:2]
        want = pf.model_u8(s, ctype, depth, 4, plte, trns).reshape(-1)
        if ref is not None:
            err, px, ww, hh = ref.lodepng_decode(data, 4)
            assert err == 0 and (ww, hh) == (w, h)
            np.testing.assert_array_equal(px, want, err_msg=str(("lodepng", ctype, depth, il, t)))
        if ver is not None:
            rc, px, ww, hh = ver.wuffs_decode_rgba(data, w, h)
            assert rc == 0 and (ww, hh) == (w, h)
            if not (trns is not None and ctype in (0, 2)) and (ctype, depth) != (0, 16):   # wuffs ignores color keys and differs
                # on 16-bit gray; lodepng, PIL and libpng pin those
                np.testing.assert_array_equal(px, want, err_msg=str(("wuffs", ctype, depth, il, t)))


def test_typed_rule_recovers_16_bits():
    s = np.arange(65536, dtype=np.int64)
    v = s.astype(np.float32) / np.float32(257.0)
    assert np.array_equal(np.round(v * np.float32(257.0)).astype(np.int64), s)
    k = np.arange(256)
    assert np.array_equal((k * 257).astype(np.float32) / np.float32(257.0), k.astype(np.float32))
