"""encode_png_device(reduce=True) on the GPU at the edges of its analysis and conversion kernels (tests/reduce_edges.py): the
deciding pixel at the analysis partition's edges, the early stop, colour-set collisions and races, the rule's every branch,
conversion widths and layouts, and image boundaries inside one call.  Every file is checked three ways: byte for byte against the
existing call on the model-reduced input (tests/reduce_model.py), read back exactly by an independent numpy + zlib reader
(tests/pngwrite_formats.py) in the format the rule picks, and with the guard bytes after the call's slots untouched."""
from __future__ import annotations

import numpy as np
import pytest

import pngwrite_formats as pf
import reduce_edges as ree
from reduce_model import choose
from test_encode_reduce_gpu import GUARD, dev, expected_file, reduce_encode

pytestmark = pytest.mark.gpu


def canon16(img):
    """[h, w, 4] RGBA in the 16-bit domain, as pngwrite_formats.model16 reads a file: 8-bit v as v * 257, gray replicated,
    missing alpha 0xFFFF"""
    a = np.asarray(img).astype(np.int64) * (257 if np.asarray(img).dtype == np.uint8 else 1)
    c = a.shape[2]
    rgb = np.repeat(a[..., :1], 3, -1) if c <= 2 else a[..., :3]
    al = a[..., c - 1:] if c in (2, 4) else np.full(a.shape[:2] + (1,), 0xFFFF, np.int64)
    return np.concatenate([rgb, al], -1)


def verify(gpu, img, f, flags=0):
    """(a) the existing call's file on the model-reduced input; (b) the independent reader gets img back, in choose's format"""
    img = np.asarray(img)
    assert f == expected_file(gpu, img, flags), choose(img)
    fmt, _, depth = choose(img)
    info = pf.parse(f)
    assert (info["ctype"], info["depth"]) == (ree.CTYPE[fmt], depth), (fmt, depth, info["ctype"], info["depth"])
    assert (info["w"], info["h"]) == (img.shape[1], img.shape[0])
    got = pf.model16(info["samples"], info["ctype"], info["depth"], info["plte"], info["trns"])
    assert np.array_equal(got, canon16(img)), (fmt, depth)


def run(gpu, imgs, flags=0):
    """one reduce call over imgs (numpy arrays or device tensors); every file verified, the guard after the slots untouched"""
    files, tail, _ = reduce_encode(gpu, [t if hasattr(t, "is_cuda") else dev(t) for t in imgs], flags)
    assert (tail == GUARD).all()
    for t, f in zip(imgs, files):
        verify(gpu, t.cpu().numpy() if hasattr(t, "is_cuda") else t, f, flags)
    return files


def run_pairs(gpu, cases):
    bases, seen = [], set()
    for c in cases:
        if id(c.base) not in seen:
            seen.add(id(c.base))
            bases.append(c.base)
    files = run(gpu, bases + [c.changed for c in cases])
    for c, f in zip(cases, files[len(bases):]):
        assert pf.parse(f)["ctype"] == ree.CTYPE[c.want_changed[0]], c.name


@pytest.mark.parametrize("prop", ["not_opaque", "not_gray", "not_rep8", "lattice", "colour_257"])
def test_deciding_pixel_at_partition_edges(gpu, prop):
    cases = [c for c in ree.edge_cases() if c.meta["prop"] == prop]
    assert cases
    run_pairs(gpu, cases)


def test_early_stop_never_skips_a_deciding_read(gpu):
    cases = ree.early_stop_cases()
    run_pairs(gpu, cases)
    for c in cases:                                                   # one image per call as well: no other image's CTAs around
        files, tail, _ = reduce_encode(gpu, [dev(c.changed)])
        assert (tail == GUARD).all() and pf.parse(files[0])["ctype"] == ree.CTYPE[c.want_changed[0]], c.name


def test_colour_set_edges(gpu):
    imgs = ree.colour_set_images()
    files = run(gpu, [img for _, img, _, _ in imgs])
    for (name, img, want, _), f in zip(imgs, files):
        info = pf.parse(f)
        assert (info["ctype"], info["depth"]) == (ree.CTYPE[want[0]], want[1]), name
    for name, img, want, _ in imgs:                                   # alone in its call
        run(gpu, [img])


def test_ctas_racing_on_the_same_colours(gpu):
    img = ree.racing_same_colours(1024)
    files = run(gpu, [img])
    info = pf.parse(files[0])
    assert (info["ctype"], info["depth"], len(info["plte"])) == (3, 8, 256)


@pytest.mark.parametrize("chans", [3, 4])
def test_16k_colours_fill_the_global_set(gpu, chans):
    img = ree.overflow_16k_colours(chans)
    files = run(gpu, [img])
    assert pf.parse(files[0])["ctype"] == (2 if chans == 3 else 6)


def test_rule_sweep_mixed_and_single(gpu):
    imgs = [img for _, img, _ in ree.sweep_images()]
    files = run(gpu, imgs)
    for img, f in zip(imgs, files):
        one, tail, _ = reduce_encode(gpu, [dev(img)])
        assert one[0] == f and (tail == GUARD).all()


def layouts(t, k):
    """t in one of five layouts, by k: contiguous, a row-pitched crop, CHW planes, stride-0 rows, an odd storage offset (8-bit)"""
    import torch
    h, w, c = t.shape
    k %= 5
    if k == 1:
        full = torch.zeros((h + 2, w + 3, c), dtype=t.dtype, device=t.device)
        full[1:1 + h, 2:2 + w] = t
        return full[1:1 + h, 2:2 + w]
    if k == 2:
        return t.permute(2, 0, 1).contiguous().permute(1, 2, 0)
    if k == 3:
        return t[:1].expand(h, -1, -1)
    if k == 4 and t.dtype == torch.uint8:
        buf = torch.zeros(t.numel() + 1, dtype=torch.uint8, device=t.device)
        buf[1:].copy_(t.reshape(-1))
        return buf[1:].view(h, w, c)
    return t


@pytest.mark.parametrize("mode", list(ree.conversion_modes()))
def test_conversion_widths_and_layouts(gpu, mode):
    want = ree.conversion_modes()[mode][3]
    plain = [ree.conversion_image(mode, w) for w in ree.CONV_WIDTHS]
    assert all(ree.fmt_of(a) == want for a in plain)
    run(gpu, plain)
    run(gpu, [layouts(dev(a), k) for k, a in enumerate(plain)])
    shaped = [ree.conversion_image(mode, w, h) for w, h, _ in ree.cta_shapes(mode)]
    run(gpu, shaped)
    run(gpu, [layouts(dev(a), k + 1) for k, a in enumerate(shaped)])


def test_image_boundaries_in_one_call(gpu):
    named = ree.boundary_images()
    single = {name: run(gpu, [img])[0] for name, img in named}
    n = len(named)
    for order in (list(range(n)), list(range(n))[::-1], [1, 0, 3, 2, 4], [4, 2, 0, 1, 3], [0, 0, 4, 4, 2, 1]):
        imgs = [named[i] for i in order]
        files, tail, _ = reduce_encode(gpu, [dev(img) for _, img in imgs])
        assert (tail == GUARD).all()
        for (name, _), f in zip(imgs, files):
            assert f == single[name], (order, name)
