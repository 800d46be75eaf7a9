"""The colour-type reduction rule of encode_png_device(reduce=True), without a GPU: the numpy model (tests/reduce_model.py) on
hand-built images for every branch and tie, the slot bound against every candidate format's bound, and the Python argument
rules."""
from __future__ import annotations

import numpy as np
import pytest

from reduce_model import analyse, choose, hash_slot, palette_order, reduced_call


def gray(v, h=4, w=5, dtype=np.uint8):
    return np.full((h, w, 1), v, dtype=dtype)


def test_constant_zero_is_gray_1bit_not_palette():
    assert choose(gray(0)) == ("gray", 1, 1)                              # ties with a 1-entry palette: gray first


def test_constant_100_is_palette_1bit():
    assert choose(gray(100)) == ("palette", 1, 1)
    kind, ids, pal, depth = reduced_call(gray(100))
    assert kind == "labels" and depth == 1 and (ids == 0).all() and pal.tolist() == [[100, 100, 100, 255]]


def test_lattice_levels_against_off_lattice():
    on = np.arange(16, dtype=np.uint8).reshape(4, 4, 1) * 17              # the 4-bit lattice: gray 4-bit
    assert choose(on) == ("gray", 4, 4)
    off = on.copy()
    off[0, 0, 0] = 1                                                      # 16 levels, one off the lattice: palette 4-bit
    assert choose(off) == ("palette", 4, 4)
    assert choose(np.array([[[0], [85], [170], [255]]], np.uint8)) == ("gray", 2, 2)
    assert choose(np.array([[[0], [255]]], np.uint8)) == ("gray", 1, 1)
    rgb = np.repeat(on, 3, axis=2)                                        # gray-valued RGB takes the same branch
    assert choose(rgb) == ("gray", 4, 4)


def test_gray_with_varying_alpha_is_palette():
    a = np.zeros((4, 4, 2), np.uint8)
    a[..., 0] = 200
    a[..., 1] = np.arange(16).reshape(4, 4) * 16
    assert choose(a) == ("palette", 4, 4)
    k = np.arange(300)                                                    # 300 (gray, alpha) pairs: GA8
    a = np.stack([k % 256, k // 256 + 1], axis=1).astype(np.uint8).reshape(10, 30, 2)
    assert choose(a) == ("ga", 16, 8)


def test_256_against_257_colours():
    k = np.arange(256, dtype=np.uint32)
    img = np.stack([k, 255 - k, k // 2], axis=1).astype(np.uint8).reshape(16, 16, 3)
    assert choose(img) == ("palette", 8, 8)
    img2 = np.concatenate([img.reshape(256, 3), [[1, 2, 3]]]).astype(np.uint8).reshape(1, 257, 3)
    assert analyse(img2).colours is None and choose(img2) == ("rgb", 24, 8)


def test_uint16_one_sample_off_257():
    img = (np.arange(12, dtype=np.uint16).reshape(2, 2, 3) * 257)
    assert analyse(img).rep8 and choose(img) == ("palette", 2, 2)                # 4 colours
    img[1, 1, 2] += 1
    assert not analyse(img).rep8 and choose(img) == ("rgb", 48, 16)
    g = (np.arange(6, dtype=np.uint16).reshape(2, 3, 1) * 257)
    assert choose(g) == ("palette", 4, 4)
    g[0, 0, 0] = 1
    assert choose(g) == ("gray", 16, 16)


def test_opaque_rgba_and_binary_rgb():
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (8, 40, 4), dtype=np.uint8)
    img[..., 3] = 255
    assert choose(img) == ("rgb", 24, 8)
    kind, arr = reduced_call(img)
    assert kind == "png" and arr.shape == (8, 40, 3) and (arr == img[..., :3]).all()
    img[0, 0, 3] = 254
    assert choose(img) == ("rgba", 32, 8)
    mask = np.repeat(rng.integers(0, 2, (8, 9, 1), dtype=np.uint8) * 255, 3, axis=2)
    assert choose(mask) == ("gray", 1, 1)


def test_palette_order_transparent_first():
    keys = np.array([0xFFFFFFFF, 0x00000000, 0x10203040, 0x102030FF, 0x000000FF, 0x05000001], np.uint32)
    pal = palette_order(keys)
    assert pal.tolist() == [[0, 0, 0, 0], [5, 0, 0, 1], [16, 32, 48, 64], [0, 0, 0, 255], [16, 32, 48, 255], [255, 255, 255, 255]]


def test_hash_is_the_documented_one():
    assert hash_slot(0) == 0 and hash_slot(1) == 0x9E3779B1 >> 23
    assert all(0 <= hash_slot(k) < 512 for k in (1, 0xFFFFFFFF, 0x12345678))


@pytest.mark.parametrize("chans,depth", [(c, d) for c in (1, 2, 3, 4) for d in (8, 16)])
def test_slot_bound_covers_every_candidate(chans, depth):
    import fpng_b200 as f
    full = np.zeros((256, 4), np.uint8)
    for w in (1, 2, 3, 7, 8, 9, 31, 100, 1000, 4097):
        for h in (1, 2, 5, 64):
            bound = f.max_reduced_encoded_size(w, h, chans, depth)
            bpp = chans * depth // 8
            assert bound >= f.max_encoded_size(w, h, bpp)
            for d in (1, 2, 4, 8):
                assert bound >= f.max_label_encoded_size(w, h, d)
                k = min(256, 1 << d)
                assert bound >= f.max_label_encoded_size(w, h, d, full[:k])
            for b in (2, 3, 4, 6, 8):                                     # gray16, GA8 / RGB8 / RGBA8 (fpng), GA16, RGB16, RGBA16
                if b <= bpp:
                    assert bound >= f.max_encoded_size(w, h, b)
            assert bound == max(f.max_encoded_size(w, h, bpp), f.max_label_encoded_size(w, h, 8, full))
    assert f.max_reduced_encoded_size(1, 1, 3, 8) == f.max_label_encoded_size(1, 1, 8, full)   # PLTE dominates at 1 x 1


def test_python_argument_rules():
    import torch
    import fpng_b200 as f
    with pytest.raises(ValueError):
        f.encode_png_device([torch.zeros(2, 2, 3, dtype=torch.float32)], depth=8, reduce=True)
    with pytest.raises(ValueError):
        f.encode_png_device([torch.zeros(2, 2, 3, dtype=torch.float16)], reduce=True)
    with pytest.raises(ValueError):
        f.max_reduced_encoded_size(4, 4, 5, 8)
    with pytest.raises(ValueError):
        f.max_reduced_encoded_size(4, 4, 3, 12)
    ofs = f.reduced_slot_offsets([(4, 5, 3, 8), (1, 1, 1, 16)])
    assert ofs.tolist() == [0, (f.max_reduced_encoded_size(5, 4, 3, 8) + 15) // 16 * 16,
                            (f.max_reduced_encoded_size(5, 4, 3, 8) + 15) // 16 * 16 + (f.max_reduced_encoded_size(1, 1, 1, 16) + 15) // 16 * 16]
    assert f.FPNGB_ENCODE_REDUCE == 256
