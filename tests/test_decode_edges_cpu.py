"""CPU checks of tests/decode_edges.py: every case reaches the construct it names (tiles past the grid, tap counts in the thousands,
source rows and outputs past 4 GiB, fp32 centres that round, unfilter CTA and band edges), the sparse model equals the dense one of
test_decode_resized_cpu.py, and the fp32 emulation of the kernel's summation order stays within the bound E on every resize case."""
import numpy as np
import pytest

import decode_edges as de
from test_decode_resized_cpu import resize_model

TWO32 = 1 << 32


def test_tile_loop_cases_pass_the_grid():
    for c in de.tile_loop_cases():
        assert c.tiles() > de.GRID_X, (c.name, c.tiles())
        print(c.name, "tiles", c.tiles(), "taps", c.taps())
    assert [c.tiles() for c in de.tile_loop_cases()] == [524288, 524288, 65792]


def test_fp32_centre_rounds_past_2_23():
    """at output indices >= 2^23, (float)i + 0.5f rounds: some outputs of the 2^24-wide case have taps other than those of the
    correctly rounded centre, so the GPU comparison checks the fp32 rule and not only an approximation of it"""
    n_out = 1 << 24
    for c in de.tile_loop_cases()[:2]:
        w = c.src[1]
        below = de.center_rounds(w, n_out, c.aa, lo=(1 << 23) - 4096, hi=1 << 23)
        above = de.center_rounds(w, n_out, c.aa, lo=1 << 23, hi=(1 << 23) + (1 << 16))
        assert len(below) == 0 and len(above) > 0, (c.name, len(below), len(above))
        i = int(above[0])
        print(c.name, "first index with other taps", i, "of", len(above), "in 2^16")
        a, sa, wa = de.spans(w, n_out, c.aa, [i])
        b, sb, wb = de.spans(w, n_out, c.aa, [i], exact_center=True)
        assert (a[0], sa[0]) != (b[0], sb[0]) or not np.array_equal(wa, wb)


def test_tap_counts():
    want = {"taps_3840x8_to_1x1_aa1": (3840, 8), "taps_3840x8_to_3x2_aa1": (2560, 6), "taps_8x2160_to_1x1_aa1": (8, 2160),
            "taps_16384x2_to_1x1_aa1": (16384, 2), "taps_1920x1080_to_7x5_aa1": (549, 432),
            "taps_3840x8_to_1x1_aa0": (2, 2), "taps_16384x2_to_1x1_aa0": (2, 2)}
    got = {c.name: c.taps() for c in de.tap_cases()}
    for c in de.tap_cases() + de.native_tap_cases():
        print(c.name, "taps (nx, ny)", c.taps())
    for k, v in want.items():
        assert got[k] == v, (k, got[k])
    assert max(c.taps()[0] for c in de.native_tap_cases()) == 4096


def test_big_intermediate_offsets():
    """the bottom-right box's first source row lies past 4 GiB of its file's uint16 intermediate; the control box's at 0"""
    assert de.BIG_W * de.BIG_H * 4 < TWO32                         # not TOO_LARGE at 4 channels
    br, tl = de.big_cases()
    print("first source row byte offsets", br.first_row_offset(), tl.first_row_offset())
    assert br.first_row_offset() > TWO32 and tl.first_row_offset() < TWO32
    assert de.BIG_W * de.BIG_H * 4 * 2 > TWO32 and (de.BIG_H - 1) * de.BIG_W * 8 > TWO32       # the ragged output's last rows


def test_batch_past_4_gib():
    per = de.batch_bytes() // de.BATCH_N
    assert per == 512 << 20 and (de.BATCH_N - 1) * per >= TWO32


def test_fpng_shapes_reach_cta_and_row_edges():
    s = de.fpng_shapes()
    assert {w for w, _, _, _ in s} == set(de.FPNG_WIDTHS)
    assert any(w > de.UNFILTER_CTA_PX and w % de.UNFILTER_CTA_PX == 1 for w, _, _, _ in s)
    assert any(h % de.ROWS_AHEAD for _, h, _, _ in s) and any(h > de.ROWS_AHEAD and h % de.ROWS_AHEAD for _, h, _, _ in s)
    assert {st for *_, st in s} == {False, True} and {c for _, _, c, _ in s} == {3, 4}


def test_stored_images_are_stored(oracle):
    """the noise images fpng writes as stored blocks (BTYPE 0, which the decoder unfilters without its running sum), the pattern
    ones mostly Huffman coded (fpng stores the smallest of them too)"""
    coded = {}
    for w, h, c, stored in de.fpng_shapes():
        img = de.fpng_image(w, h, c, stored, w + h)
        png = oracle.encode(img, w, h, c, 0)
        btype = png[png.index(b"IDAT") + 6] >> 1 & 3                 # the first block header, after the 2-byte zlib header
        assert btype == 0 or not stored, (w, h, c)
        if not stored:
            coded[(w, h)] = btype != 0
    print("Huffman-coded pattern files", sum(coded.values()), "of", len(coded))
    assert all(v for (w, h), v in coded.items() if h >= 9)
    assert {w for (w, h), v in coded.items() if v} == set(de.FPNG_WIDTHS)


def test_band_edges():
    g = de.general_shapes()
    assert {h // de.BAND for _, h, _ in g} >= {0, 1, 2, 3} and {ct for *_, ct in g} == {0, 2, 4, 6}
    for ct, depth, il, trns, w, h in de.ext_specs():
        if il:
            assert de.ext_passes_min_rows(w, h) > de.BAND, (w, h)
        elif depth < 8:
            assert w % 8 in (7, 0, 1) and h > 2 * de.BAND


@pytest.mark.parametrize("aa", [True, False])
def test_sparse_model_equals_dense(aa):
    rs = np.random.RandomState(4)
    for (h, w, H, W, box) in ((37, 53, 24, 30, None), (48, 64, 200, 97, None), (90, 120, 7, 5, (3, 11, 80, 100)), (8, 300, 1, 1, None),
                              (1, 9, 5, 2, None), (30, 2, 1000, 3, (29, 1, 1, 1))):
        px = rs.randint(0, 65536, (h, w, 2))
        bh, bw = (h, w) if box is None else box[2:]
        rows = np.arange(H)
        got = de.model_rows(de.array_fetch(px, box), bh, bw, H, W, aa, rows)
        want = resize_model(px, H, W, aa, box)
        assert np.abs(got - want).max() <= 1e-9 * 65535, (h, w, H, W)


def _check_bound(c, px, cols=None):
    _, _, bh, bw = c.crop
    rows = np.arange(c.out[0]) if c.rows is None else c.rows
    fetch = de.array_fetch(px, c.box)
    r = de.model_rows(fetch, bh, bw, c.out[0], c.out[1], c.aa, rows, cols)
    e = de.emulate_rows(fetch, bh, bw, c.out[0], c.out[1], c.aa, rows, cols)
    nx, ny = de.taps(bh, bw, c.out[0], c.out[1], c.aa, rows, cols)
    E = de.bound(nx[None, :, None], ny[:, None, None], int(px.max()))
    d = np.abs(e - r)
    assert (d <= E).all(), (c.name, float((d / E).max()))
    return float(d.max()), float((d / E).max())


def test_bound_holds_for_the_kernel_order():
    """the fp32 emulation of the kernel's order against the float64 model, on every resize case (columns sampled where the output
    is 2^24 wide): within E everywhere.  Prints the largest error and its ratio to E per family."""
    rs = np.random.RandomState(9)
    fam = {}
    for c in de.tile_loop_cases():
        px = de.smooth(c.src[0], c.src[1], 3, 1)
        cols = None
        if c.out[1] > 65536:
            cols = np.unique(np.concatenate([rs.randint(0, c.out[1], 256), np.arange((1 << 23) - 16, (1 << 23) + 240), [c.out[1] - 1]]))
        rows = c.rows[:3] if c.rows is not None else None
        c2 = de.ResizeCase(c.name, c.src, c.out, rows=rows)
        fam.setdefault("tile_loop", []).append(_check_bound(c2, px, cols))
    for c in de.tap_cases():
        fam.setdefault("taps", []).append(_check_bound(c, de.smooth(c.src[0], c.src[1], 3, 2)))
    for c in de.native_tap_cases():
        fam.setdefault("native_taps", []).append(_check_bound(c, de.smooth(c.src[0], c.src[1], c.chans, 3, depth=16)))
    big = de.smooth(2160, 3840, 3, 4)
    for c in de.crop_cases(2160, 3840)[::3]:
        fam.setdefault("crops", []).append(_check_bound(c, big))
    for c in de.big_cases():
        _, _, bh, bw = c.crop
        rows = np.arange(c.out[0])
        r = de.model_rows(de.big_fetch(c.box), bh, bw, c.out[0], c.out[1], c.aa, rows)
        e = de.emulate_rows(de.big_fetch(c.box), bh, bw, c.out[0], c.out[1], c.aa, rows)
        nx, ny = de.taps(bh, bw, c.out[0], c.out[1], c.aa, rows)
        E = de.bound(nx[None, :, None], ny[:, None, None], 65535)
        assert (np.abs(e - r) <= E).all()
        fam.setdefault("big", []).append((float(np.abs(e - r).max()), float((np.abs(e - r) / E).max())))
    for k, v in fam.items():
        print(k, "max |emulated - model|", max(a for a, _ in v), "max ratio to E", max(b for _, b in v))
