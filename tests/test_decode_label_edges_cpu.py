"""CPU checks that every case of tests/label_edges.py reaches the construct it names: the nearest kernel's grid-stride loop and
its carry, fp32 source indices that differ from exact arithmetic past 2^23 and hit the clamp, row-end residues and strided
layouts, 64-bit offsets past 4 GiB, and the index store's bands, Adam7 passes and sub-byte widths."""
import numpy as np

import decode_edges as de
import label_edges as le
from test_decode_labels_cpu import nearest_model, nearest_src


def test_grid_cases_run_the_grid_stride_loop():
    want = {(16384, 8195): (2049, 33_570_816, 8187, 1797), (1 << 24, 1): (1, 16_777_216, 16_776_960, 0),
            (5, 1 << 24): (1 << 22, 20_971_520, 3, 4_194_048)}
    assert le.STEP == 16_776_960
    for name, out in le.GRID_CASES:
        g = le.nearest_grid(*out)
        assert g["step"] == le.STEP and g["groups"] > le.STEP, name
        assert (g["gx"], g["groups"], g["dy"], g["dq"]) == want[out], (name, g)
        assert (g["dq"] == 0) == (name == "tall_no_carry"), name
        iters, carries = le.carry_steps(*out)
        assert iters.max() >= 2 and iters.sum() == g["groups"], name
        if name == "iterates_twice_with_and_without_carry":
            assert iters.min() == 2 and (carries[iters >= 2] > 0).any() and (carries[iters >= 2] == 0).any()
        elif name == "tall_no_carry":
            assert not carries.any()
        else:
            twice = iters >= 2
            assert carries[twice].mean() > 0.4, carries[twice].mean()
    assert len(le.GRID_SOURCES) >= 2 and len({tuple(b) for b in le.grid_boxes((5, 5), 0)}) == len(le.GRID_SOURCES)


def test_carry_steps_agree_with_a_step_by_step_walk():
    """the closed form of carry_steps against the kernel's running (row, group) sums, on a shrunken grid"""
    for out_h, out_w in ((7, 33), (50, 1), (3, 101)):
        gx = -(-out_w // 4)
        groups, step = gx * out_h, 64
        for t in range(step):
            if t >= groups:
                continue
            oy, xq, n, c = t // gx, t % gx, 0, 0
            for g in range(t, groups, step):
                assert (oy, xq) == divmod(g, gx)
                n += 1
                oy += step // gx
                xq += step % gx
                if xq >= gx:
                    xq -= gx
                    oy += 1
                    c += 1 if g + step < groups else 0
            iters = -(-(groups - t) // step)
            assert n == iters and c == (t % gx + (iters - 1) * (step % gx)) // gx


def test_fp32_index_differs_past_2_23_and_hits_the_clamp():
    """(indices where fp32 and exact arithmetic differ, those of them >= 2^23, clamped indices) per source length and mode.  With
    n_in = 2^24 - 1 the scale 1 - 2^-24 is exact, so every difference comes from (float)i + 0.5f rounding past 2^23; the other
    lengths add the rounding of the scale itself."""
    want = {((1 << 24) - 1, "nearest"): (0, 0, 0), ((1 << 24) - 1, "nearest-exact"): (4_194_303, 4_194_303, 1),
            (10_000_019, "nearest"): (3_697_372, 2_773_028, 0), (10_000_019, "nearest-exact"): (3_970_391, 3_046_054, 1),
            (5000, "nearest"): (1860, 1395, 0), (5000, "nearest-exact"): (2005, 1541, 1)}
    for n_in in le.FP32_LENGTHS:
        for mode in le.MODES:
            diff, clamp = le.fp32_report(n_in, le.FP32_OUT, mode == "nearest-exact")
            assert (diff.size, int((diff >= 1 << 23).sum()), clamp.size) == want[(n_in, mode)], (n_in, mode)
            if clamp.size:
                assert clamp.tolist() == [le.FP32_OUT - 1]
    diff, _ = le.fp32_report((1 << 24) - 1, le.FP32_OUT, True)
    assert diff.min() >= 1 << 23
    # the model is the fp32 rule, not exact arithmetic: it follows the rounding where the two differ
    diff, _ = le.fp32_report((1 << 24) - 1, le.FP32_OUT, True)
    assert not np.array_equal(nearest_src((1 << 24) - 1, le.FP32_OUT, True)[diff], le.exact_src((1 << 24) - 1, le.FP32_OUT, True)[diff])


def test_fp32_rule_against_torch_cpu_at_2_24():
    """torch's CPU nearest follows the fp32 rule at the fp32 cases.  Its nearest-exact does not past 2^23: it does not form
    (float)i + 0.5f as the CUDA kernel and the header do, so the GPU tests compare with torch's CUDA F.interpolate there."""
    import torch
    import torch.nn.functional as F
    for n_in in le.FP32_LENGTHS:
        x = torch.arange(n_in, dtype=torch.float32).view(1, 1, 1, n_in)
        for mode in le.MODES:
            got = F.interpolate(x, size=(1, le.FP32_OUT), mode=mode).view(-1).numpy().astype(np.int64)
            d = np.nonzero(got != nearest_src(n_in, le.FP32_OUT, mode == "nearest-exact"))[0]
            if mode == "nearest":
                assert d.size == 0, n_in
            else:
                assert (d >= 1 << 23).all(), (n_in, d[:4])


def test_line_pixel_neighbours_differ():
    v = le.line_pixel(np.arange(le.FP32_LENGTHS[0])).astype(np.int64)
    assert (np.diff(v) != 0).all()


def test_layout_cases_cover_every_row_end_and_stride():
    assert sorted(w % 4 for w in le.LAYOUT_WIDTHS) == [0, 1, 2, 3]
    v = le.layout_variants()
    for dt in ("uint8", "uint16", "float16", "bfloat16", "float32"):
        assert {d for (t, d, native, idx) in v if t == dt and native and not idx} == {1, 2, 3, 4}, dt
    assert {(t, d) for (t, d, native, idx) in v if not native} == {(t, d) for t in ("uint8", "float16", "bfloat16", "float32") for d in (3, 4)}
    for layout in le.LAYOUTS:
        for d in (1, 2, 3, 4):
            shape, strides, offset, total = le.layout_strides(layout, 3, le.LAYOUT_OUT_H, 37, d)
            e = le.element_offsets(strides, offset, shape)
            assert np.unique(e).size == e.size and e.min() >= 0 and e.max() < total - 1, (layout, d)
            assert total - e.size >= 3 * 37 * d, (layout, d)                  # guard elements around the view
            if layout == "canvas_odd_offset":
                assert offset % 2 == 1
            if layout == "nchw_padded":
                assert strides[1] > 37 and strides[3] > le.LAYOUT_OUT_H * 37
            if layout == "hcw":
                assert strides[2] == 1 and strides[3] == 38 and strides[1] == 38 * d


def test_big_offsets_pass_4_gib():
    boxes = dict(le.BIG_BOXES)
    for exact in (False, True):
        base, row = le.big_offsets(boxes["bottom_right"], exact)
        assert base > le.FOUR_GIB and row < le.FOUR_GIB
        base, row = le.big_offsets(boxes["top_left"], exact)
        assert base + row < le.FOUR_GIB
        base, row = le.big_offsets(boxes["full_height_strip"], exact)
        assert base < le.FOUR_GIB < row
    assert le.BATCH_IMAGE == 512 << 20 and (le.BATCH_N - 1) * le.BATCH_IMAGE >= le.FOUR_GIB
    place = le.index_big_placement()
    assert place[le.INDEX_BIG_N] >= le.FOUR_GIB and place[le.INDEX_BIG_N + 1] >= le.FOUR_GIB
    assert le.index_big_bytes() < 4.4e9
    assert le.INDEX_BIG_TAIL[0][:3] == (3, 4, 1) and le.INDEX_BIG_TAIL[1][:2] == (0, 16)
    ids = le.index_big_id(3, np.arange(64)[:, None], np.arange(64)[None, :])
    assert len({tuple(r) for r in ids}) > 8 and (ids != le.index_big_id(4, np.arange(64)[:, None], np.arange(64)[None, :])).all()


def test_index_specs_reach_bands_passes_and_sub_byte_widths():
    specs = le.index_specs()
    for ct, d in le.INDEX_FORMATS:
        mine = [s for s in specs if s[:2] == (ct, d)]
        flat = [s for s in mine if s[2] == 0]
        assert {le.bands(s[5]) for s in flat} == {1, 2, 3, 4}, (ct, d)
        assert {s[5] % 32 for s in flat} >= {31, 0, 1}, (ct, d)
        if d < 8:
            per = 8 // d
            assert {s[4] % per for s in flat} == ({0, per - 1, 1} if per > 2 else {0, 1}), (ct, d)
            assert {s[4] * d % 8 for s in flat} >= {0, 8 - d}, (ct, d)
        adam7 = [s for s in mine if s[2] == 1]
        assert adam7 and all(s[5] > 264 and de.ext_passes_min_rows(s[4], s[5]) > 32 for s in adam7), (ct, d)
        if ct == 3:
            assert any(s[7] for s in mine), (ct, d)
    kernels = {le.unfilter_kernel(s) for s in specs if s[:2] == (0, 8)}
    assert kernels == {"png_unfilter_kernel", "png_unfilter_ext_kernel"}
    assert any(s[:4] == (0, 8, 0, True) for s in specs)


def test_index_files_hold_their_samples():
    """each spec's file parses back to the samples the GPU test expects, and palettes stop short of the samples where asked"""
    import pngwrite_formats as pf
    rs = np.random.RandomState(5)
    for k, spec in enumerate(le.index_specs()[::7]):
        png, s = le.index_file(rs, spec, k)
        p = pf.parse(png)
        assert np.array_equal(p["samples"][..., 0].astype(np.int64), s) and (p["w"], p["h"]) == spec[4:6]
        assert p["interlace"] == spec[2] and p["depth"] == spec[1] and p["ctype"] == spec[0]
        if spec[7]:
            assert s.max() >= len(p["plte"])


def test_nearest_model_on_a_crop_is_the_gather_of_nearest_src():
    rs = np.random.RandomState(8)
    px = rs.randint(0, 256, (40, 50)).astype(np.uint8)
    for exact in (False, True):
        for box in ((3, 4, 20, 30), (0, 0, 40, 50), (39, 49, 1, 1)):
            got = nearest_model(px, 17, 61, exact, box)
            iy, ix = nearest_src(box[2], 17, exact), nearest_src(box[3], 61, exact)
            assert np.array_equal(got, px[box[0] + iy][:, box[1] + ix])
