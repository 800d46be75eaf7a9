"""CPU checks of tests/reduce_edges.py: the partition constants match the kernel sources, every paired case changes format at its
deciding pixel (by tests/reduce_model.py), each deciding pixel sits where its case says in the analysis partition, the early-stop
cases put their early evidence in every CTA's first steps, the colliding colours share a slot, and the colour-count, sweep,
conversion and boundary images are what they are named."""
import collections

import numpy as np
import pytest

import reduce_edges as ree
from reduce_model import analyse, choose, hash_slot


@pytest.fixture(scope="module")
def edges():
    return ree.edge_cases()


@pytest.fixture(scope="module")
def early():
    return ree.early_stop_cases()


def test_constants_match_sources():
    found = ree.source_constants()
    assert found == {k: v for k, (_, v) in ree.KERNEL_CONSTANTS.items()}, found


def test_partition_round_trip():
    for p in (0, 255, 256, 7936, 8191, 8192, 123457):
        assert ree.pixel_at(*ree.place(p)) == p
    assert ree.place(8191) == (0, 31, 255) and ree.place(8192) == (1, 0, 0)


def test_every_pair_changes_format(edges, early):
    for c in edges + early:
        assert c.want != c.want_changed, c.name
        assert (c.want, c.want_changed) == (ree.fmt_of(c.base), ree.fmt_of(c.changed)), c.name
        diff = np.flatnonzero((c.base != c.changed).reshape(c.base.shape[0] * c.base.shape[1], -1).any(1))
        assert diff.tolist() == [c.pixel], c.name


def test_edge_positions_and_widths(edges):
    by_prop = collections.defaultdict(set)
    for c in edges:
        by_prop[c.meta["prop"]].add(c.meta["w"])
        h, w = c.base.shape[:2]
        cta, step, thread = c.place
        pos = c.meta["pos"]
        ctas = ree.analyze_ctas(w, h)
        want = {"first": (0, 0, 0), "step0_last_thread": (0, 0, 255), "cta0_last_step": (0, 31, 0), "cta0_last": (0, 31, 255),
                "cta1_first": (1, 0, 0), "last_cta_first": (ctas - 1, 0, 0)}
        if pos in want:
            assert (cta, step, thread) == want[pos], c.name
        elif pos == "mid_cta_last_step":
            assert 0 < cta < ctas - 1 and step == 31, c.name
        else:
            assert c.pixel == w * h - 1 and cta == ctas - 1, c.name
        assert ctas >= 3
    assert set(by_prop) == {"not_opaque", "not_gray", "not_rep8", "lattice", "colour_257"}
    for prop, ws in by_prop.items():
        assert ws == set(ree.WIDTHS), (prop, ws)
    partial = {c.meta["w"] for c in edges if (c.base.shape[0] * c.base.shape[1]) % ree.RED_PIXELS}
    assert partial == set(ree.WIDTHS) - {8192}                        # 8192 | w * h only at w = 8192
    classes = collections.defaultdict(set)
    for c in edges:
        classes[c.meta["prop"]].add((c.chans, c.depth))
    assert classes["lattice"] == set(ree.CLASSES)
    assert classes["not_rep8"] == {(c, 16) for c in (1, 2, 3, 4)}
    assert classes["colour_257"] == {(c, d) for c in (2, 3, 4) for d in (8, 16)}
    rep8 = {(c.chans, c.name.split("_")[2], int(c.changed.reshape(-1, c.chans)[c.pixel]["rgba".index(c.name.split("_")[2])
            if c.chans > 2 else "ra".index(c.name.split("_")[2])])) for c in edges if c.meta["prop"] == "not_rep8"}
    for ch in (1, 2, 3, 4):
        for name in {1: "r", 2: "ra", 3: "rgb", 4: "rgba"}[ch]:
            assert {v for (c, n, v) in rep8 if (c, n) == (ch, name)} == set(ree.REP8_BREAKERS), (ch, name)


def test_need_mask_classes():
    """1 and 2 channels never stop early (not-gray cannot be set); RGB8 stops only when nothing is left to decide"""
    for c, d in ree.CLASSES:
        assert ree.can_stop(c, d) == ((c, d) not in ree.NEVER_STOPS), (c, d)
    rng = np.random.default_rng(0)
    for _ in range(20):                                                # overflow + not gray in RGB8: always RGB
        img = rng.integers(0, 256, (20, 20, 3), dtype=np.uint8)
        assert choose(img)[0] == "rgb"
    stopping = {ree.EARLY_CLASS[r] for r in ree.EARLY_ROWS}
    assert stopping == {(c, d) for (c, d) in ree.CLASSES if ree.can_stop(c, d)} - set(ree.FINAL_WHEN_STOPPED)


def test_early_evidence_in_first_steps(early):
    """every CTA of every base image has read its row's early bits by the end of step 1; the late bit is nowhere in the base, and
    in the changed image only from the deciding pixel's step on"""
    for c in early:
        early_bits, late_bit = ree.EARLY_BITS[c.meta["row"]]
        assert ree.need_mask(c.chans, c.depth) == early_bits | late_bit, c.name
        steps = ree.early_evidence_steps(c.base)
        for b, seen in steps.items():
            if len(seen) >= 2 and c.meta["row"] != "rgba8_palette_vs_rgba":
                assert seen[1] & early_bits == early_bits, (c.name, b, seen[:2])
            elif c.meta["row"] == "rgba8_palette_vs_rgba":
                assert seen[0] & early_bits == early_bits, (c.name, b)
            assert not seen[-1] & late_bit or late_bit == ree.OVERFLOW, (c.name, b)
        cta, step, _ = c.place
        assert step >= 2 or cta == len(steps) - 1, c.name
        assert c.meta["pos"] in ree.FAR


def test_colour_set_images():
    for name, img, want, facts in ree.colour_set_images():
        assert ree.fmt_of(img) == want, name
        an = analyse(img)
        if "K" in facts and facts["K"] <= 256:
            assert len(an.colours) == facts["K"], name
        if "K" in facts and facts["K"] > 256:
            assert an.colours is None, name
        if "slot" in facts:
            assert {hash_slot(int(k)) for k in facts["keys"]} == {facts["slot"]}, name
            assert len(facts["keys"]) in (255, 256, 257), name
        if name.startswith("zero_last"):
            flat = img.reshape(-1, 4)
            z = np.flatnonzero((flat == 0).all(1))
            assert z.tolist() == [facts["zero_at"]], name
        if name.startswith("hi_bytes"):
            assert not an.rep8 and len(np.unique(img >> 8, axis=None)) <= 256
    one = [x for x in ree.colour_set_images() if x[0] == "one_cta_257"][0][1].reshape(-1, 3)
    per_cta = [len(np.unique(ree.key_of(np.concatenate([one[b * 8192:(b + 1) * 8192], np.full((8192, 1), 255, np.uint8)], 1))))
               for b in range(3)]
    assert per_cta[1] == 257 + 1 and per_cta[0] == per_cta[2] == 1


def test_racing_and_16k_images():
    img = ree.racing_same_colours(16)
    assert img.shape == (16, ree.RED_PIXELS, 3)
    firsts = set()
    for r in range(16):
        assert len(np.unique(ree.key_of(np.concatenate([img[r], np.full((ree.RED_PIXELS, 1), 255, np.uint8)], 1)))) == 256
        firsts.add(tuple(img[r, 0]))
    assert len(firsts) == 16 and ree.fmt_of(img) == ("palette", 8)
    for ch in (3, 4):
        big = ree.overflow_16k_colours(ch, 8)
        keys = [np.unique(ree.key_of(np.concatenate([big[r], np.full((ree.RED_PIXELS, 4 - ch), 255, np.uint8)], 1)
                                     if ch == 3 else big[r])) for r in range(8)]
        assert all(len(k) == 256 for k in keys) and len(np.unique(np.concatenate(keys))) == 8 * 256
    assert ree.fmt_of(ree.overflow_16k_colours(3)) == ("rgb", 8) and ree.fmt_of(ree.overflow_16k_colours(4)) == ("rgba", 8)


def test_sweep_intents():
    imgs = ree.sweep_images()
    reached, choices = set(), set()
    for name, img, it in imgs:
        an = analyse(img)
        assert an.gray == it["gray"] and an.rep8 == it["rep8"], name
        assert an.opaque == (it["alpha"] == "opaque"), name
        if it["rep8"]:
            assert (an.colours is None) == (it["K"] > 256), name
            if an.colours is not None:
                assert len(an.colours) == it["K"], name
                assert (0 in an.colours) == it["zero"], name
                translucent = int(((an.colours & 0xFF) != 0xFF).sum())
                assert translucent == {"opaque": 0, "one": 1, "all": it["K"]}[it["alpha"]], name
        if "lattice" in it:
            assert an.lattice == it["lattice"], name
        f, bits, depth = choose(img)
        reached.add((img.shape[2], 16 if img.dtype == np.uint16 else 8, f, depth))
        choices.add((f, depth))
    assert choices == {("gray", d) for d in (1, 2, 4, 8, 16)} | {("palette", d) for d in (1, 2, 4, 8)} | \
        {(f, d) for f in ("ga", "rgb", "rgba") for d in (8, 16)}
    ks = collections.Counter(it["K"] for _, _, it in imgs)
    assert set(ks) == set(ree.SWEEP_K)
    assert any(it["zero"] and it["K"] in (256, 257) for _, _, it in imgs)


def test_conversion_modes_and_shapes():
    modes = ree.conversion_modes()
    seen = set()
    for m, (c, d, cols, want) in modes.items():
        for w in ree.CONV_WIDTHS:
            img = ree.conversion_image(m, w)
            assert img.shape[1:] == (w, c) and ree.fmt_of(img) == want, (m, w)
        for w, h, wh in ree.cta_shapes(m):
            assert ree.fmt_of(ree.conversion_image(m, w, h)) == want, (m, w, h)
            seen.add(wh)
    assert {255, 256, 257} <= seen
    bits_mod = {(w * b) % 32 for w in ree.CONV_WIDTHS for b in (1, 2, 4, 8)}
    assert bits_mod == set(range(0, 32))
    assert {(w * b) % 4 for w in ree.CONV_WIDTHS for b in (1, 2, 3, 4, 6, 8)} == {0, 1, 2, 3}


def test_boundary_images():
    imgs = ree.boundary_images()
    assert [img.shape[0] * img.shape[1] for _, img in imgs] == list(ree.BOUNDARY_PIXELS)
    allcols = set()
    for i, (name, img) in enumerate(imgs):
        f = ree.fmt_of(img)
        if name.endswith("keep"):
            assert f == ("gray", 8) and img.shape[2] == 1
            cut = img[:, 1:-1]
            assert ree.fmt_of(cut) == ("gray", 4)                     # the first and the last pixel decide it
        else:
            assert f[0] == "palette"
            K = len(analyse(img).colours)
            assert K <= 256
            allcols |= set(analyse(img).colours.tolist())
            if img.shape[1] > 2:
                assert K == len(analyse(img[:, 1:-1]).colours) + 2
    assert len(allcols) > 256
