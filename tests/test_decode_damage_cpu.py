"""CPU tests of the damaged-stream corpus (tests/decode_damage.py): the oracle decodes every large, stored and placed case as the
reference does, status and pixels, at both desired channel counts (the small files are the CPU stream fuzz of
tests/test_oracle_cpu.py, compared there); every placed case lands where its name says; and every large base file's damage
reaches both outcomes the GPU comparison needs: a file that still decodes, to other pixels, and one that fails."""
from collections import Counter

import numpy as np

import decode_damage as dd
import deflatetrace
import streamgen


def test_oracle_equals_reference(oracle, ref):
    cases, _ = dd.corpus(oracle)
    n, classes = 0, Counter()
    for c in cases:
        if c.group == "small":
            continue
        for d in (3, 4):
            a, b = oracle.decode(c.file, d), ref.decode(c.file, d)
            assert a[0] == b[0], (c.name, d, a[0], b[0])
            if a[0] == 0:
                assert np.array_equal(a[1], b[1]), (c.name, d)
            classes[(c.group.split("_c")[0] if c.group.startswith("placed") else c.group, "decodes" if a[0] == 0 else "fails")] += 1
            n += 1
    print(f"{n} decodes:", dict(sorted(classes.items())))
    assert n > 1300


def test_placed_cases_land_where_they_claim(oracle):
    cases, _ = dd.corpus(oracle)
    placed = [c for c in cases if c.group.startswith("placed")]
    where = Counter()
    for c in placed:
        assert dd.claim_holds(c), (c.name, c.bit)
        if c.sym is not None:
            assert dd.symbol_at(c.file, c.bit) == c.sym, c.name             # the violating token is read there
        where[c.where] += 1
    print("placed cases per boundary:", dict(where))
    assert set(where) == {"first", "last"} | set(dd.BOUNDS)
    assert {c.family for c in placed} == set(dd.MID_KINDS + dd.ROW_KINDS + dd.END_KINDS + dd.FIRST_KINDS)
    # random damage near a boundary is within NEAR_BYTES of it
    large = {x[0] for x in dd.LARGE}
    for c in cases:
        if c.group in large and c.where in dd.BOUNDS:
            assert abs(c.bit - dd.BOUNDS[c.where]) <= 8 * dd.NEAR_BYTES + 8, c.name


def test_token_offsets_against_deflatetrace():
    """the offsets dynamic_file records and the vectorised writer of the placed cases agree with an independent Deflate reader on
    small files: same tokens, and the symbol each offset points at"""
    for chans in (3, 4):
        for code in dd.codes_for(chans):
            rs = np.random.RandomState(chans)
            kind, val, *_ = dd.base_tokens(code, rs, w=24, h=6)
            toks = [("L", int(v)) if k == 0 else (("M", int(v)) if k == 1 else ("E",)) for k, v in zip(kind, val)]
            f, data, offs = streamgen.dynamic_file(24, 6, chans, code.lit, code.dist, toks, offsets=True)
            blk, starts = code.pack(kind, val)
            o, n = dd.idat(f)
            assert f[o + 10:o + 10 + len(blk)] == blk and list(starts + 16) == offs
            assert dd.filtered(kind, val, chans) == data
            tr = deflatetrace.trace(f[o + 8:o + 8 + n])
            want = [t[1] if t[0] == "L" else (t[1], chans) for t in toks if t[0] != "E"]
            assert tr.blocks[0].tokens == want and tr.data == data
            lit, tok0 = dd.dynamic_header(f)
            assert lit == code.lit and tok0 == offs[0] + dd.bit0(o)
            for t, at in zip(toks, offs):
                sym = 256 if t[0] == "E" else (t[1] if t[0] == "L" else streamgen.length_symbol(t[1])[0])
                assert dd.symbol_at(f, at + dd.bit0(o)) == sym


def test_large_files_reach_both_outcomes(oracle):
    cases, bases = dd.corpus(oracle)
    for name, (png, w, h, c, fl) in bases.items():
        clean = oracle.decode(png, c)[1]
        seen = set()
        for k in [k for k in cases if k.group == name]:
            st, px, *_ = oracle.decode(k.file, c)
            seen.add("fails" if st else ("other_pixels" if not np.array_equal(px, clean) else "same_pixels"))
        assert {"fails", "other_pixels"} <= seen, (name, seen)


def test_cpu_fuzz_is_the_stream_fuzz(oracle):
    """the small files are the 2500 mutants of the CPU stream fuzz, five families, every one inside the IDAT payload"""
    fz = dd.cpu_fuzz(oracle)
    assert len(fz) == 2500 and {m for *_, m, _ in fz} == set(range(5))
