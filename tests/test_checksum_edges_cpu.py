"""CPU checks of tests/checksum_edges.py: the partition constants match the kernel sources, every case reaches the construct it
was built for (by the pure-Python model of the kernel's partition), every expected status is zlib's, and with the check off the
oracle decodes the fpng cases as expected (transplanted files are valid streams of A')."""
import collections

import numpy as np
import pytest

import checksum_edges as ce


@pytest.fixture(scope="module")
def fpng(oracle):
    return ce.fpng_cases(oracle)


@pytest.fixture(scope="module")
def general():
    return ce.general_cases()


def by_prefix(cases, prefix):
    out = [c for c in cases if c.name.startswith(prefix)]
    assert out, prefix
    return out


def test_constants_match_sources():
    found = ce.source_constants()
    assert found == {k: v for k, (_, v) in ce.KERNEL_CONSTANTS.items()}, found


def test_statuses_are_zlibs(fpng, general):
    for c in fpng + general:
        assert c.recheck() == (c.want, c.want_off if c.kind != "fpng" else c.recheck()[1]), c.name
    counts = collections.Counter(c.want for c in fpng + general)
    assert set(counts) == {ce.OK, ce.CRC, ce.INVALID_IDAT, ce.ADLER}, counts


def test_crc_tails_and_alignments(fpng):
    cases = by_prefix(fpng, "crc_tail")
    assert {(c.reach["m0_mod4"], c.reach["tail"]) for c in cases} == {(a, t) for a in range(4) for t in range(4)}
    for c in cases:
        assert c.want == ce.OK
        masked = bytes.fromhex(c.reach["masked"])
        assert len(masked) == c.reach["m0_mod4"] and (masked[-1:] != b"\0"), c.name   # the byte before "IDAT" is not 0: reading it changes the CRC


def test_crc_sizes(fpng):
    cases = by_prefix(fpng, "crc_size")
    assert all(c.want == ce.OK for c in cases)
    ctas = {c.reach["ctas"] for c in cases}
    assert {1, 2, 3, 5, 6} <= ctas, ctas
    assert any(c.reach["first_chunk_words"] < ce.CS2_WARP_WORDS for c in cases)       # first warp chunk partly inside
    assert any(c.reach["first_chunk_words"] == ce.CS2_WARP_WORDS for c in cases)
    assert len({c.reach["first_lane"] for c in cases}) >= 8
    words = {c.reach["words"] % ce.CS2_CTA_WORDS for c in cases}
    assert {0, 1, ce.CS2_CTA_WORDS - 1} <= words, words
    for c in cases:
        assert c.reach["ctas"] <= c.reach["grid"] - 1


def test_crc_damage_places(fpng):
    cases = by_prefix(fpng, "crc_damage")
    assert all(c.want == ce.CRC for c in cases)
    assert max(c.reach["place"].get("cta", 0) for c in cases) == cases[0].reach["ctas"] - 1 >= 5
    tails = {c.reach["place"]["tail"] for c in cases if c.reach["place"]["tail"] is not None}
    assert tails == {0, 1, 2} and cases[0].reach["tail"] == 3
    places = [c.reach["place"] for c in cases if c.reach["place"]["tail"] is None]
    edges = {(p["cta"], p["warp"], p["step"], p["lane"]) for p in places}
    assert (2, ce.CS2_WARPS - 1, 0, 0) in edges and (2, 0, ce.CS2_WARP_WORDS // ce.LANES - 1, ce.LANES - 1) in edges   # a CTA's ends
    assert (1, 3, 0, 0) in edges and (1, 3, ce.CS2_WARP_WORDS // ce.LANES - 1, ce.LANES - 1) in edges                 # a chunk's ends
    assert (0, 5, 17, 0) in edges and (0, 5, 17, ce.LANES - 1) in edges                                              # a step's ends
    assert (0, 0, ce.CS2_WARP_WORDS // ce.LANES - 1, ce.LANES - 1) in edges                                           # the last whole word
    first = [c for c in cases if c.name == "crc_damage_first_data_byte"][0]
    assert first.reach["place"]["cta"] == first.reach["ctas"] - 1


def test_crc_grid(fpng):
    for c in by_prefix(fpng, "crc_grid"):
        assert c.want == ce.OK and c.reach["ctas"] == c.reach["grid"] - 1 and c.reach["words"] % ce.CS2_CTA_WORDS == 1


def test_adler_sizes(fpng):
    cases = by_prefix(fpng, "adler_1pass") + by_prefix(fpng, "adler_2pass") + by_prefix(fpng, "adler_stored")
    assert all(c.want == ce.OK for c in cases)
    assert {c.reach["rem"] for c in cases} == set(range(ce.VEC))
    assert {ce.LANES - 1, ce.LANES, ce.LANES + 1} <= {c.reach["nvec"] for c in cases}
    assert {1, 2, 7, 8, 9, 41, 70000} <= {c.reach["h"] for c in cases}
    assert {c.reach["last_rows"] for c in cases} >= {1, 2, 7, 8}
    assert sum(c.reach["row_mod"] == 0 for c in cases) == 6                    # w * c + 1 = 65521, both shapes, three modes
    assert any(c.reach["h"] > ce.ADLER_MOD for c in cases)
    for c in cases:
        stored = c.reach["stored_blocks"]
        assert stored or not c.name.startswith("adler_stored")
        assert c.reach["filters"] == ([0] if stored or c.reach["h"] == 1 else [0, 2]), c.name
    compressed = [c for c in cases if not c.reach["stored_blocks"]]
    assert {2, 7, 8, 9, 41, 70000} <= {c.reach["h"] for c in compressed}            # the closed-form filter term at h = 2 and past 65521
    assert any(c.reach["row_mod"] == 0 for c in compressed) and {0, 1, 15} <= {c.reach["rem"] for c in compressed}


def test_adler_transplants(fpng, oracle):
    cases = by_prefix(fpng, "adler_transplant")
    assert len(cases) == 3 * len(ce.T_SPOTS) and all(c.want == ce.ADLER for c in cases)
    places = [c.reach["place"] for c in cases]
    assert any(p["masked"] for p in places) and any(p["cta"] == c.reach["row_ctas"][0] - 1 for p, c in zip(places, cases))
    assert {c.reach["y"] for c in cases} >= {0, ce.T_H - 1} and {c.reach["x"] for c in cases} >= {0, ce.T_W * ce.T_C - 1}
    for c in cases:
        st, px = oracle.decode(c.png, ce.T_C)[:2]
        assert st == 0 and np.array_equal(px, c.pixels.reshape(-1)), c.name


def test_fpng_verify_off_oracle(fpng, oracle):
    """every clean and transplanted fpng file is a valid stream the oracle decodes; the damaged ones are recorded as it decodes them"""
    for c in fpng:
        if c.want in (ce.OK, ce.ADLER):
            w, h, ch = ce.fpng_shape(c.png)[:3]
            assert oracle.decode(c.png, ch)[0] == 0, c.name


def test_gather_runs(general):
    cases = by_prefix(general, "gather_")
    runs = [c for c in cases if "damage" not in c.name]
    for c in runs:
        assert c.want == ce.OK
        assert set(ce.GATHER_LENS) <= set(c.reach["lens"])
    zeros = [c.reach["lens"].index(0) for c in runs]
    assert zeros[0] == 0 and 0 < zeros[1] < len(runs[1].reach["lens"]) - 1 and zeros[2] == len(runs[2].reach["lens"]) - 1
    segs = {s for c in runs for s in c.reach["segments"]}
    assert any(s[1] == 1 for s in segs) and any(s[2] == ce.GATHER_THREADS for s in segs) and any(s[3] < s[1] for s in segs)
    damaged = [c for c in cases if "damage" in c.name]
    assert all(c.want == ce.CRC for c in damaged)
    assert {c.reach["chunk"] for c in damaged} >= {0, len(runs[1].reach["lens"]) - 1, runs[1].reach["lens"].index(8192)}
    shifts = {c.reach["place"]["shift"] for c in damaged if "place" in c.reach}
    assert 0 in shifts and len(shifts) >= 4


def test_inflate_lanes(general):
    cases = by_prefix(general, "inflate_N")
    assert all(c.want == ce.OK for c in cases)
    lanes = [c.reach["lanes"] for c in cases]
    assert any(c.reach["N"] < ce.LANES and c.reach["lanes"]["empty"] > 0 for c in cases)
    assert any(x["wrap_lanes"] for x in lanes)
    assert any(x["start_past_mod"] and x["per"] >= ce.ADLER_MOD for x in lanes)
    assert {c.reach["N"] % ce.ADLER_MOD for c in cases} >= {1, ce.ADLER_MOD - 1}
    split = by_prefix(general, "inflate_adler_split")
    assert all(c.want == ce.OK for c in split) and {c.reach["adler_bytes_in_last_chunk"] for c in split} == {1, 2, 3}


def test_inflate_transplants(general):
    cases = by_prefix(general, "inflate_transplant")
    assert all(c.want == ce.ADLER and c.want_off == ce.OK for c in cases)
    places = [c.reach["place"] for c in cases]
    assert any(p["lane_offset"] == 0 and p["lane"] > 0 for p in places)
    assert any(p["lane_offset"] == -(-c.reach["N"] // ce.LANES) - 1 for p, c in zip(places, cases))
    assert sum(p["mod_pos"] == ce.ADLER_MOD - 1 for p in places) >= 3
    ext = by_prefix(general, "ext_transplant")
    assert len(ext) == 4 and all(c.want == ce.ADLER and c.want_off == ce.OK for c in ext)
    bad = by_prefix(general, "ext_bad_filter_and_adler") + by_prefix(general, "inflate_bad_filter_and_adler")
    assert len(bad) == 3 and all((c.want, c.want_off) == (ce.INVALID_IDAT, ce.INVALID_IDAT) for c in bad)
    for c in bad:
        run = ce.idat_run(c.png)
        raw, adler = ce.inflate(b"".join(x[2] for x in run))
        assert adler != (__import__("zlib").adler32(raw) & 0xFFFFFFFF)                  # the Adler-32 is wrong as well


def test_big_case_places():
    """the big file's message passes 2^29 bytes, so the final shift 8 (L - m0) and the first CTAs' shifts need exponent bits >= 32"""
    t = ce.big_message_len()
    assert t > 1 << 29
    m0, L = ce.FPNG_MSG_START, ce.FPNG_MSG_START + t
    assert 8 * (L - m0) >= 1 << 32
    places = [ce.crc_place(m0, L, b) for b in ce.big_damage_spots()]
    assert places[0]["cta"] == ce.crc_ctas(m0, L) - 1 and places[0]["cta_shift"] >= 1 << 32
    assert places[1]["cta_shift"] >= 1 << 32
