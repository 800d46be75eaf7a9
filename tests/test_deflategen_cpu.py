"""CPU checks of tests/deflategen.py, the Deflate writer of the inflate differential tests (test_inflate_streams_gpu.py): every
valid stream inflates with zlib to its input, a pure-Python Deflate walker (below, independent of the writer) finds every construct
the writer is meant to reach in the corpus the GPU test decodes, zlib rejects every named invalid stream, and the zlib header model
of `expect` agrees with zlib on all 65536 two-byte headers."""
import struct
import zlib
from bisect import bisect_right
from collections import Counter

import pytest

import deflategen as dg
from streamgen import CL_ORDER, LEN_BASE, LEN_XBITS

FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8


class WalkError(Exception):
    pass


def decode_table(lens):
    """(table of 2^15 entries: (symbol, length) by the next 15 bits, or None where no code starts)"""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    tab = [None] * (1 << 15)
    for s, l in enumerate(lens):
        if l:
            c = nxt[l]
            nxt[l] += 1
            r = int(format(c, "0%db" % l)[::-1], 2)
            tab[r::1 << l] = [(s, l)] * (1 << (15 - l))
    return tab


def kraft_left(lens):
    """zlib's inftrees measure: < 0 over-subscribed, > 0 incomplete, 0 complete (or no codes)"""
    left = 1
    for l in range(1, 16):
        left = 2 * left - lens.count(l)
        if left < 0:
            return -1
    return left if any(lens) else 0


def check_tree(lens, what, lax):
    """zlib's acceptance of a lit/len or distance code; an incomplete one passes with "incomplete" in lax"""
    left = kraft_left(lens)
    if left < 0:
        raise WalkError("over-subscribed " + what)
    if left > 0 and sorted(l for l in lens if l) != [1] and "incomplete" not in lax:
        raise WalkError("incomplete " + what)


def walk(z, lax=()):
    """inflates the zlib stream z with zlib's rules and counts its constructs; returns (output, Counter).  lax names rules to leave
    out: "fields" (HLIT > 286, HDIST > 30), "incomplete CL", "incomplete" (lit/len, distance), "16 first" (repeats length 0),
    "repeat past" (cut at HLIT + HDIST), "nlen", "distance" (bytes before the start read as 0)"""
    buf = bytes(z) + b"\0" * 8
    pos = 16
    out = bytearray()
    seen = Counter()
    stored = []                                                         # output ranges written by stored blocks

    def bits(n):
        nonlocal pos
        v = (int.from_bytes(buf[pos >> 3:(pos >> 3) + 4], "little") >> (pos & 7)) & ((1 << n) - 1)
        pos += n
        return v

    def sym(tab):
        nonlocal pos
        e = tab[(int.from_bytes(buf[pos >> 3:(pos >> 3) + 4], "little") >> (pos & 7)) & 0x7FFF]
        if e is None or pos > 8 * len(z):
            raise WalkError("no code")
        pos += e[1]
        return e

    prev_huff_end = None
    final = 0
    while not final:
        if pos > 8 * len(z):
            raise WalkError("past the end")
        final, btype = bits(1), bits(2)
        start = len(out)
        if btype == 0:
            if prev_huff_end is not None:
                seen["stored after bit %d" % (prev_huff_end & 7)] += 1
            pos = (pos + 7) & ~7
            n, nn = struct.unpack("<HH", buf[pos >> 3:(pos >> 3) + 4])
            if n != nn ^ 0xFFFF and "nlen" not in lax:
                raise WalkError("nlen")
            q = (pos >> 3) + 4
            out += buf[q:q + n]
            pos = 8 * (q + n)
            seen["stored"] += 1
            seen["stored end mod4 %d" % ((q + n) & 3)] += 1
            seen["stored len %s" % {0: "0", 1: "1", 65535: "65535"}.get(n, "other")] += 1
            stored.append((start, start + n))
            prev_huff_end = None
            continue
        if btype == 3:
            raise WalkError("type 3")
        if btype == 1:
            lit, dist = FIXED_LIT, [5] * 32
            seen["fixed"] += 1
        else:
            seen["dynamic"] += 1
            hlit, hdist, hclen = bits(5) + 257, bits(5) + 1, bits(4) + 4
            seen["hlit %d" % hlit] += 1
            seen["hdist %d" % hdist] += 1
            seen["hclen %d" % hclen] += 1
            if (hlit > 286 or hdist > 30) and "fields" not in lax:
                raise WalkError("HLIT / HDIST")
            cl = [0] * 19
            for s in CL_ORDER[:hclen]:
                cl[s] = bits(3)
            if hclen == 19 and cl[CL_ORDER[18]] == 0:
                seen["hclen 19 trailing zero"] += 1
            left = kraft_left(cl)
            if left < 0 or left > 0 and "incomplete CL" not in lax:
                raise WalkError("CL code")
            ct = decode_table(cl)
            lens = []
            while len(lens) < hlit + hdist:
                s, _ = sym(ct)
                k = len(lens)
                if s < 16:
                    lens.append(s)
                    continue
                rep = bits(2) + 3 if s == 16 else bits(3) + 3 if s == 17 else bits(7) + 11
                if s == 16 and k == 0 and "16 first" not in lax:
                    raise WalkError("16 first")
                if k + rep > hlit + hdist:
                    if "repeat past" not in lax:
                        raise WalkError("repeat past the end")
                    rep = hlit + hdist - k
                seen["cl %d" % s] += 1
                if s == 18 and rep == 138:
                    seen["cl 18 x138"] += 1
                if s == 16 and k == hlit:
                    seen["16 from last lit/len length"] += 1
                if k < hlit < k + rep:
                    seen["%d across lit/dist" % s] += 1
                lens += [lens[-1] if s == 16 and k else 0] * rep
            lit, dist = lens[:hlit], lens[hlit:]
            if lit[256] == 0:
                raise WalkError("no end-of-block code")
            check_tree(lit, "lit/len", lax)
            check_tree(dist, "distance", lax)
            nz = [l for l in lit if l]
            if nz == [1] and lit[256] == 1:
                seen["eob alone"] += 1
            dz = [l for l in dist if l]
            if not dz:
                seen["no distance codes"] += 1
            elif dz == [1]:
                seen["single 1-bit distance code"] += 1
        lt, dtab = decode_table(lit), decode_table(dist)
        used = set()
        while True:
            s, l = sym(lt)
            used.add(s)
            seen["code %d bits" % l] += 1
            if s < 256:
                out.append(s)
                continue
            if s == 256:
                break
            if s > 285:
                raise WalkError("lit/len %d" % s)
            n = LEN_BASE[s - 257] + bits(LEN_XBITS[s - 257])
            if n == 258:
                seen["length 258 as %d" % s] += 1
            ds, l = sym(dtab)
            seen["code %d bits" % l] += 1
            if ds > 29:
                raise WalkError("distance %d" % ds)
            d = dg.DIST_BASE[ds] + bits(dg.DIST_XBITS[ds])
            o = len(out)
            if d > o and "distance" not in lax:
                raise WalkError("distance too far")
            if d <= 4 and d < n:
                seen["distance %d overlapping" % d] += 1
            if d == 32768:
                seen["distance 32768"] += 1
            if d == o:
                seen["distance to byte 0"] += 1
            i = bisect_right(stored, (o - d, 1 << 62)) - 1
            if i >= 0 and stored[i][0] <= o - d < stored[i][1] or i + 1 < len(stored) and stored[i + 1][0] < o - d + n:
                seen["match into a stored block"] += 1
            for j in range(n):
                out.append(out[o - d + j] if o - d + j >= 0 else 0)
        if len(out) == start:
            seen["empty %s" % ("fixed" if btype == 1 else "dynamic")] += 1
        if btype == 2 and any(l and s not in used for s, l in enumerate(lit)):
            seen["unused symbol coded"] += 1
        prev_huff_end = pos
    if pos > 8 * len(z):
        raise WalkError("past the end")
    return bytes(out), seen


# every construct the corpus must contain.  HCLEN 4 is not among them: with code-length symbols 16, 17, 18 and 0 alone no lit/len
# length is nonzero, so no valid block has it (the invalid streams do not need it either: zlib and the kernel read HCLEN alike)
REQUIRED = (["stored", "fixed", "dynamic", "empty fixed", "empty dynamic", "stored len 0", "stored len 1", "stored len 65535",
             "stored len other", "code 10 bits", "code 11 bits", "code 15 bits", "unused symbol coded", "hlit 257", "hlit 286",
             "hdist 1", "hdist 30", "hclen 19 trailing zero", "cl 16", "cl 17", "cl 18", "cl 18 x138", "16 from last lit/len length",
             "16 across lit/dist", "17 across lit/dist", "18 across lit/dist", "single 1-bit distance code", "no distance codes",
             "eob alone", "distance 1 overlapping", "distance 2 overlapping", "distance 3 overlapping", "distance 4 overlapping",
             "distance 32768", "distance to byte 0", "match into a stored block", "length 258 as 285", "length 258 as 284"]
            + ["stored after bit %d" % b for b in range(8)] + ["stored end mod4 %d" % m for m in range(4)]
            + ["hclen %d" % h for h in range(5, 20)])


@pytest.fixture(scope="module")
def walked():
    """(Stream, walk) of the decoded corpora (the GPU test decodes these streams as they are), then of the fuzz bases"""
    streams = [s for *_, s in dg.corpus()] + [s for *_, s in dg.ext_corpus()] + [s for *_, s in dg.fuzz_bases()]
    return [(s, walk(s.z)) for s in streams]


def decoded(walked):
    return walked[:len(dg.corpus()) + len(dg.ext_corpus())]


def test_valid_streams_inflate_to_their_input(walked):
    for raw, s in [(x[3], x[4]) for x in dg.corpus() + dg.fuzz_bases()] + [(x[5], x[6]) for x in dg.ext_corpus()]:
        assert zlib.decompress(s.z) == raw
        assert dg.expect(s.z, len(raw)) == (raw, "ok")
    for (s, (out, _)) in walked:
        assert out == zlib.decompress(s.z)


def test_corpus_covers_every_construct(walked):
    """counted over the streams the GPU test decodes with a pixel check; the fuzz bases reach it only through mutants"""
    walked = decoded(walked)
    seen = Counter()
    for _, (_, c) in walked:
        seen += c
    missing = [k for k in REQUIRED if not seen[k]]
    assert not missing, missing
    assert len({k for k in seen if k.startswith("hlit ")}) >= 10 and len({k for k in seen if k.startswith("hdist ")}) >= 10
    # what the writer says it did, the walker finds
    tags = Counter(t for s, _ in walked for t in s.tags)
    assert tags["stored"] == seen["stored"]
    assert seen["16 from last lit/len length"] + seen["16 across lit/dist"] >= tags["cross16"] > 0
    assert seen["eob alone"] >= tags["eob alone"] > 0


def test_block_plan_offsets(walked):
    """Stream.blocks points at each block's header and each stored block's LEN (the mutation fuzz edits them)"""
    for s, _ in walked:
        for t, at, ln in s.blocks:
            assert int.from_bytes(s.z[at >> 3:(at >> 3) + 2], "little") >> (at & 7) >> 1 & 3 == t
            if t == 0:
                n, nn = struct.unpack("<HH", s.z[ln:ln + 4])
                assert n == nn ^ 0xFFFF


def invalid_cases():
    """(name, stream, raw): the invalid streams of the GPU test, 8-bit and ext"""
    out = []
    for k, (w, h, c, raw, _) in enumerate(dg.corpus()[3:7]):
        out += [(name, z, raw) for name, z in dg.invalid_streams(raw, 50 + k).items()]
    for k, x in enumerate([dg.ext_corpus()[i] for i in (0, 1, 3, 5)]):
        out += [(name, z, x[5]) for name, z in dg.invalid_streams(x[5], 60 + k).items()]
    return out


INVALID_NAMES = ["oversubscribed lit/len code", "oversubscribed distance code", "oversubscribed CL code", "incomplete CL code",
                 "incomplete CL code, one 1-bit code", "incomplete lit/len code", "incomplete distance code", "no end-of-block code",
                 "HLIT field 30", "HLIT field 31", "HDIST field 30", "HDIST field 31", "16 repeat first", "repeat past HLIT + HDIST",
                 "fixed lit/len 286", "fixed lit/len 287", "fixed distance 30", "fixed distance 31", "distance one past the output",
                 "stored NLEN mismatch", "stored length past the end", "block type 3 after a good block", "no final block",
                 "truncated inside a symbol", "one byte short", "one byte long"]


def test_zlib_rejects_every_named_invalid_stream():
    cases = invalid_cases()
    assert sorted({n for n, _, _ in cases}) == sorted(INVALID_NAMES)
    for name, z, raw in cases:
        n_raw = len(raw)
        assert dg.expect(z, n_raw) is None, name
        with pytest.raises(zlib.error):
            r = zlib.decompress(z)
            if len(r) != n_raw:
                raise zlib.error("length")


def test_header_model_matches_zlib():
    body = zlib.compress(b"header model body " * 5)[2:]
    for h in range(65536):
        z = struct.pack(">H", h) + body
        try:
            ok = zlib.decompress(z) is not None
        except zlib.error:
            ok = False
        assert dg.header_ok(z) == ok, hex(h)


def test_expect_adler_verdicts():
    raw = bytes(range(256)) * 3
    z = dg.write(raw, 1).z
    assert dg.expect(z, len(raw)) == (raw, "ok")
    assert dg.expect(z[:-1] + bytes([z[-1] ^ 1]), len(raw)) == (raw, "bad")
    assert dg.expect(z[:-1], len(raw)) == (raw, "missing")
    assert dg.expect(z, len(raw) + 1) is None and dg.expect(z, len(raw) - 1) is None


# the rule each named stream breaks, where a decoder without it has an obvious reading.  The others have none: an over-subscribed
# code, a missing EOB, a one-code CL code (it can send one length value only), lit/len 286 / 287, distance 30 / 31, block type 3,
# a stored length or a symbol past the end, no final block, a wrong output length.
ONE_RULE = {"HLIT field 30": "fields", "HLIT field 31": "fields", "HDIST field 30": "fields", "HDIST field 31": "fields",
            "incomplete CL code": "incomplete CL", "incomplete lit/len code": "incomplete", "incomplete distance code": "incomplete",
            "16 repeat first": "16 first", "repeat past HLIT + HDIST": "repeat past", "stored NLEN mismatch": "nlen",
            "distance one past the output": "distance"}


def test_each_invalid_stream_breaks_one_rule():
    """without its one rule each stream inflates to the full output, so a decoder that dropped only that rule would be caught: the
    stream is not also rejected for a second reason (a short output, another bad tree)"""
    for name, z, raw in invalid_cases():
        rule = ONE_RULE.get(name)
        if rule is None:
            continue
        with pytest.raises(WalkError):
            walk(z)
        out, _ = walk(z, lax={rule})
        assert len(out) == len(raw), name
        if rule != "distance":                                          # that one reads a 0 for the byte before the start
            assert out == raw, name
