"""Test-only writer of hand-built fpng files, from the Deflate (RFC 1951), zlib (RFC 1950) and PNG specifications.

An fpng file is a PNG whose IDAT holds one zlib stream; the decoders accept more shapes of that stream than any encoder
writes: other code-length tables, HLIT / HDIST / HCLEN values, one or two 1-bit distance codes, code-length runs across the
literal / distance boundary, any length symbol.  `dynamic_file` writes such a file from explicit code sizes, a code-length
run-length choice and a token list; `stored_file` writes stored blocks of any size.  `cases()` is the corpus the CPU test
(oracle vs the reference decoder, zlib.decompress as an independent check of this writer) and the GPU test share.
"""
from __future__ import annotations

import struct
import zlib

import numpy as np

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_XBITS = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]     # RFC 1951 3.2.7
EOB = 256


class BitWriter:
    """Deflate bit order: fields least significant bit first, Huffman codes most significant bit first"""

    def __init__(self):
        self.v, self.n = 0, 0

    def bits(self, value: int, count: int) -> None:
        self.v |= (value & ((1 << count) - 1)) << self.n
        self.n += count

    def code(self, code: int, length: int) -> None:
        assert length > 0, "symbol without a code"
        self.bits(int(format(code, "0%db" % length)[::-1], 2), length)

    def tobytes(self) -> bytes:
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical_codes(sizes):
    """RFC 1951 3.2.2: code of every symbol from the code sizes"""
    count = [0] * 17
    for s in sizes:
        count[s] += 1
    count[0] = 0
    nxt, code = [0] * 17, 0
    for bits in range(1, 17):
        code = (code + count[bits - 1]) << 1
        nxt[bits] = code
    codes = [0] * len(sizes)
    for i, s in enumerate(sizes):
        if s:
            codes[i] = nxt[s]
            nxt[s] += 1
    return codes


def kraft(sizes) -> float:
    return sum(2.0 ** -s for s in sizes if s)


def length_symbol(n: int):
    """(symbol, extra bit count, extra value) of match length n (3..258)"""
    if n == 258:
        return 285, 0, 0
    for i in range(28):
        if LEN_BASE[i] <= n < LEN_BASE[i] + (1 << LEN_XBITS[i]):
            return 257 + i, LEN_XBITS[i], n - LEN_BASE[i]
    raise ValueError(n)


def flat_sizes(n: int):
    """sizes of a complete code of n >= 2 symbols whose lengths differ by at most one (near fixed length)"""
    k = (n - 1).bit_length()
    short = (1 << k) - n
    return [k - 1] * short + [k] * (n - short)


def fill_sizes(sizes, fillers, spread=False, max_len=12):
    """gives symbols of `fillers` (in order) the code sizes that make `sizes` a complete code and returns `sizes`: as few
    fillers as possible at the shortest lengths, or (spread) as many as possible at the longest"""
    unit = 1 << max_len
    left = unit - sum(unit >> s for s in sizes if s)
    assert left >= 0
    fillers = list(fillers)
    while left:
        r = len(fillers) - 1
        assert r >= 0, "not enough filler symbols"
        c = 1 << (left.bit_length() - 1)
        if spread:
            c = 1
            while bin(left - c).count("1") > r:
                c <<= 1
        sizes[fillers.pop(0)] = max_len - (c.bit_length() - 1)
        left -= c
    return sizes


def code_length_tokens(seq, mode: str):
    """the code-length alphabet sequence (symbol, extra bits, extra value) for code sizes `seq` (RFC 1951 3.2.7):
    mode "plain" sends every size as itself, "rle" uses 16 / 17 / 18 runs over the whole sequence"""
    if mode == "plain":
        return [(s, 0, 0) for s in seq]
    out, i = [], 0
    while i < len(seq):
        v, j = seq[i], i
        while j < len(seq) and seq[j] == v:
            j += 1
        run = j - i
        if v == 0 and run >= 3:
            while run >= 11:
                k = min(run, 138); out.append((18, 7, k - 11)); run -= k
            if run >= 3:
                out.append((17, 3, run - 3)); run = 0
            out += [(0, 0, 0)] * run
        elif v != 0 and run >= 4:
            out.append((v, 0, 0)); run -= 1
            while run >= 3:
                k = min(run, 6); out.append((16, 2, k - 3)); run -= k
            out += [(v, 0, 0)] * run
        else:
            out += [(v, 0, 0)] * run
        i = j
    return out


def filtered_stream(tokens, chans: int, dist: int | None = None) -> bytes | None:
    """what a Deflate decoder makes of the token list (matches copy from `dist` = chans bytes back); None when a match reaches
    before the start of the stream"""
    out = bytearray()
    d = dist or chans
    for t in tokens:
        if t[0] == "L":
            out.append(t[1])
        elif t[0] == "M":
            if len(out) < d:
                return None
            for _ in range(t[1]):
                out.append(out[-d])
        else:
            break
    return bytes(out)


def dynamic_block(lit_sizes, dist_sizes, tokens, chans: int, rle: str = "rle", hclen: int | None = None, single_cl: bool = False,
                  dist_sym: int | None = None, offsets: bool = False):
    """one final dynamic Huffman block (BFINAL = 1, BTYPE = 2) holding `tokens`: ("L", byte), ("M", length), ("E",).
    hclen: code-length code sizes sent (default: as few as the table needs, at least 4; fewer than needed truncates the
    table).  single_cl: the code-length code has one code word (all sizes must then be one code-length symbol).
    offsets: return (block, [bit offset of each token from the block's first bit]) instead of the block alone."""
    nlit, ndist = len(lit_sizes), len(dist_sizes)
    cl_toks = code_length_tokens(list(lit_sizes) + list(dist_sizes), rle)
    used = sorted({s for s, _, _ in cl_toks})
    cl_sizes = [0] * 19
    if single_cl:
        assert len(used) == 1
        cl_sizes[used[0]] = 1
    else:
        for s, l in zip(used, flat_sizes(max(len(used), 2))):
            cl_sizes[s] = l
    need = max(i + 1 for i in range(19) if cl_sizes[CL_ORDER[i]]) if any(cl_sizes) else 4
    ncl = max(need, 4) if hclen is None else hclen
    cl_codes = canonical_codes(cl_sizes)
    lit_codes, dist_codes = canonical_codes(lit_sizes), canonical_codes(dist_sizes)
    ds = chans - 1 if dist_sym is None else dist_sym
    bw = BitWriter()
    bw.bits(1, 1); bw.bits(2, 2)
    bw.bits(nlit - 257, 5); bw.bits(ndist - 1, 5); bw.bits(ncl - 4, 4)
    for i in range(ncl):
        bw.bits(cl_sizes[CL_ORDER[i]], 3)
    for s, xb, xv in cl_toks:
        bw.code(cl_codes[s], cl_sizes[s])
        if xb:
            bw.bits(xv, xb)
    at = []
    for t in tokens:
        at.append(bw.n)
        if t[0] == "L":
            bw.code(lit_codes[t[1]], lit_sizes[t[1]])
        elif t[0] == "M":
            sym, xb, xv = length_symbol(t[1])
            bw.code(lit_codes[sym], lit_sizes[sym])
            if xb:
                bw.bits(xv, xb)
            bw.code(dist_codes[ds], dist_sizes[ds])                        # distance symbol chans - 1 = distance chans, no extra bits
        else:
            bw.code(lit_codes[EOB], lit_sizes[EOB])
    return (bw.tobytes(), at) if offsets else bw.tobytes()


def _chunk(tag: bytes, body: bytes) -> bytes:
    return struct.pack(">I", len(body)) + tag + body + struct.pack(">I", zlib.crc32(tag + body) & 0xFFFFFFFF)


def png_file(w: int, h: int, chans: int, zstream: bytes) -> bytes:
    """signature, IHDR (8-bit RGB / RGBA), fdEC (fpng's marker chunk), one IDAT, IEND"""
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 2 if chans == 3 else 6, 0, 0, 0)
    return (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", ihdr) + _chunk(b"fdEC", bytes([82, 36, 147, 227, 0])) + _chunk(b"IDAT", zstream)
            + _chunk(b"IEND", b""))


def zlib_stream(deflate: bytes, data: bytes) -> bytes:
    """zlib header (deflate, 32 KiB window, no dictionary, fastest level: 0x78 0x01), the blocks, Adler-32 of the data"""
    return b"\x78\x01" + deflate + struct.pack(">I", zlib.adler32(data) & 0xFFFFFFFF)


def dynamic_file(w, h, chans, lit_sizes, dist_sizes, tokens, trailing: bytes = b"", offsets: bool = False, **kw):
    """-> (file, the filtered stream a Deflate decoder produces or None); offsets: (file, stream, [bit offset of each token from
    the zlib stream's first bit])"""
    data = filtered_stream(tokens, chans, kw.get("dist_sym", chans - 1) + 1)
    blk, at = dynamic_block(lit_sizes, dist_sizes, tokens, chans, offsets=True, **kw)
    f = png_file(w, h, chans, zlib_stream(blk + trailing, data or b""))
    return (f, data, [16 + a for a in at]) if offsets else (f, data)


def stored_file(w, h, chans, data: bytes, block: int):
    """stored blocks of `block` bytes (the last one shorter)"""
    out = bytearray()
    for i in range(0, max(len(data), 1), block):
        part = data[i:i + block]
        out.append(1 if i + block >= len(data) else 0)
        out += struct.pack("<HH", len(part), len(part) ^ 0xFFFF) + part
    return png_file(w, h, chans, zlib_stream(bytes(out), data)), data


# ------------------------------------------------------------------------------------------------------------------------------
# the corpus
# ------------------------------------------------------------------------------------------------------------------------------
def image_tokens(w, h, chans, lits, rs, run_lengths=(), match_rate=0.3, filters=None):
    """tokens of an h-row image in fpng's grammar, EOB at the end: a filter byte per scanline (0 on the first, 2 below unless
    `filters`), pixels of `chans` literals drawn from `lits`, after a pixel matches that repeat it (lengths from `run_lengths`
    in turn, multiples of chans, where they fit)"""
    toks, bpl, runs = [], w * chans, list(run_lengths)
    for y in range(h):
        toks.append(("L", filters[y] if filters else (2 if y else 0)))
        x = 0
        while x < bpl:
            if x and runs and rs.rand() < match_rate and x + runs[0] <= bpl:
                toks.append(("M", runs[0])); x += runs[0]
                runs.append(runs.pop(0))
                continue
            toks += [("L", int(v)) for v in rs.choice(lits, chans)]
            x += chans
    return toks + [("E",)]


def scanlines(tokens, bpl):
    """image_tokens' list without its EOB as one token list per scanline (filter byte first)"""
    rows, i, body = [], 0, tokens[:-1]
    while i < len(body):
        row, n = [body[i]], 0
        i += 1
        while n < bpl:
            t = body[i]
            n += 1 if t[0] == "L" else t[1]
            row.append(t); i += 1
        rows.append(row)
    return rows


def coded_runs(lit_sizes, runs):
    return [n for n in runs if length_symbol(n)[0] < len(lit_sizes) and lit_sizes[length_symbol(n)[0]]]


def fpng_dist(chans, two=False, ndist=None):
    """fpng's distance code: one 1-bit code for distance chans (symbol chans - 1), optionally a second one at symbol chans"""
    d = [0] * (ndist or (chans + 1 if two else chans))
    d[chans - 1] = 1
    if two:
        d[chans] = 1
    return d


def hclen_needed(lit_sizes, dist_sizes, rle="rle"):
    used = {s for s, _, _ in code_length_tokens(list(lit_sizes) + list(dist_sizes), rle)}
    return max(4, max(i + 1 for i in range(19) if CL_ORDER[i] in used))


def cases():
    """[(name, file, chans, deflate_ok, deviation, filtered stream)]: deflate_ok = valid Deflate, zlib.decompress must return the
    filtered stream; deviation = the GPU decoder rejects the file by design where the reference accepts it (INTEGRATION.md
    section 7).  Everything else is expected to decode exactly as the reference decodes it, success or not."""
    out = []
    rs = np.random.RandomState(11)

    def add(name, chans, made, ok=True, deviation=False):
        out.append((name, made[0], chans, ok, deviation, made[1]))

    for chans in (3, 4):
        w, h = 96, 24
        bpl = w * chans
        runs = [n for n in range(3, 259) if n % chans == 0 and n <= bpl - chans]
        fd = fpng_dist(chans)
        # ---- tables
        # near-fixed-length complete code over every literal, EOB and every length symbol (8 and 9 bits): slowest to resynchronise
        flat = flat_sizes(286)
        toks = image_tokens(w, h, chans, np.arange(256), rs, runs)
        lit_toks = image_tokens(w, h, chans, np.arange(256), rs)
        add(f"flat286_c{chans}", chans, dynamic_file(w, h, chans, flat, fd, toks))
        add(f"flat286_plain_c{chans}", chans, dynamic_file(w, h, chans, flat, fd, toks, rle="plain"))
        add(f"flat286_two_dist_c{chans}", chans, dynamic_file(w, h, chans, flat, fpng_dist(chans, True), toks))
        # maximally skewed: sizes 1..7 (a 1-bit literal), then 32 codes of 12 bits (EOB, every length symbol, filters 0 and 2)
        lit = [0] * 286
        order = [7, 1, 250, 3, 130, 5, 66]
        for i, s in enumerate(order):
            lit[s] = i + 1
        fill_sizes(lit, [EOB] + [257 + i for i in range(29)] + [s for s in range(256) if s not in order], spread=True)
        assert kraft(lit) == 1.0 and lit.count(12) == 32 and lit[0] == lit[2] == lit[285] == 12
        coded = [s for s in range(256) if lit[s]]
        add(f"skewed12_c{chans}", chans, dynamic_file(w, h, chans, lit, fd, image_tokens(w, h, chans, coded, rs, coded_runs(lit, runs), 0.5)))
        # filter symbols 0 and 2 at 12 bits
        lit = [0] * 286
        for s in range(3, 200):
            lit[s] = 8
        lit[0] = lit[2] = 12
        fill_sizes(lit, [EOB] + [257 + i for i in range(29)] + list(range(200, 256)) + [1], spread=True)
        assert lit[0] == lit[2] == 12 and kraft(lit) == 1.0
        coded = [s for s in range(256) if lit[s]]
        add(f"filters12_c{chans}", chans, dynamic_file(w, h, chans, lit, fd, image_tokens(w, h, chans, coded, rs, coded_runs(lit, runs))))
        # HLIT 257 (no length symbols), 286 and 288 with trailing zero sizes (288: not Deflate)
        lit = flat_sizes(257)
        add(f"hlit257_c{chans}", chans, dynamic_file(w, h, chans, lit, fd, lit_toks))
        add(f"hlit286_zeros_c{chans}", chans, dynamic_file(w, h, chans, lit + [0] * 29, fd, lit_toks))
        add(f"hlit288_zeros_c{chans}", chans, dynamic_file(w, h, chans, lit + [0] * 31, fd, lit_toks), ok=False)
        # HDIST 1..32 (31, 32: not Deflate) with one and two fpng distance codes where they fit; below chans the table has a
        # valid Deflate distance code but not fpng's
        for nd in range(1, 33):
            for two in (False, True):
                if two and nd < chans + 1:
                    continue
                if nd >= chans:
                    add(f"hdist{nd}{'_two' if two else ''}_c{chans}", chans, dynamic_file(w, h, chans, flat, fpng_dist(chans, two, nd), toks), ok=nd <= 30)
                else:
                    d = [0] * nd
                    d[0] = 1
                    add(f"hdist{nd}_c{chans}", chans, dynamic_file(w, h, chans, flat, d, lit_toks))
        # one 1-bit distance code plus longer ones (a complete distance code; the decoders read one bit per match)
        d = [0] * 8
        d[chans - 1] = 1
        for j, l in zip([x for x in range(8) if x != chans - 1], [2, 3, 3]):
            d[j] = l
        add(f"dist_1_2_3_3_c{chans}", chans, dynamic_file(w, h, chans, flat, d, toks))
        # the 1-bit code at the wrong symbol (fpng's distance code missing), three 1-bit codes (over-subscribed)
        d = [0] * 6
        d[chans] = 1
        add(f"dist_missing_c{chans}", chans, dynamic_file(w, h, chans, flat, d, lit_toks))
        d = [0] * 6
        d[chans - 2] = d[chans - 1] = d[chans] = 1
        add(f"dist_three_c{chans}", chans, dynamic_file(w, h, chans, flat, d, toks), ok=False)
        # code-length runs across the literal / distance boundary: zeros (18), and a repeat (16) of the last literal size
        lit = flat_sizes(264) + [0] * 22
        add(f"cross_zero_run_c{chans}", chans, dynamic_file(w, h, chans, lit, fpng_dist(chans, ndist=10),
                                                            image_tokens(w, h, chans, np.arange(256), rs, coded_runs(lit, runs))))
        d = [flat[-1]] * 6
        d[chans - 1] = 1
        add(f"cross_repeat_run_c{chans}", chans, dynamic_file(w, h, chans, flat, d, lit_toks), ok=False)
        # HCLEN 4..19: fewer code-length sizes than the table needs truncate it
        need = hclen_needed(flat, fd)
        for hc in range(4, 20):
            add(f"hclen{hc}_c{chans}", chans, dynamic_file(w, h, chans, flat, fd, toks, hclen=hc), ok=hc >= need)
        # a code-length code with a single code word (every size is the same symbol)
        add(f"single_cl_zeros_c{chans}", chans, dynamic_file(w, h, chans, [0] * 257, [0] * chans, [], rle="plain", single_cl=True), ok=False)
        add(f"single_cl_nines_c{chans}", chans, dynamic_file(w, h, chans, [9] * 257, [9] * chans, [], rle="plain", single_cl=True), ok=False)
        # invalid literal tables: over- and under-subscribed, a size over 12 (still Deflate: one 9-bit code split down to 13 bits)
        add(f"over_subscribed_c{chans}", chans, dynamic_file(w, h, chans, flat + [9], fd, toks), ok=False)
        under = list(flat)
        under[100] = 0
        add(f"under_subscribed_c{chans}", chans, dynamic_file(w, h, chans, under, fd, [t for t in toks if t != ("L", 100)]), ok=False)
        lit = flat_sizes(282) + [0] * 4
        assert lit[281] == 9
        lit[281:286] = [10, 11, 12, 13, 13]
        assert kraft(lit) == 1.0
        add(f"size13_c{chans}", chans, dynamic_file(w, h, chans, lit, fd, image_tokens(w, h, chans, np.arange(256), rs, coded_runs(lit[:281], runs))))
        # ---- tokens
        # every length symbol that gives a multiple of chans (258 = symbol 285 for RGB)
        every = [n for n in range(3, 259) if n % chans == 0]
        t = image_tokens(120, 80, chans, np.arange(256), rs, every, match_rate=0.6)
        assert {x[1] for x in t if x[0] == "M"} == set(every)
        add(f"every_length_c{chans}", chans, dynamic_file(120, 80, chans, flat, fd, t))
        base = image_tokens(w, 8, chans, np.arange(256), rs, runs)
        rows = scanlines(base, bpl)

        def edit(fn):
            r = [list(x) for x in rows]
            fn(r)
            return [t for row in r for t in row] + [("E",)]

        def cross(row):                                                     # the last pixel becomes a two-pixel match
            del row[-chans:]
            row.append(("M", 2 * chans))

        def first_pixel_match(row):                                         # the scanline's first pixel becomes a match
            del row[1:1 + chans]
            row.insert(1, ("M", chans))

        add(f"length_not_multiple_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: r[2].insert(1 + chans, ("M", chans + 1)))))
        add(f"match_crosses_scanline_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: cross(r[3]))))
        add(f"match_not_pixel_aligned_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: r[5].insert(2, ("M", chans)))))
        add(f"wrong_filter_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: r[4].__setitem__(0, ("L", 1)))))
        add(f"first_filter_up_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: r[0].__setitem__(0, ("L", 2)))))
        add(f"eob_early_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: r[7].__delitem__(slice(-chans, None)))))
        add(f"eob_late_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: r[7].extend([("L", 9)] * chans))))
        add(f"eob_missing_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, base[:-1]), ok=False)
        add(f"bytes_after_eob_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, base, trailing=b"\x00\x00"), ok=False)
        # documented deviations: a scanline that starts with a match (the reference repeats a zero pixel there), stored blocks
        # in another layout than the reference writer's 65535-byte blocks
        add(f"row_starts_with_match_c{chans}", chans, dynamic_file(w, 8, chans, flat, fd, edit(lambda r: first_pixel_match(r[3]))), deviation=True)
        raw = b"".join(b"\x00" + rs.randint(0, 256, bpl).astype(np.uint8).tobytes() for _ in range(12))
        add(f"stored_1000_byte_blocks_c{chans}", chans, stored_file(w, 12, chans, raw, 1000), deviation=True)
    return out
