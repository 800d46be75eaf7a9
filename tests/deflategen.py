"""Seeded Deflate (RFC 1951) writer with an explicit block plan, for the differential tests of the any-PNG inflate
(png_inflate_kernel).  zlib only ever writes a small part of what Deflate allows; this writer mixes stored, fixed and dynamic
blocks (empty ones included), builds random complete and length-limited codes up to 15 bits, runs the code-length RLE across the
literal / distance boundary, and parses matches over any earlier occurrence, distance 32768 and distance = bytes so far included.
`invalid_streams` writes named streams a decoder must reject.  The expected result of any stream, valid or not, comes from zlib
(`expect`), never from this writer; test_deflategen_cpu.py walks the streams to count the constructs they contain."""
from __future__ import annotations

import functools
import random
import struct
import zlib
from collections import Counter, namedtuple

from streamgen import CL_ORDER, canonical_codes, length_symbol

DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577]
DIST_XBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32
EOB = 256

# match length -> (symbol, extra bits, extra value); distance -> (symbol, extra bits, extra value)
LSYM = [None] * 3 + [length_symbol(n) for n in range(3, 259)]
DSYM = [None]
for _i, (_b, _x) in enumerate(zip(DIST_BASE, DIST_XBITS)):
    DSYM += [(_i, _x, v) for v in range(1 << _x)]

Stream = namedtuple("Stream", "z tags blocks")   # blocks: [(type, bit offset of BFINAL in z, byte offset of LEN for stored or -1)]


def rev(code: int, n: int) -> int:
    return int(format(code, "0%db" % n)[::-1], 2) if n else 0


class BitWriter:
    """Deflate bit order into a bytearray: linear in the stream length (fields LSB first; Huffman codes are pre-reversed)"""

    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def bits(self, v: int, n: int) -> None:
        self.acc |= v << self.n
        self.n += n
        if self.n >= 32:
            self.out += (self.acc & 0xFFFFFFFF).to_bytes(4, "little")
            self.acc >>= 32
            self.n -= 32

    def pos(self) -> int:
        return 8 * len(self.out) + self.n

    def align(self) -> None:
        self.bits(0, -self.n & 7)
        self.out += self.acc.to_bytes(self.n // 8, "little")
        self.acc, self.n = 0, 0

    def raw(self, data) -> None:
        self.align()
        self.out += data

    def getvalue(self) -> bytes:
        return bytes(self.out) + self.acc.to_bytes((self.n + 7) // 8, "little")


def table(lens):
    """[(reversed code, length)] per symbol (oversubscribed lengths still get codes, for the invalid streams)"""
    return [(rev(c & ((1 << l) - 1), l), l) for c, l in zip(canonical_codes(lens), lens)]


# ---- codes --------------------------------------------------------------------------------------------------------------------
def random_complete(rng, n: int, top: int):
    """n code lengths of a random complete code whose longest code has exactly `top` bits (top + 1 <= n <= 2 ** top)"""
    cnt = [0] * (top + 1)
    for l in range(1, top):
        cnt[l] = 1
    cnt[top] = 2
    for _ in range(n - top - 1):
        l = rng.choice([l for l in range(1, top) if cnt[l]])
        cnt[l] -= 1
        cnt[l + 1] += 2
    out = [l for l in range(1, top + 1) for _ in range(cnt[l])]
    rng.shuffle(out)
    return out


def limited_huffman(freqs, limit: int):
    """{symbol: length}: Huffman code lengths of freqs {symbol: count > 0}, limited to `limit` bits (miniz's count fix-up)"""
    syms = sorted(freqs, key=lambda s: (-freqs[s], s))
    if len(syms) == 1:
        return {syms[0]: 1}
    import heapq
    heap = [(freqs[s], i, [s]) for i, s in enumerate(syms)]
    heapq.heapify(heap)
    depth = dict.fromkeys(syms, 0)
    k = len(heap)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(heap, (f1 + f2, k, a + b))
        k += 1
    cnt = [0] * (max(limit, max(depth.values())) + 1)
    for s in syms:
        cnt[min(depth[s], limit)] += 1
    total = sum(cnt[l] << (limit - l) for l in range(1, limit + 1))
    while total > 1 << limit:
        cnt[limit] -= 1
        for l in range(limit - 1, 0, -1):
            if cnt[l]:
                cnt[l] -= 1
                cnt[l + 1] += 2
                break
        total -= 1
    lens = [l for l in range(1, limit + 1) for _ in range(cnt[l])]
    return dict(zip(syms, lens))


def make_code(rng, used: Counter, alphabet: int, tags, kind: str):
    """code lengths [alphabet] covering every used symbol: random complete (longest code 10, 11, 15 or any) or length-limited
    Huffman of the counts, some unused symbols coded as well"""
    lens = [0] * alphabet
    free = [s for s in range(alphabet) if s not in used]
    extra = rng.sample(free, rng.randint(0, min(len(free), 40))) if rng.random() < 0.5 else []
    if extra:
        tags.append(kind + " unused coded")
    syms = list(used) + extra
    if rng.random() < 0.5:
        top = rng.choice([10, 11, 15, 15, rng.randint(1, 15)])
        top = max(top, (len(syms) - 1).bit_length(), 1)
        need = top + 1 - len(syms)
        if need > 0:
            if need > len(free) - len(extra):
                top = len(syms) - 1 if len(syms) > 1 else 1
                need = top + 1 - len(syms)
            more = rng.sample([s for s in free if s not in extra], max(0, need))
            syms += more
        for s, l in zip(syms, random_complete(rng, len(syms), top)):
            lens[s] = l
    else:
        f = dict(used)
        f.update({s: 1 for s in extra})
        if len(f) == 1:
            f[rng.choice(free)] = 1
        limit = rng.choice([15, 15, 12, 11, 10, 9])
        limit = max(limit, (len(f) - 1).bit_length())
        for s, l in limited_huffman(f, limit).items():
            lens[s] = l
    return lens


def cl_tokens(rng, seq, mode: str):
    """code-length alphabet tokens (symbol, extra bits, extra value) of seq: "plain", or RLE with random run splits"""
    if mode == "plain":
        return [(s, 0, 0) for s in seq]
    out, i = [], 0
    while i < len(seq):
        v, j = seq[i], i
        while j < len(seq) and seq[j] == v:
            j += 1
        run = j - i
        if v == 0 and run >= 3:
            while run >= 3:
                k = min(run, 138 if rng.random() < 0.7 else rng.randint(3, 138))
                if k >= 11:
                    out.append((18, 7, k - 11))
                else:
                    out.append((17, 3, k - 3))
                run -= k
            out += [(0, 0, 0)] * run
        elif v != 0 and run >= 4:
            out.append((v, 0, 0))
            run -= 1
            while run >= 3:
                k = min(run, rng.randint(3, 6))
                out.append((16, 2, k - 3))
                run -= k
            out += [(v, 0, 0)] * run
        else:
            out += [(v, 0, 0)] * run
        i = j
    return out


def code_lengths_header(w: BitWriter, rng, lit_lens, dist_lens, tags, hlit=None, hdist=None, hclen=None, mode=None, cl_lens=None,
                        cl_toks=None):
    """HLIT, HDIST, HCLEN, the CL code and the code lengths; every field may be forced (the invalid streams)"""
    hlit = hlit if hlit is not None else len(lit_lens)
    hdist = hdist if hdist is not None else len(dist_lens)
    toks = cl_toks
    if toks is None:
        mode = mode or rng.choice(["joined", "joined", "split", "plain"])
        if mode == "split":
            toks = cl_tokens(rng, lit_lens[:hlit], "rle") + cl_tokens(rng, dist_lens[:hdist], "rle")
        else:
            toks = cl_tokens(rng, list(lit_lens[:hlit]) + list(dist_lens[:hdist]), mode)
    if cl_lens is None:
        used = Counter(t[0] for t in toks)
        cl_lens = make_code(rng, used, 19, [], "cl") if hclen is None and (len(used) > 1 or rng.random() < 0.5) else None
        if cl_lens is None or max(cl_lens) > 7:
            f = dict(used)
            if len(f) == 1:
                f[next(s for s in CL_ORDER if s not in f)] = 1
            hl = limited_huffman(f, 7)
            cl_lens = [hl.get(s, 0) for s in range(19)]
    if hclen is None:
        need = max([4] + [i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]])
        hclen = rng.randint(need, 19) if rng.random() < 0.5 else need
    w.bits(hlit - 257, 5)
    w.bits(hdist - 1, 5)
    w.bits(hclen - 4, 4)
    for s in CL_ORDER[:hclen]:
        w.bits(cl_lens[s], 3)
    ct = table(cl_lens)
    for s, nx, xv in toks:
        w.bits(*ct[s])
        if nx:
            w.bits(xv, nx)
    return toks


def huffman_block(w: BitWriter, rng, toks, final: int, btype: int, tags, lit_lens=None, dist_lens=None, **hdr):
    """a fixed (btype 1) or dynamic (2) block of toks: literal ints, (length, distance, length 258 as 284 + 31) matches"""
    lits, dists = Counter(), Counter()
    for t in toks:
        if type(t) is int:
            lits[t] += 1
        else:
            lits[284 if t[2] else LSYM[t[0]][0]] += 1
            dists[DSYM[t[1]][0]] += 1
    lits[EOB] += 1
    w.bits(final | btype << 1, 3)
    if btype == 1:
        lt, dt = table(FIXED_LIT), table(FIXED_DIST)
    else:
        crossed = False
        if hdr.pop("cross16", False):                                   # every symbol below HLIT / HDIST coded, then permuted
            hl = rng.randint(max(257, max(lits) + 1), 286)
            hd = rng.randint(max([3] + [s + 1 for s in dists]), 30)
            lit_lens = random_complete(rng, hl, rng.randint(9, 15))
            dist_lens = random_complete(rng, hd, rng.randint((hd - 1).bit_length(), min(15, hd - 1)))
            crossed = cross16(rng, lit_lens, dist_lens, hl)
            if crossed:
                tags.append("cross16")
                hdr.update(hlit=hl, hdist=hd, mode="joined")
        if lit_lens is None and not dists and rng.random() < 0.3:    # literals only: the least HCLEN a valid block can have
            hc = rng.randint(5, 10)
            lit_lens = flat_code(rng, lits, hc)
            if lit_lens is not None:
                dist_lens = [0] * 30
                hdr.update(hclen=hc, mode="joined")
                tags.append("hclen %d" % hc)
        if lit_lens is None:
            if len(lits) == 1 and rng.random() < 0.5:
                lit_lens = [0] * 256 + [1]
                tags.append("eob alone")
            else:
                lit_lens = make_code(rng, lits, 286, tags, "lit")
        if dist_lens is None:
            if not dists:
                dist_lens = [0] * 30 if rng.random() < 0.6 else make_code(rng, Counter({rng.randrange(30): 1}), 30, tags, "dist")
            elif len(dists) == 1 and rng.random() < 0.5:
                dist_lens = [0] * 30
                dist_lens[next(iter(dists))] = 1
                tags.append("dist single 1-bit")
            else:
                dist_lens = make_code(rng, dists, 30, tags, "dist")
        hlit = max([257] + [s + 1 for s, l in enumerate(lit_lens) if l])
        hdist = max([1] + [s + 1 for s, l in enumerate(dist_lens) if l])
        hlit = hdr.pop("hlit", rng.randint(hlit, 286) if rng.random() < 0.5 else hlit)
        hdist = hdr.pop("hdist", rng.randint(hdist, 30) if rng.random() < 0.5 else hdist)
        lit_lens, dist_lens = list(lit_lens) + [0] * (hlit - len(lit_lens)), list(dist_lens) + [0] * (hdist - len(dist_lens))
        code_lengths_header(w, rng, lit_lens, dist_lens, tags, hlit=hlit, hdist=hdist, **hdr)
        lt, dt = table(lit_lens[:hlit] + [0] * (288 - hlit)), table(dist_lens[:hdist] + [0] * (32 - hdist))
    bits = w.bits
    for t in toks:
        if type(t) is int:
            bits(*lt[t])
        else:
            n, d, alt = t
            if alt:
                bits(*lt[284])
                bits(31, 5)
            else:
                s, nx, xv = LSYM[n]
                bits(*lt[s])
                if nx:
                    bits(xv, nx)
            s, nx, xv = DSYM[d]
            bits(*dt[s])
            if nx:
                bits(xv, nx)
    bits(*lt[EOB])


def cross16(rng, lit_lens, dist_lens, hlit) -> bool:
    """permutes complete codes over every symbol below HLIT / HDIST so that the last lit/len length v also starts the distance
    lengths 3 times: the joined RLE then sends v and a 16 at k == HLIT, or (v twice at the end) a 16 from HLIT - 1 across HLIT"""
    for v in sorted(set(dist_lens)):
        if dist_lens.count(v) >= 3 and v in lit_lens and len(set(lit_lens)) > 1:
            break
    else:
        return False
    dist_lens.sort(key=lambda l: l != v)
    i = lit_lens.index(v)
    lit_lens[i], lit_lens[hlit - 1] = lit_lens[hlit - 1], lit_lens[i]
    at = hlit - 2
    if lit_lens.count(v) >= 2 and rng.random() < 0.5:
        i = lit_lens.index(v)
        lit_lens[i], lit_lens[at] = lit_lens[at], lit_lens[i]
        at -= 1
    if lit_lens[at] == v:
        j = next(j for j in range(hlit) if lit_lens[j] != v)
        lit_lens[j], lit_lens[at] = lit_lens[at], lit_lens[j]
    return True


def flat_code(rng, lits: Counter, hclen: int):
    """a lit/len code over the used symbols and fillers whose lengths need exactly `hclen` (5-10) code-length codes: 8 (HCLEN 5),
    7 and 8 (6), 7, 8 and 9 (7), then one code of 6, 10 or 5 bits among 8-bit codes; None when too many symbols are used"""
    n = len(lits)
    if n > (286 if hclen == 7 else 249):
        return None
    if hclen == 5:
        sizes = [8] * 256
    elif hclen == 6:
        m = rng.randint(max(n, 129), 256)
        sizes = [7] * (256 - m) + [8] * (2 * m - 256)
    elif hclen == 7:
        b = rng.randint(223, min(254, 509 - n))
        sizes = [7] + [8] * b + [9] * (508 - 2 * b)
    else:                                                               # 6 (index 7 of CL_ORDER), 10 (8) or 5 (9) once
        sizes = {8: [6] + [8] * 252, 9: [6] + [8] * 251 + [10] * 4, 10: [5] + [8] * 248}[hclen]
    if len(sizes) < n or len(sizes) > 286:
        return None
    syms = list(lits) + rng.sample([s for s in range(286) if s not in lits], len(sizes) - n)
    rng.shuffle(sizes)
    lens = [0] * 286
    for s, l in zip(syms, sizes):
        lens[s] = l
    return lens


def stored_block(w: BitWriter, data, final: int):
    w.bits(final, 3)
    w.align()
    at = len(w.out)
    w.out += struct.pack("<HH", len(data), len(data) ^ 0xFFFF)
    w.out += data
    return at


# ---- parse ----------------------------------------------------------------------------------------------------------------------
def match_len(data, p: int, q: int, cap: int) -> int:
    """longest k <= cap with data[p:p + k] == data[q:q + k] (q < p; the ranges may overlap)"""
    if data[p:p + cap] == data[q:q + cap]:
        return cap
    lo, hi = 0, cap
    while hi - lo > 1:
        m = (lo + hi) // 2
        if data[p:p + m] == data[q:q + m]:
            lo = m
        else:
            hi = m
    return lo


def push(heads: dict, key, q: int) -> None:
    h = heads.get(key)
    if h is None:
        heads[key] = [q]
    else:
        h.append(q)
        if len(h) > 8:
            del h[0]


def parse(rng, data, a: int, b: int, heads: dict, pm: float):
    """tokens of data[a:b]: literal runs and matches over earlier occurrences within 32 KiB (hash heads), distances 1-4, 32768 and
    distance = bytes so far; heads maps 3-byte keys to recent positions and is updated for later blocks"""
    toks, p = [], a
    head = data[:3]
    while p < b:
        cap = min(258, b - p)
        if cap >= 3 and rng.random() < pm:
            key = data[p:p + 3]
            cands = [d for d in (1, 2, 3, 4, 32768, p) if 0 < d <= min(p, 32768)]
            cands += [p - q for q in heads.get(key, ()) if 0 < p - q <= 32768]
            best = []
            for d in cands:
                n = match_len(data, p, p - d, cap)
                if n >= 3:
                    best.append((d, n))
            if best:
                special = [x for x in best if x[0] in (32768, p) or (x[0] <= 4 and x[0] < x[1])]
                d, n = rng.choice(special if special and rng.random() < 0.7 else best)
                if rng.random() < 0.3:
                    n = rng.randint(3, n)
                toks.append((n, d, n == 258 and rng.random() < 0.5))
                push(heads, key, p)
                for q in range(p + 1, p + n, 7):
                    push(heads, data[q:q + 3], q)
                p += n
                continue
        r = min(b - p, rng.choice([1, 1, 2, 5, 20, 100]))
        if p < 32768:
            nxt = data.find(head, p + 1, min(p + r + 2, 32770))      # stop a literal run where data[0:3] recurs
            if nxt > 0:
                r = min(r, nxt - p)
        for q in range(p, p + r, 3):
            push(heads, data[q:q + 3], q)
        toks.extend(data[p:p + r])
        p += r
    return toks


# ---- streams --------------------------------------------------------------------------------------------------------------------
def header(rng) -> bytes:
    """a random valid zlib header: CM 8, CINFO 0-7, any FLEVEL, no dictionary"""
    cmf = rng.randint(0, 7) << 4 | 8
    flg = rng.randint(0, 3) << 6
    flg |= 31 - (cmf << 8 | flg) % 31
    return bytes([cmf, flg])


def plan(rng, n: int, max_blocks: int):
    """[(type, start, end)] covering [0, n): 0 stored, 1 fixed, 2 dynamic; empty blocks of every type; stored blocks of 0, 1, random
    and 65535 bytes"""
    k = rng.randint(1, max(1, min(max_blocks, n // 8 + 1)))
    cuts = {0, n} | {rng.randint(0, n) for _ in range(k - 1)}
    forced = {}
    if n >= 65535 + 10 and rng.random() < 0.7:
        a = rng.randint(0, n - 65535)
        cuts = {c for c in cuts if not a < c < a + 65535} | {a, a + 65535}
        forced[a] = a + 65535
    if n >= 2 and rng.random() < 0.5:
        a = rng.randint(0, n - 1)
        if not any(s <= a < e for s, e in forced.items()):
            cuts = {c for c in cuts if not a < c < a + 1} | {a, a + 1}
            forced[a] = a + 1
    cuts = sorted(cuts)
    out = []
    for a, b in zip(cuts, cuts[1:]):
        t = 0 if forced.get(a) == b else rng.choice([0, 1, 2, 2])
        out.append((2 if t == 0 and b - a > 65535 else t, a, b))
        if rng.random() < 0.15:
            out.append((rng.randint(0, 2), b, b))
    return out


def write(data: bytes, seed: int, max_blocks: int = 50) -> Stream:
    """a zlib stream of data from a seeded block plan; returns Stream(z, tags, blocks)"""
    rng = random.Random(seed)
    data = bytes(data)
    w = BitWriter()
    tags, blocks, heads = [], [], {}
    pl = plan(rng, len(data), max_blocks)
    for i, (t, a, b) in enumerate(pl):
        final = int(i == len(pl) - 1)
        at = w.pos()
        if t == 0:
            blocks.append((0, at, stored_block(w, data[a:b], final)))
            tags.append("stored")
            continue
        toks = parse(rng, data, a, b, heads, rng.choice([0.0, 0.3, 0.7, 0.95]))
        hdr = {"cross16": rng.random() < 0.25} if t == 2 else {}
        huffman_block(w, rng, toks, final, t, tags, **hdr)
        blocks.append((t, at, -1))
    z = header(rng) + w.getvalue() + struct.pack(">I", zlib.adler32(data) & 0xFFFFFFFF)
    return Stream(z, tags, [(t, at + 16, sa + 2 if sa >= 0 else -1) for t, at, sa in blocks])


# ---- the expected result: zlib ------------------------------------------------------------------------------------------------
def header_ok(z) -> bool:
    """RFC 1950 as zlib reads it with a 32 KiB window: CM 8, CINFO <= 7, FCHECK, no preset dictionary"""
    return len(z) >= 2 and z[0] & 15 == 8 and z[0] >> 4 <= 7 and (z[0] << 8 | z[1]) % 31 == 0 and not z[1] & 0x20


def expect(z, n_raw: int):
    """(inflated bytes, Adler verdict "ok" / "bad" / "missing"), or None when a decoder must reject z for an output of n_raw bytes"""
    if not header_ok(z):
        return None
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(bytes(z[2:]), n_raw + 1)
    except zlib.error:
        return None
    if not d.eof or len(out) != n_raw:
        return None
    t = d.unused_data
    if len(t) < 4:
        return out, "missing"
    return out, "ok" if struct.unpack(">I", t[:4])[0] == zlib.adler32(out) & 0xFFFFFFFF else "bad"


# ---- invalid streams ----------------------------------------------------------------------------------------------------------
def invalid_streams(data: bytes, seed: int) -> dict:
    """{name: zlib stream} that every decoder must reject for an output of len(data) bytes; each follows a good first block where
    the rule allows one.  Each breaks its one rule only: where a decoder without that rule has an obvious reading (a longer HLIT /
    HDIST, an incomplete code, a repeat cut at the end, ...) the stream then inflates to exactly `data` (test_deflategen_cpu.py)"""
    rng = random.Random(seed)
    data = bytes(data)
    n = len(data)
    k = n // 2
    out = {}

    def stream(body, adler=True, prefix=k):
        w = BitWriter()
        if prefix:
            huffman_block(w, rng, list(data[:prefix]), 0, 1, [])
        body(w)
        z = b"\x78\x01" + w.getvalue()
        return z + struct.pack(">I", zlib.adler32(data) & 0xFFFFFFFF) if adler else z

    rest = list(data[k:])
    lits = Counter(rest + [EOB])
    full = make_code(random.Random(seed), lits, 286, [], "lit")
    top = max(full)
    used = [s for s in range(286) if full[s]]

    def dyn(lit_lens=None, dist_lens=None, toks=rest, **hdr):
        return lambda w: huffman_block(w, rng, toks, 1, 2, [], lit_lens=lit_lens if lit_lens is not None else full,
                                       dist_lens=dist_lens if dist_lens is not None else [0] * 30, **hdr)

    free = [s for s in range(286) if not full[s]]
    over = list(full)
    over[free[0] if free else 285] = 1
    out["oversubscribed lit/len code"] = stream(dyn(over))
    out["oversubscribed distance code"] = stream(dyn(dist_lens=[1, 1, 1] + [0] * 27))
    out["oversubscribed CL code"] = stream(dyn(cl_lens=[1] * 19))
    vals = set(full) | {0}
    out["incomplete CL code"] = stream(dyn(cl_lens=[5 if s in vals else 0 for s in range(19)], mode="plain"))
    # one CL symbol can only send one length value (or zero runs): without the rule the lengths would still fail (here: no EOB)
    out["incomplete CL code, one 1-bit code"] =stream(lambda w: raw_cl(w, [0] * 18 + [1], [(18, 7, 127), (18, 7, 108)]))
    x = free[0] if free else 285                                         # a symbol the block never sends
    inc = [0] * 286
    for sy, l in limited_huffman({**{sy: f for sy, f in lits.items() if sy != x}, x: 1}, 15).items():
        inc[sy] = l
    inc[x] = 0                                                           # incomplete, longest code > 1 bit, every sent symbol coded
    out["incomplete lit/len code"] = stream(dyn(inc))
    out["incomplete distance code"] = stream(dyn(dist_lens=[1, 2] + [0] * 28))
    no_eob = list(full)
    no_eob[EOB] = 0
    no_eob[free[0] if free else 285] = full[EOB]
    out["no end-of-block code"] = stream(dyn(no_eob, toks=[]))
    for f in (30, 31):                                                   # HLIT 287 / 288, HDIST 31 / 32, trees otherwise valid
        out["HLIT field %d" % f] = stream(dyn(full + [0] * (f - 29), hlit=257 + f))
        out["HDIST field %d" % f] = stream(dyn(dist_lens=[1, 1] + [0] * (f - 1), hdist=f + 1))
    # the last block holds EOB alone after a good block of all the data: the code lengths break one rule and are otherwise valid
    cl = [0] * 19
    cl[0] = cl[1] = cl[16] = cl[18] = 2
    # a 16 first (3 lengths), 138 + 115 zeros, EOB 1 bit at 256, distance length 0: HLIT + HDIST = 258
    out["16 repeat first"] = stream(lambda w: raw_cl(w, cl, [(16, 2, 0), (18, 7, 127), (18, 7, 104), (1, 0, 0), (0, 0, 0)]), prefix=n)
    cl = [0] * 19
    cl[1], cl[16], cl[18] = 1, 2, 2
    # 138 + 118 zeros, EOB 1 bit at 256, then a 16 of 3 from k = 257: two past HLIT + HDIST = 258
    out["repeat past HLIT + HDIST"] = stream(lambda w: raw_cl(w, cl, [(18, 7, 127), (18, 7, 107), (1, 0, 0), (16, 2, 0)]), prefix=n)
    for s in (286, 287):
        out["fixed lit/len %d" % s] = stream(lambda w, s=s: fixed_syms(w, [s]))
    for s in (30, 31):
        out["fixed distance %d" % s] = stream(lambda w, s=s: fixed_syms(w, [257, ("d", s)]))
    j = min(k, 30000)
    w = BitWriter()
    huffman_block(w, rng, list(data[:j]), 0, 1, [])
    huffman_block(w, rng, [(3, j + 1, False)] + list(data[j + 3:]), 1, 1, [])
    out["distance one past the output"] = b"\x78\x01" + w.getvalue() + struct.pack(">I", zlib.adler32(data) & 0xFFFFFFFF)
    out["stored NLEN mismatch"] = stream(lambda w: (w.bits(1, 3), w.raw(struct.pack("<HH", n - k, (n - k) ^ 0xFFFE) + data[k:])))
    out["stored length past the end"] = stream(lambda w: (w.bits(1, 3), w.raw(struct.pack("<HH", n - k + 5, (n - k + 5) ^ 0xFFFF)
                                                                                  + data[k:])), adler=False)
    out["block type 3 after a good block"] = stream(lambda w: (w.bits(1 | 3 << 1, 3), w.bits(0, 16)))
    out["no final block"] = stream(lambda w: huffman_block(w, rng, rest, 0, 1, []), adler=False)
    # the stream ends between the bits of a code of more than 8 bits
    w = BitWriter()
    huffman_block(w, rng, list(data[:k]), 0, 1, [])
    lens = random_complete(random.Random(seed), 286, 15)
    w.bits(1 | 2 << 1, 3)
    code_lengths_header(w, rng, lens, [0] * 30, [], hlit=286, hdist=30)
    lt = table(lens)
    cut = None
    for t in rest:
        if cut is None and lt[t][1] > 8:
            cut = w.pos() // 8 + 1
        w.bits(*lt[t])
    if cut is not None:
        out["truncated inside a symbol"] = b"\x78\x01" + w.getvalue()[:cut]
    out["one byte short"] = write(data[:-1], seed, 4).z
    out["one byte long"] = write(data + b"\0", seed + 1, 4).z
    return out


def raw_cl(w: BitWriter, cl_lens, toks, hlit=257, hdist=1):
    """a final dynamic block header with the given CL code and code-length tokens (sent as they are)"""
    w.bits(1 | 2 << 1, 3)
    code_lengths_header(w, None, None, None, [], hlit=hlit, hdist=hdist, hclen=19, cl_lens=cl_lens, cl_toks=toks)
    w.bits(0, 16)


def fixed_syms(w: BitWriter, syms):
    """a final fixed block of raw symbols: lit/len symbols and ("d", distance symbol) entries, no extra bits"""
    lt, dt = table(FIXED_LIT), table(FIXED_DIST)
    w.bits(1 | 1 << 1, 3)
    for s in syms:
        w.bits(*(dt[s[1]] if isinstance(s, tuple) else lt[s]))
    w.bits(*lt[EOB])


# ---- the filtered rows the corpus encodes -------------------------------------------------------------------------------------
def rows(seed: int, w: int, h: int, c: int, filters=(0, 1, 2, 3, 4)) -> bytes:
    """h filtered scanlines of 1 + w*c bytes: filter bytes from `filters`, bodies of noise, constant runs, short periods (distances
    1-4), copies from up to 32 KiB back and few-symbol noise; row 0's start recurs at a later row start (a match back to byte 0)
    and a stretch of a long row repeats what stood 32768 bytes before it"""
    rng = random.Random(seed)
    stride = w * c + 1
    out = bytearray()
    for y in range(h):
        out.append(rng.choice(filters))
        end = len(out) + w * c
        while len(out) < end:
            n = min(end - len(out), rng.choice([1, 3, 8, 40, 300, 2000]))
            kind = rng.randrange(6)
            if kind == 0:
                out += rng.randbytes(n)
            elif kind == 1:
                out += bytes([rng.randrange(256)]) * n
            elif kind == 2:
                pat = rng.randbytes(rng.randint(2, 4))
                out += (pat * (n // len(pat) + 1))[:n]
            elif kind == 3 and len(out) > 0:
                d = rng.randint(1, min(32768, len(out)))
                for i in range(n):
                    out.append(out[-d])
            elif kind == 4:
                alpha = rng.randbytes(rng.randint(2, 12))
                out += bytes(rng.choice(alpha) for _ in range(n))
            else:
                out += bytes(n)
    if h > 1:
        y = min(h - 1, max(1, 32768 // stride))
        n = min(stride, 64)
        out[y * stride:y * stride + n] = out[:n]
    for y in range(h):
        if stride > 300 and y * stride + 1 > 32768:
            p = y * stride + 1 + rng.randint(0, stride - 300)
            n = min(stride - 1 - (p - y * stride - 1), 600)
            out[p:p + n] = out[p - 32768:p - 32768 + n]
            break
    for y in range(h):
        if out[y * stride] > 4:
            out[y * stride] = rng.choice(filters)
    return bytes(out)


CORPUS_SHAPES = [(1, 1, 1), (2, 3, 2), (5, 3, 3), (17, 9, 4), (64, 33, 1), (100, 60, 3), (33, 200, 2), (255, 129, 1), (257, 129, 4),
                 (300, 300, 3), (1000, 250, 4), (700, 500, 3), (1024, 1024, 4)]
CHEAP = 20000      # raw bytes above which rows use only filters None / Up (a cheap numpy unfilter)


@functools.lru_cache(maxsize=None)
def corpus():
    """[(w, h, c, raw, Stream)]: the valid 8-bit corpus of the GPU test"""
    out = []
    for k, (w, h, c) in enumerate(CORPUS_SHAPES):
        n = h * (w * c + 1)
        raw = rows(1000 + k, w, h, c, (0, 1, 2, 3, 4) if n <= CHEAP else (0, 2))
        out.append((w, h, c, raw, write(raw, 2000 + k)))
    return out


@functools.lru_cache(maxsize=None)
def fuzz_bases(count: int = 24):
    """[(w, h, c, raw, Stream)]: generated files of 50 B to 256 KB raw, log-uniform, the bases of the mutation fuzz"""
    rng = random.Random(77)
    out = []
    for k in range(count):
        target = int(50 * (256 * 1024 / 50) ** rng.random())
        c = rng.randint(1, 4)
        w = max(1, min(target // c, rng.randint(1, 2048)))
        h = max(1, target // (w * c + 1))
        n = h * (w * c + 1)
        raw = rows(3000 + k, w, h, c, (0, 1, 2, 3, 4) if n <= CHEAP else (0, 2))
        out.append((w, h, c, raw, write(raw, 4000 + k)))
    return out


EXT_SHAPES = [(37, 23, 3, 2, 1), (301, 211, 3, 2, 1), (1, 1, 3, 2, 1), (50, 30, 2, 16, 0), (200, 150, 2, 16, 0), (9, 7, 2, 16, 1)]


@functools.lru_cache(maxsize=None)
def ext_corpus():
    """[(samples, color type, depth, interlace, palette, raw, Stream)]: 2-bit palette Adam7 and 16-bit RGB files (pngwrite_formats)
    whose inflated length is PngDesc::raw_len rather than h * (1 + w * c)"""
    import numpy as np
    import pngwrite_formats as pf
    out = []
    for k, (w, h, ctype, depth, il) in enumerate(EXT_SHAPES):
        rs = np.random.RandomState(k)
        plte = rs.randint(0, 256, (4, 3)).astype(np.uint8) if ctype == 3 else None
        s = pf.random_samples(rs, w, h, ctype, depth, 4)
        raw = pf.raw_stream(s, ctype, depth, il, seed=k)
        out.append((s, ctype, depth, il, plte, raw, write(raw, 5000 + k)))
    return out
