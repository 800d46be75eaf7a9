"""Seeded damaged fpng streams for the fpng decode (decode_prepare_kernel, decode_scan_kernel, decode_link_kernel,
decode_write_kernel, decode_stored_kernel), placed at the boundaries where those kernels split a stream between them.

The kernels cut a file's stream into subsequences of SUB_BITS bits, counted from the 4-byte aligned file byte
(idat_ofs + 8) & ~3 ("aligned bits" below).  A scan or write CTA covers DEC_THREADS subsequences (32 KiB), and the link kernel
walks chunks of LINK_THREADS subsequences (128 KiB) with a carry between them.  The WS_THREADS boundary (28 KiB) is where the CTAs
of an earlier, shared-memory staged write kernel met; the cases placed there are kept as a boundary that falls inside a CTA.  Every
case names the construct it reaches: its family and, where it was placed, the boundary and the aligned bit of the damage.
tests/test_decode_damage_cpu.py checks that each placed case lands where it claims and that the oracle equals the reference on
every case; tests/test_decode_damage_gpu.py compares every decode entry point with the reference.

  * large base files (oracle-written, byte-identical to the reference's): 1-pass, 2-pass, run- and match-dominated, stored;
  * random damage: the five families of the CPU stream fuzz (tests/test_oracle_cpu.py) plus a resized IDAT (its length and
    CRC rewritten) and damage to the stream's last 16 bytes and its Adler-32, half at uniform positions, half within +-8 bytes
    of a boundary;
  * small files: exactly the CPU fuzz's 2500 mutants (cpu_fuzz, which that test also uses);
  * placed violations: each token violation of streamgen.cases() in a 1024 x 128 image, its token within +-32 bits of a
    boundary, or inside the first or the last subsequence;
  * stored files: filter bytes, LEN / NLEN and BFINAL damage at chosen blocks and rows.
"""
from __future__ import annotations

import struct
import zlib
from dataclasses import dataclass

import numpy as np

import imagegen
import streamgen

SUB_BITS = 1024                 # decode.cuh kSubBits
DEC_THREADS = 256               # decode.cuh kDecThreads: subsequences per scan / write CTA
WS_THREADS = 224                # subsequences per CTA of the removed staged write kernel
LINK_THREADS = 1024             # decode.cuh kLinkThreads: subsequences per link chunk
PRE_ROLL = 256                  # decode.cuh kPreRoll: default speculative lead-in of the scan

# named boundaries, in aligned bits: the first two subsequence boundaries, WS_THREADS subsequences, one scan CTA, one and two
# link chunks
BOUNDS = {"sub1": SUB_BITS, "sub2": 2 * SUB_BITS, "ws_cta": WS_THREADS * SUB_BITS, "cta": DEC_THREADS * SUB_BITS,
          "link": LINK_THREADS * SUB_BITS, "link2": 2 * LINK_THREADS * SUB_BITS}
NEAR_BYTES = 8                  # random damage "near" a boundary: within +-8 bytes
NEAR_BITS = 32                  # a placed violation "at" a boundary: its token starts within +-32 bits


@dataclass
class Case:
    name: str
    group: str                  # base file (large), "small", "placed_<code>_c<chans>" or "stored"
    file: bytes
    chans: int
    family: str                 # damage family or violation kind
    where: str | None = None    # boundary name, "first", "last", or None (uniform)
    bit: int | None = None      # aligned bit of the damage / the violating token
    crc_ok: bool = False        # the IDAT CRC matches the damaged data
    sym: int | None = None      # placed: the Deflate symbol at `bit`


# ---- stream geometry ---------------------------------------------------------------------------------------------------------
def idat(png: bytes):
    """(idat_ofs, idat_len): the IDAT chunk's length field offset and data length (one IDAT, as fpng writes)"""
    o = png.index(b"IDAT") - 4
    return o, struct.unpack(">I", png[o:o + 4])[0]


def origin(idat_ofs: int) -> int:
    """file byte of aligned bit 0"""
    return (idat_ofs + 8) & ~3


def bit0(idat_ofs: int) -> int:
    """aligned bit of the zlib stream's first bit"""
    return ((idat_ofs + 8) & 3) * 8


def last_sub(idat_ofs: int, idat_len: int) -> int:
    """index of the last subsequence (file_span's g1: tokens end before the Adler bytes)"""
    end = max(idat_len - 4, 0) * 8 + bit0(idat_ofs)
    return (end - 1) // SUB_BITS if end else 0


def bounds_of(png: bytes) -> dict:
    """the named boundaries inside the file's token bits, aligned bits; "last" is the last subsequence's first bit"""
    o, n = idat(png)
    end = (n - 4) * 8 + bit0(o)
    out = {k: v for k, v in BOUNDS.items() if v < end}
    out["last"] = last_sub(o, n) * SUB_BITS
    return out


def with_idat(png: bytes, data: bytes) -> bytes:
    """png with its IDAT data replaced: length and CRC rewritten"""
    o, n = idat(png)
    body = b"IDAT" + data
    return png[:o] + struct.pack(">I", len(data)) + body + struct.pack(">I", zlib.crc32(body) & 0xFFFFFFFF) + png[o + 12 + n:]


def crc_ok(png: bytes) -> bool:
    o, n = idat(png)
    return struct.unpack(">I", png[o + 8 + n:o + 12 + n])[0] == zlib.crc32(png[o + 4:o + 8 + n]) & 0xFFFFFFFF


def filtered_from_pixels(px: np.ndarray, stored: bool) -> bytes:
    """the filtered stream fpng writes for pixels [h, w, c]: filter 0 on row 0 and Up below, or (stored) filter 0 on every row"""
    h = px.shape[0]
    rows = px.reshape(h, -1).astype(np.uint8)
    if stored:
        body, filt = rows, np.zeros((h, 1), np.uint8)
    else:
        body = rows.copy()
        body[1:] = rows[1:] - rows[:-1]
        filt = np.full((h, 1), 2, np.uint8)
        filt[0] = 0
    return np.hstack([filt, body]).tobytes()


def stored_adler(png: bytes) -> int:
    o, n = idat(png)
    return struct.unpack(">I", png[o + 8 + n - 4:o + 8 + n])[0]


# ---- large base files --------------------------------------------------------------------------------------------------------
# (name, imagegen kind, w, h, chans, flags): 1-pass RGB / RGBA over 3+ link chunks, 2-pass (u128: a near-fixed-length code, most
# speculative starts wrong), run- and match-dominated streams, and a stored file of six 65535-byte blocks
LARGE = (("g1_1pass_c3", "g1", 1024, 200, 3, 0), ("g1_1pass_c4", "g1", 1024, 160, 4, 0), ("u128_2pass_c3", "u128", 1024, 160, 3, 1),
         ("g1_2pass_c3", "g1", 1024, 200, 3, 1), ("runs_1pass_c4", "runs", 1536, 768, 4, 0), ("g0_1pass_c3", "g0", 2048, 1024, 3, 0),
         ("g1_stored_c3", "g1", 640, 200, 3, 2))
RANDOM_PER_FILE = 70
FAMILIES = ("overwrite", "bit_flip", "splice", "swap", "header", "resize", "tail")


def large_bases(oracle):
    """{name: (file, w, h, chans, flags)}"""
    return {name: (oracle.encode(imagegen.make(kind, w, h, c, 5), w, h, c, fl), w, h, c, fl) for name, kind, w, h, c, fl in LARGE}


def _near_positions(png):
    """{boundary: file byte} of the boundaries inside the IDAT data"""
    o, n = idat(png)
    return {k: origin(o) + v // 8 for k, v in bounds_of(png).items()}


def random_cases(bases):
    out = []
    for gi, (name, (png, w, h, c, fl)) in enumerate(bases.items()):
        rs = np.random.RandomState(1000 + gi)
        o, n = idat(png)
        z0, z1 = o + 8, o + 8 + n                                     # IDAT data bytes
        near = [(k, v) for k, v in _near_positions(png).items() if z0 <= v < z1 - 4]
        for t in range(RANDOM_PER_FILE):
            fam = FAMILIES[t % len(FAMILIES)]
            if t % 2 and near:
                where, b = near[(t // 2) % len(near)]
                p = int(np.clip(b + rs.randint(-NEAR_BYTES, NEAR_BYTES + 1), z0, z1 - 5))
            else:
                where, p = None, int(rs.randint(z0, z1 - 4))
            bad = bytearray(png)
            if fam == "overwrite":
                for k in range(rs.randint(1, 4)):
                    bad[min(p + k, z1 - 1)] = rs.randint(0, 256)
            elif fam == "bit_flip":
                bad[p] ^= 1 << rs.randint(0, 8)
            elif fam == "splice":
                L = rs.randint(1, 9)
                bad[p:p + L] = bytes(rs.randint(0, 256, L, dtype=np.uint8))
                bad = bad[:len(png)]
            elif fam == "swap":
                q = int(rs.randint(z0, z1))
                bad[p], bad[q] = bad[q], bad[p]
            elif fam == "header":
                where, p = "header", int(rs.randint(z0, min(z0 + 70, z1)))
                bad[p] = rs.randint(0, 256)
            elif fam == "resize":
                k = int(rs.randint(1, 10))
                data = bytes(png[z0:z1])
                q = p - z0
                data = data[:q] + bytes(rs.randint(0, 256, k, dtype=np.uint8)) + data[q:] if rs.rand() < 0.5 else data[:q] + data[q + k:]
                bad = bytearray(with_idat(png, data))
            else:                                                      # the last 16 stream bytes and the 4 Adler bytes
                where, p = "tail", int(rs.randint(z1 - 20, z1))
                if rs.rand() < 0.5:
                    bad[p] ^= 1 << rs.randint(0, 8)
                else:
                    bad[p] = rs.randint(0, 256)
            bad = bytes(bad)
            out.append(Case(f"{name}_{t}_{fam}", name, bad, c, fam, where, 8 * (p - origin(o)), crc_ok(bad)))
    return out


# ---- the CPU stream fuzz's small files ---------------------------------------------------------------------------------------
CPU_FUZZ_FILES = (("g1", 97, 31, 4, 0), ("g1", 160, 24, 3, 0), ("g0", 256, 40, 4, 0), ("runs", 300, 17, 3, 0), ("g1", 128, 32, 3, 1),
                  ("runs", 301, 9, 4, 1), ("g2", 40, 9, 3, 0), ("mut", 120, 33, 4, 0), ("g0", 333, 20, 3, 1), ("g1", 40, 12, 4, 2))


def cpu_fuzz(oracle):
    """[(kind, w, h, c, flags, trial, family index, mutant)]: the 2500 mutants of the CPU stream fuzz (seed 77), in its order:
    byte overwrites, bit flips, short random splices, byte swaps and block-header damage inside the IDAT payload"""
    rs = np.random.RandomState(77)
    out = []
    for kind, w, h, c, fl in CPU_FUZZ_FILES:
        png = oracle.encode(imagegen.make(kind, w, h, c, 5), w, h, c, fl)
        idat_, end = png.index(b"IDAT") + 4, len(png) - 16
        for trial in range(250):
            bad = bytearray(png)
            m = rs.randint(0, 5)
            if m == 0:
                for _ in range(rs.randint(1, 4)):
                    bad[rs.randint(idat_, end)] = rs.randint(0, 256)
            elif m == 1:
                bad[rs.randint(idat_, end)] ^= 1 << rs.randint(0, 8)
            elif m == 2:
                p, L = rs.randint(idat_, end - 8), rs.randint(1, 8)
                bad[p:p + L] = bytes(rs.randint(0, 256, L, dtype=np.uint8))
            elif m == 3:
                a, b = rs.randint(idat_, end), rs.randint(idat_, end)
                bad[a], bad[b] = bad[b], bad[a]
            else:
                bad[rs.randint(idat_, min(idat_ + 70, end))] = rs.randint(0, 256)
            out.append((kind, w, h, c, fl, trial, int(m), bytes(bad)))
    return out


def small_cases(oracle):
    names = ("overwrite", "bit_flip", "splice", "swap", "header")
    return [Case(f"{kind}_{w}x{h}_c{c}_f{fl}_{t}", "small", bad, c, names[m], crc_ok=crc_ok(bad))
            for kind, w, h, c, fl, t, m, bad in cpu_fuzz(oracle)]


# ---- stored files ------------------------------------------------------------------------------------------------------------
def stored_cases(bases):
    """filter bytes and block headers of the stored base file (raw = h * (w*c + 1) bytes in 65535-byte blocks)"""
    png, w, h, c, fl = bases["g1_stored_c3"]
    o, n = idat(png)
    z = o + 8
    rb = w * c + 1
    raw = rb * h
    nblk = -(-raw // 65535)
    hdr = lambda j: z + 2 + 65540 * j                                   # noqa: E731  file byte of block j's header
    at = lambda s: z + 2 + 5 * (s // 65535 + 1) + s                     # noqa: E731  file byte of raw byte s
    straddle = next(y for y in range(h) if (y * rb) // 65535 != (y * rb + rb - 1) // 65535)
    out = []

    def add(name, edits, where=None, byte=None):
        b = bytearray(png)
        for p, v in edits:
            b[p] = v(b[p])
        b = bytes(b)
        out.append(Case(f"stored_{name}", "stored", b, c, name, where, None if byte is None else 8 * (byte - origin(o)), crc_ok(b)))

    for name, y in (("filter_first_row", 0), ("filter_last_row", h - 1), (f"filter_row{straddle}_straddles_block", straddle)):
        add(name, [(at(y * rb), lambda v: v | 1)], byte=at(y * rb))
    for j in (1, nblk - 1):
        add(f"len_block{j}", [(hdr(j) + 1, lambda v: v ^ 1)], byte=hdr(j) + 1)
        add(f"nlen_block{j}", [(hdr(j) + 4, lambda v: v ^ 0x80)], byte=hdr(j) + 4)
        add(f"len_nlen_block{j}", [(hdr(j) + 1, lambda v: v ^ 1), (hdr(j) + 3, lambda v: v ^ 1)], byte=hdr(j) + 1)
    for j in (0, nblk - 2):
        add(f"bfinal_block{j}", [(hdr(j), lambda v: v | 1)], byte=hdr(j))
    add(f"bfinal_cleared_block{nblk - 1}", [(hdr(nblk - 1), lambda v: v & ~1)], byte=hdr(nblk - 1))
    add("btype_block2", [(hdr(2), lambda v: v | 2)], byte=hdr(2))
    return out


# ---- placed token violations -------------------------------------------------------------------------------------------------
PLACED_W, PLACED_H = 1024, 128
# anywhere a pixel starts; "realigned": a match of chans + 1 bytes and chans - 1 literals in place of two pixels, so that every
# later token is where it belongs and the match length is the only rule broken
MID_KINDS = ("length_not_multiple", "length_not_multiple_realigned", "match_not_pixel_aligned", "eob_early", "eob_missing")
ROW_KINDS = ("wrong_filter", "match_crosses_scanline")                                       # where a scanline starts / ends
END_KINDS = ("eob_late", "bytes_after_eob")                                                  # after the last scanline
FIRST_KINDS = ("first_filter_up", "wrong_filter_row0")                                       # the first scanline's filter byte


LEN_SYM, LEN_XB, LEN_XV = (np.array([streamgen.length_symbol(max(n, 3))[k] for n in range(259)], np.int64) for k in range(3))


def _rev(code, n):
    return int(format(code, f"0{n}b")[::-1], 2) if n else 0


class Code:
    """a literal / length and distance code (streamgen's flat286 or skewed12) with fpng's distance code, and a vectorised writer"""

    def __init__(self, name, chans, lit_sizes, pool_weights):
        self.name, self.chans = name, chans
        self.lit = list(lit_sizes)
        self.dist = streamgen.fpng_dist(chans)
        codes = streamgen.canonical_codes(self.lit)
        self.rev = np.array([_rev(codes[s], self.lit[s]) for s in range(len(self.lit))], np.uint64)
        self.size = np.array(self.lit, np.int64)
        self.dbits = self.dist[chans - 1]
        self.pool = np.array([v for v in range(256) if self.lit[v]])
        self.weights = pool_weights(self.pool, self.size[self.pool])
        hdr, at = streamgen.dynamic_block(self.lit, self.dist, [("E",)], chans, offsets=True)
        self.hbits = at[0]
        self.hdr = np.unpackbits(np.frombuffer(hdr, np.uint8), bitorder="little")[:self.hbits]
        self.by_size = {}
        for v in self.pool:
            self.by_size.setdefault(int(self.size[v]), []).append(int(v))

    def token_bits(self, kind, val):
        """(value LSB first, bit count) of every token; kind 0 literal, 1 match (distance chans), 2 EOB"""
        m = np.nonzero(kind == 1)[0]
        lv = np.clip(val, 3, 258)
        sym = np.where(kind == 0, val, np.where(kind == 2, 256, LEN_SYM[lv])).astype(np.int64)
        xb = np.where(kind == 1, LEN_XB[lv], 0)
        xv = np.where(kind == 1, LEN_XV[lv], 0).astype(np.uint64)
        ls = self.size[sym]
        v = self.rev[sym].copy()
        n = ls.copy()
        v[m] |= xv[m] << ls[m].astype(np.uint64)
        n[m] += xb[m] + self.dbits                                    # the distance code: fpng's single 1-bit code word, 0
        return v, n

    def pack(self, kind, val):
        """(deflate block bytes, bit offset of every token from the block's first bit)"""
        v, n = self.token_bits(kind, val)
        starts = np.concatenate([[0], np.cumsum(n)[:-1]]) + self.hbits
        total = int(n.sum())
        rv = np.repeat(v, n)
        idx = (np.arange(total, dtype=np.int64) - np.repeat(starts - self.hbits, n)).astype(np.uint64)
        bits = np.concatenate([self.hdr, ((rv >> idx) & np.uint64(1)).astype(np.uint8)])
        return np.packbits(bits, bitorder="little").tobytes(), starts


def filtered(kind, val, chans):
    """what a Deflate decoder makes of the token arrays (matches copy chans bytes back), up to the first EOB; None when a match
    reaches before the stream start"""
    e = np.nonzero(kind == 2)[0]
    stop = int(e[0]) if len(e) else len(kind)
    k, v = kind[:stop], val[:stop]
    n = np.where(k == 0, 1, v)
    at = np.concatenate([[0], np.cumsum(n)])
    out = np.zeros(int(at[-1]), np.uint8)
    lit = np.zeros(int(at[-1]), bool)
    li = k == 0
    out[at[:-1][li]] = v[li]
    lit[at[:-1][li]] = True
    src = np.arange(len(out)) - chans
    todo = ~lit
    while todo.any():
        s = src[todo]
        if (s < 0).any():
            return None
        ok = lit[s]
        idx = np.nonzero(todo)[0]
        out[idx[ok]] = out[s[ok]]
        src[idx[~ok]] -= chans
        todo[idx[ok]] = False
    return out.tobytes()


def codes_for(chans):
    flat = streamgen.flat_sizes(286)
    lit = [0] * 286
    for i, s in enumerate([7, 1, 250, 3, 130, 5, 66]):
        lit[s] = i + 1
    streamgen.fill_sizes(lit, [streamgen.EOB] + [257 + i for i in range(29)] + [s for s in range(256) if s not in (7, 1, 250, 3, 130, 5, 66)],
                         spread=True)
    # flat286: as many 9-bit as 8-bit literals, so that a steered stream can move a token either way
    return [Code("flat286", chans, flat, lambda p, s: np.where(s == s.max(), 0.5 / (s == s.max()).sum(), 0.5 / (s != s.max()).sum())),
            Code("skewed12", chans, lit, lambda p, s: np.full(len(p), 1.0 / len(p)))]


def base_tokens(code, rs, w=PLACED_W, h=PLACED_H, match_rate=0.2):
    """token arrays (kind, val, unit) of an h-row image in fpng's grammar, EOB last: per scanline a filter byte (unit -1), then w
    pixels (unit = pixel index): chans literals from the code's pool, or (not the first pixel) a match of chans bytes"""
    c = code.chans
    pm = rs.rand(h, w) < match_rate
    pm[:, 0] = False
    ntok = np.hstack([np.ones((h, 1), np.int64), np.where(pm, 1, c)]).ravel()
    utype = np.hstack([np.full((h, 1), 2), pm.astype(np.int64)]).ravel()
    unit = np.repeat(np.tile(np.arange(-1, w), h), ntok)
    row = np.repeat(np.repeat(np.arange(h), w + 1), ntok)
    ut = np.repeat(utype, ntok)
    kind = np.where(ut == 1, 1, 0)
    val = rs.choice(code.pool, len(kind), p=code.weights).astype(np.int64)
    val[ut == 1] = c
    val[ut == 2] = np.where(row[ut == 2] == 0, 0, 2)
    first = np.concatenate([[True], unit[1:] != unit[:-1]])
    return (np.append(kind, 2), np.append(val, 0), np.append(unit, -2), np.append(row, h), np.append(first, True))


def _steer(code, kind, val, unit, i, delta):
    """changes pixel literals before token i so that token i moves by delta bits; returns the bits it could not move"""
    sizes = sorted(code.by_size)
    sign = 1 if delta > 0 else -1
    lits = np.nonzero((kind[:i] == 0) & (unit[:i] >= 0))[0][::-1]
    for j in lits:
        if not delta:
            break
        a = int(code.size[val[j]])
        cand = [s for s in sizes if 0 < (s - a) * sign <= abs(delta)]
        if cand:
            s = max(cand, key=lambda s: abs(s - a))
            val[j] = code.by_size[s][j % len(code.by_size[s])]
            delta -= s - a
    return delta


def _build(code, kind, val, trailing=b""):
    blk, starts = code.pack(kind, val)
    data = filtered(kind, val, code.chans)
    f = streamgen.png_file(PLACED_W, PLACED_H, code.chans, streamgen.zlib_stream(blk + trailing, data or b""))
    o, _ = idat(f)
    return f, starts + 16 + bit0(o)                                   # token aligned bits


def _sym(kind, val):
    if kind == 0:
        return int(val)
    if kind == 2:
        return 256
    return streamgen.length_symbol(int(val))[0]


def dynamic_header(png: bytes):
    """(literal / length code sizes, aligned bit of the first token) of the file's dynamic block, read with deflatetrace's bit
    reader and code tables (not with the writer above)"""
    import deflatetrace as dt
    o, n = idat(png)
    bits = dt._Bits(png[o + 8:o + 8 + n], 16)
    bits.get(3)
    hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
    cl = [0] * 19
    for k in range(hclen):
        cl[dt._CL_ORDER[k]] = bits.get(3)
    clt = dt._table(cl)
    lens = []
    while len(lens) < hlit + hdist:
        s = dt._decode(bits, clt)
        if s < 16:
            lens.append(s)
        elif s == 16:
            lens += [lens[-1]] * (3 + bits.get(2))
        else:
            lens += [0] * ((3 + bits.get(3)) if s == 17 else (11 + bits.get(7)))
    return lens[:hlit], bits.pos + bit0(o)


def symbol_at(png: bytes, bit: int) -> int:
    """the literal / length symbol the file's code reads at aligned bit `bit`"""
    import deflatetrace as dt
    o, n = idat(png)
    lit, _ = dynamic_header(png)
    return dt._decode(dt._Bits(png[o + 8:o + 8 + n], bit - bit0(o)), dt._table(lit))


def _claim(f, where, bit):
    o, n = idat(f)
    if where == "first":
        return bit // SUB_BITS == dynamic_header(f)[1] // SUB_BITS and bit < (n - 4) * 8 + bit0(o)
    if where == "last":
        return bit // SUB_BITS == last_sub(o, n)
    return abs(bit - BOUNDS[where]) <= NEAR_BITS


def claim_holds(case: Case) -> bool:
    """the placed case's damage starts where its name says: within NEAR_BITS of its boundary, or inside the first / last
    subsequence"""
    return _claim(case.file, case.where, case.bit)


def _place(code, base, kname, where, target, rs):
    kind0, val0, unit0, row0, first0, starts0 = base
    c = code.chans
    cands = []
    if kname in MID_KINDS:
        ok = first0 & (unit0 >= 1)
        if kname == "match_not_pixel_aligned":
            ok &= kind0 == 0
        if kname == "length_not_multiple_realigned":
            ok &= unit0 <= PLACED_W - 2
        idx = np.nonzero(ok)[0]
        cands = idx[np.argsort(np.abs(starts0[idx] - target))][:6]
    elif kname == "wrong_filter":
        idx = np.nonzero((unit0 == -1) & (row0 >= 1))[0]
        cands = idx[np.argsort(np.abs(starts0[idx] - target))][:4]
    elif kname == "match_crosses_scanline":
        idx = np.nonzero(first0 & (unit0 == PLACED_W - 1) & (row0 < PLACED_H - 1))[0]
        cands = idx[np.argsort(np.abs(starts0[idx] - target))][:4]
    for i in map(int, cands):
        kind, val = kind0.copy(), val0.copy()
        v = i                                                          # index of the violating token
        trailing = b""
        if kname == "wrong_filter":
            if _steer(code, kind, val, unit0, i, target - int(starts0[i])):
                continue
            val[i] = 1
        elif kname == "match_crosses_scanline":
            if _steer(code, kind, val, unit0, i, target - int(starts0[i])):
                continue
            end = i + 1
            while end < len(kind) and unit0[end] == unit0[i] and not first0[end]:
                end += 1
            kind = np.concatenate([kind[:i], [1], kind[end:]])
            val = np.concatenate([val[:i], [2 * c], val[end:]])
        elif kname == "length_not_multiple":
            kind, val = np.insert(kind, i, 1), np.insert(val, i, c + 1)
        elif kname == "length_not_multiple_realigned":
            end = i + 1
            while unit0[end] in (unit0[i], unit0[i] + 1) and row0[end] == row0[i]:
                end += 1
            kind = np.concatenate([kind[:i], [1] + [0] * (c - 1), kind[end:]])
            val = np.concatenate([val[:i], [c + 1] + [int(code.pool[1])] * (c - 1), val[end:]])
        elif kname == "match_not_pixel_aligned":
            kind, val = np.insert(kind, i + 1, 1), np.insert(val, i + 1, c)
            v = i + 1
        elif kname == "eob_early":
            kind, val = np.append(kind[:i], 2), np.append(val[:i], 0)
        elif kname == "eob_missing":
            kind, val = kind[:i].copy(), val[:i].copy()
        f, starts = _build(code, kind, val, trailing)
        bit = int(starts[v]) if v < len(starts) else int(starts[-1]) + int(code.token_bits(kind[-1:], val[-1:])[1][0])
        if _claim(f, where, bit):
            return f, bit, (None if v >= len(kind) else _sym(int(kind[v]), int(val[v])))
    return None


def _place_fixed(code, base, kname):
    """the violations whose place the grammar fixes: the first scanline's filter byte, and past the last scanline"""
    kind, val = base[0].copy(), base[1].copy()
    trailing, v = b"", None
    if kname == "first_filter_up":
        val[0], v, where = 2, 0, "first"
    elif kname == "wrong_filter_row0":
        val[0], v, where = 1, 0, "first"
    elif kname == "eob_late":
        v, where = len(kind) - 1, "last"
        kind = np.concatenate([kind[:-1], np.zeros(code.chans, np.int64), [2]])
        val = np.concatenate([val[:-1], np.full(code.chans, code.pool[1]), [0]])
    else:                                                              # bytes_after_eob
        trailing, where = b"\x00\x00", "last"
    f, starts = _build(code, kind, val, trailing)
    if v is None:
        return f, int(starts[-1]) + int(code.token_bits(kind[-1:], val[-1:])[1][0]), None, where
    return f, int(starts[v]), _sym(int(kind[v]), int(val[v])), where


def placed_cases():
    out = []
    for chans in (3, 4):
        for ci, code in enumerate(codes_for(chans)):
            rs = np.random.RandomState(40 + 2 * chans + ci)
            base = base_tokens(code, rs)
            f0, starts0 = _build(code, base[0], base[1])
            base += (starts0,)
            group = f"placed_{code.name}_c{chans}"
            targets = {k: v + int(rs.randint(-NEAR_BITS + 8, NEAR_BITS - 7)) for k, v in bounds_of(f0).items() if k != "last"}
            o, n = idat(f0)
            end = (n - 4) * 8 + bit0(o)
            targets["first"] = 16 + bit0(o) + code.hbits + 300
            targets["last"] = end - 200
            for kname in MID_KINDS + ROW_KINDS:
                for where, t in targets.items():
                    if kname in ROW_KINDS and where in ("first", "sub1", "sub2", "last"):
                        continue                                        # no scanline starts or ends there
                    r = _place(code, base, kname, where, t, rs)
                    assert r is not None, (group, kname, where)
                    f, bit, sym = r
                    out.append(Case(f"{group}_{kname}_{where}", group, f, chans, kname, where, bit, True, sym))
            for kname in FIRST_KINDS + END_KINDS:
                f, bit, sym, where = _place_fixed(code, base, kname)
                out.append(Case(f"{group}_{kname}_{where}", group, f, chans, kname, where, bit, True, sym))
    return out


# ---- everything --------------------------------------------------------------------------------------------------------------
_CACHE = {}


def corpus(oracle):
    """(cases, bases): every case of this module, and the large base files"""
    if "c" not in _CACHE:
        bases = large_bases(oracle)
        _CACHE["c"] = (random_cases(bases) + stored_cases(bases) + placed_cases() + small_cases(oracle), bases)
    return _CACHE["c"]
