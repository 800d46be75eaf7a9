"""A small pure-Python Deflate reader (RFC 1951) for the tests of the PNG encode: it returns what a stream is made of, not just
what it inflates to -- the block types, each stored block's length and position, each dynamic block's header and code lengths,
and the token stream (literals, and matches as (length, distance)).  It is written for clarity, not speed: small and medium
streams only.  tests/test_encode_png_edges_cpu.py checks its output against zlib before relying on it."""
from __future__ import annotations

from dataclasses import dataclass, field

_LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
_DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
              6145, 8193, 12289, 16385, 24577]
_DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
_CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class DeflateError(ValueError):
    pass


@dataclass
class Block:
    btype: int                                  # 0 stored, 1 fixed, 2 dynamic
    final: bool
    bit_start: int                              # bit offset of the block header in the Deflate stream
    out_start: int                              # offset of the block's first output byte
    out_end: int = 0
    stored_len: int | None = None               # stored blocks: LEN
    lit_lens: list[int] | None = None           # dynamic blocks: the HLIT literal/length and HDIST distance code lengths
    dist_lens: list[int] | None = None
    hclen: int | None = None
    tokens: list = field(default_factory=list)  # int: a literal byte; (length, distance): a match; 256 (EOB) is not listed


@dataclass
class Trace:
    blocks: list[Block]
    data: bytes                                 # the inflated stream
    end_bit: int                                # bit offset just past the last block (the stream's end, before padding)

    @property
    def end_byte(self) -> int:
        return (self.end_bit + 7) >> 3


class _Bits:
    def __init__(self, buf: bytes, pos: int = 0):
        self.buf, self.pos = buf, pos

    def get(self, n: int) -> int:
        if n == 0:
            return 0
        i, s = self.pos >> 3, self.pos & 7
        if (self.pos + n + 7) >> 3 > len(self.buf):
            raise DeflateError("stream ends inside a block")
        v = (int.from_bytes(self.buf[i:i + 4], "little") >> s) & ((1 << n) - 1)
        self.pos += n
        return v


def _table(lens: list[int]):
    """Canonical code of `lens` as a lookup table indexed by the next maxlen stream bits: (symbol, length) or None."""
    maxlen = max(lens, default=0)
    if maxlen == 0:
        return 0, []
    count = [0] * (maxlen + 1)
    for n in lens:
        if n:
            count[n] += 1
    nxt, code = [0] * (maxlen + 2), 0
    for n in range(1, maxlen + 1):
        code = (code + count[n - 1]) << 1 if n > 1 else 0
        nxt[n] = code
    left = 1
    for n in range(1, maxlen + 1):                              # over-subscribed codes are invalid
        left = (left << 1) - count[n]
        if left < 0:
            raise DeflateError("over-subscribed code")
    table = [None] * (1 << maxlen)
    for sym, n in enumerate(lens):
        if not n:
            continue
        c = nxt[n]
        nxt[n] += 1
        r = int(format(c, f"0{n}b")[::-1], 2)                   # Huffman codes are sent most significant bit first
        for k in range(1 << (maxlen - n)):
            table[r | (k << n)] = (sym, n)
    return maxlen, table


def _decode(bits: _Bits, maxlen_table) -> int:
    maxlen, table = maxlen_table
    if not maxlen:
        raise DeflateError("symbol from an empty code")
    i, s = bits.pos >> 3, bits.pos & 7
    v = (int.from_bytes(bits.buf[i:i + 3], "little") >> s) & ((1 << maxlen) - 1)
    e = table[v]
    if e is None:
        raise DeflateError("incomplete code")
    if bits.pos + e[1] > 8 * len(bits.buf):
        raise DeflateError("stream ends inside a code")
    bits.pos += e[1]
    return e[0]


_FIXED = None


def _fixed():
    global _FIXED
    if _FIXED is None:
        _FIXED = (_table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8), _table([5] * 30))
    return _FIXED


def trace(stream: bytes, zlib_header: bool = True, keep_tokens: bool = True) -> Trace:
    """Reads a Deflate stream (after a 2-byte zlib header when zlib_header) block by block."""
    bits = _Bits(stream, 16 if zlib_header else 0)
    out = bytearray()
    blocks = []
    while True:
        b = Block(btype=0, final=False, bit_start=bits.pos, out_start=len(out))
        b.final = bool(bits.get(1))
        b.btype = bits.get(2)
        if b.btype == 0:
            bits.pos = (bits.pos + 7) & ~7
            n, nn = bits.get(16), bits.get(16)
            if n != (~nn & 0xFFFF):
                raise DeflateError("stored LEN / NLEN mismatch")
            i = bits.pos >> 3
            if i + n > len(stream):
                raise DeflateError("stored block past the end")
            out += stream[i:i + n]
            bits.pos += 8 * n
            b.stored_len = n
        elif b.btype in (1, 2):
            if b.btype == 1:
                lit, dist = _fixed()
            else:
                hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
                cl = [0] * 19
                for k in range(hclen):
                    cl[_CL_ORDER[k]] = bits.get(3)
                clt = _table(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = _decode(bits, clt)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        if not lens:
                            raise DeflateError("repeat with no previous length")
                        lens += [lens[-1]] * (3 + bits.get(2))
                    elif s == 17:
                        lens += [0] * (3 + bits.get(3))
                    else:
                        lens += [0] * (11 + bits.get(7))
                if len(lens) != hlit + hdist:
                    raise DeflateError("code lengths overrun HLIT + HDIST")
                b.lit_lens, b.dist_lens, b.hclen = lens[:hlit], lens[hlit:], hclen
                lit, dist = _table(b.lit_lens), _table(b.dist_lens)
            while True:
                s = _decode(bits, lit)
                if s < 256:
                    out.append(s)
                    if keep_tokens:
                        b.tokens.append(s)
                elif s == 256:
                    break
                else:
                    if s > 285:
                        raise DeflateError("length symbol 286/287")
                    L = _LEN_BASE[s - 257] + bits.get(_LEN_EXTRA[s - 257])
                    d = _decode(bits, dist)
                    if d > 29:
                        raise DeflateError("distance symbol 30/31")
                    D = _DIST_BASE[d] + bits.get(_DIST_EXTRA[d])
                    if D > len(out):
                        raise DeflateError("distance before the start")
                    for _ in range(L):
                        out.append(out[-D])
                    if keep_tokens:
                        b.tokens.append((L, D))
        else:
            raise DeflateError("block type 3")
        b.out_end = len(out)
        blocks.append(b)
        if b.final:
            break
    return Trace(blocks, bytes(out), bits.pos)
