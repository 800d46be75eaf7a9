"""CPU model of how the default encoder gets the IDAT CRC-32 WITHOUT reading the finished file again (csrc/encode16_kernels.cu:
the pack kernel computes a raw CRC-32 of every scanline's code words while they sit in its staging buffer; csrc/crc_stream_kernel.cu
row_crc_combine_kernel folds them; reference: one fpng_crc32 call over "IDAT" + zlib stream, src/fpng.cpp:1797-1800).

Why it works -- the three facts this model checks on real files:
  1. Deflate packs bits LSB-first and the reflected CRC-32 consumes message bits LSB-first: a bit string's raw CRC (no initial value,
     no final XOR: A(x) * x^32 mod P) does not depend on its byte alignment in the file.
  2. The raw CRC is linear: pieces that overlap in 32-bit WORDS but are disjoint in BITS (a scanline's first and last word also hold
     bits of its neighbours; every piece is taken with zeros outside its own bits) can be summed,
         crc(M) = XOR_i raw(piece_i) * x^(bits from the end of piece_i's last word to the end of M)   (mod P),
     each scanline contributing independently -- no ordering, no atomics on the data path.
  3. The initial value and the final XOR are one more constant term: 0xFFFFFFFF * x^|M| + 0xFFFFFFFF.
Multiplication mod P in the reflected representation (bit 31 = x^0) is csrc/crc_math.cuh gf2_mulmod, restated here."""
import zlib

import numpy as np
import pytest

import imagegen

POLY = 0xEDB88320
ONE = 0x80000000


def mulmod(a, b):
    p = 0
    for i in range(32):
        if a & (0x80000000 >> i):
            p ^= b
        b = (b >> 1) ^ (POLY if b & 1 else 0)
    return p


def xpow(n):
    assert n >= 0
    r, base = ONE, 0x40000000                      # x
    while n:
        if n & 1:
            r = mulmod(r, base)
        base = mulmod(base, base)
        n >>= 1
    return r


def raw_crc_bits(bits):
    """A(x) * x^32 mod P of a bit sequence (first bit = highest power), register starting at 0"""
    r = 0
    for b in bits:
        r ^= int(b)
        r = (r >> 1) ^ (POLY if r & 1 else 0)
    return r


@pytest.mark.parametrize("kind,w,h,chans", [("g1", 96, 20, 3), ("g1", 64, 17, 4), ("g0", 300, 12, 4), ("runs", 257, 9, 3), ("mut", 128, 16, 3)])
def test_scanline_crcs_combine_to_the_idat_crc(oracle, kind, w, h, chans):
    img = imagegen.make(kind, w, h, chans, 4)
    png, rows, stored = oracle.encode(img, w, h, chans, 0, want_rows=True)
    assert not stored
    zsize = int.from_bytes(png[50:54], "big")
    assert len(png) == 58 + zsize + 16
    stored_crc = int.from_bytes(png[58 + zsize:58 + zsize + 4], "big")
    assert stored_crc == zlib.crc32(png[54:58 + zsize])

    fbits = np.unpackbits(np.frombuffer(png, np.uint8), bitorder="little")       # file-bit coordinate: bit i of the file
    Z = 8 * 58                                                                   # first zlib bit
    E = 8 * (58 + zsize)                                                         # end of the CRC'd message
    hdr_bits = oracle.static_table(chans)[2]                                     # zlib header + block header: tokens start here
    pieces = []                                                                  # (first bit, one past last bit) in file-bit coordinates
    pieces.append((Z - 32, Z))                                                   # "IDAT"
    for t in range((hdr_bits + 31) // 32):                                       # block header, one 32-bit piece per thread
        pieces.append((Z + 32 * t, Z + min(32 * t + 32, hdr_bits)))
    ofs = Z + hdr_bits
    for y in range(h):                                                           # one piece per scanline
        pieces.append((ofs, ofs + int(rows[y])))
        ofs += int(rows[y])
    tail_start = ofs                                                             # end-of-block code (+ zero padding: contributes nothing)
    pieces.append((tail_start, E - 32))
    pieces.append((E - 32, E))                                                   # Adler-32
    assert sorted(pieces) == pieces and all(a <= b for a, b in pieces)
    assert all(pieces[i][1] == pieces[i + 1][0] for i in range(len(pieces) - 1)) # the pieces tile the message exactly

    total = 0
    for a, b in pieces:
        if a == b:
            continue
        w0, w1 = a >> 5, ((b - 1) >> 5) + 1                                      # the 32-bit words the piece touches (file starts word aligned)
        end = min(32 * w1, E)                                                    # the message may end inside the last word (Adler-32 piece)
        span = np.zeros(end - 32 * w0, np.uint8)
        span[a - 32 * w0:b - 32 * w0] = fbits[a:b]                               # zeros outside the piece's own bits
        contribution = mulmod(raw_crc_bits(span), xpow(E - end))
        # fact 1: the same value from the bare bit string, whatever its alignment
        assert contribution == mulmod(raw_crc_bits(fbits[a:b]), xpow(E - b))
        total ^= contribution
    msg_bits = E - 8 * 54
    total ^= mulmod(0xFFFFFFFF, xpow(msg_bits)) ^ 0xFFFFFFFF                      # fact 3
    assert total == stored_crc


def test_mulmod_and_powers():
    assert mulmod(ONE, 0x12345678) == 0x12345678 and mulmod(0x40000000, ONE) == 0x40000000
    assert mulmod(xpow(5), xpow(27)) == xpow(32) == POLY                         # x^32 mod P = P's low terms
    assert mulmod(xpow(1000), 0xDB710641) == xpow(999)                           # x^-1 mod P
    # advancing a finished CRC over n zero bytes = multiplying its raw form by x^(8n)
    data = bytes(range(200))
    for n in (1, 7, 64):
        a = zlib.crc32(data) ^ 0xFFFFFFFF
        b = zlib.crc32(data + bytes(n)) ^ 0xFFFFFFFF
        init_fix = mulmod(0xFFFFFFFF, xpow(8 * len(data))), mulmod(0xFFFFFFFF, xpow(8 * (len(data) + n)))
        assert mulmod(a ^ init_fix[0], xpow(8 * n)) == b ^ init_fix[1]
