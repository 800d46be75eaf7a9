"""Seeded edge cases of the decoder's integrity check (fpngb_set_decode_verify) and a pure-Python model of how each of its four
GPU checksum paths cuts a message into pieces, so that every case can show the construct it reaches:

  * fpng files, IDAT CRC-32 -- idat_crc_stream_kernel<false, true> (csrc/crc_stream_kernel.cu).  The message "IDAT" + stream is
    bytes [m0, L) of the file.  Its whole 32-bit words [m0 / 4, L / 4) are counted from the END: CTA b takes the 64 KiB
    [wend - (b + 1) C, wend - b C) (C = kCs2WarpWords * kCs2Warps words), warp chunk m of it (from the CTA's end) 8 KiB, lane l
    word l of each 32-word step; the first word is masked below m0, the last CTA adds the L mod 4 tail bytes, and CTA b's value is
    shifted by x^(32 C b).
  * fpng files, Adler-32 -- decode_adler_kernel (csrc/decode_kernels.cu): one delta row per warp, kAdlerRows rows per CTA, each
    lane 16-byte vectors v = lane, lane + 32, ...; the last vector of a row is masked to bpl mod 16 bytes; the filter bytes are
    added in closed form (0 on row 0, 2 below in compressed files, 0 in stored files).
  * general PNGs, per-chunk CRC-32 -- png_gather_kernel (csrc/inflate_kernels.cu): the m = len + 4 message bytes of a chunk cut
    into kGatherThreads segments of ceil(m / kGatherThreads) bytes, segment t shifted by x^(8 (m - b1)).
  * general PNGs, Adler-32 -- the tail of png_inflate_kernel: the N inflated bytes in 32 lane ranges of ceil(N / 32) bytes, each
    lane's position counter starting at b0 mod 65521 and wrapping at 65521.

Every expected status comes from zlib (crc32, adler32, decompressobj) and the documented precedence: a bad IDAT CRC (4), then a
stream error (FPNG_DECODE_FAILED_INVALID_IDAT, 8, for general files), then an Adler-32 mismatch (102), then 0.  Nothing here asks
the library what the answer is.  tests/test_checksum_edges_cpu.py checks the numbers each case reports; tests/
test_checksum_edges_gpu.py runs the cases through every decode entry point.
"""
from __future__ import annotations

import os
import re
import struct
import zlib
from dataclasses import dataclass, field

import numpy as np

import imagegen
import pngwrite
import pngwrite_formats as pf
from common import with_text_chunk

# the kernels' partition constants: KERNEL_CONSTANTS ties each to its definition in the sources (checked by the CPU test)
CS2_WARP_WORDS = 2048            # crc_stream_kernel.cu: 8 KiB per warp
CS2_WARPS = 8                    # crc_stream_kernel.cu: warps per CTA
CS2_CTA_WORDS = CS2_WARP_WORDS * CS2_WARPS
ADLER_ROWS = 8                   # decode_kernels.cu: delta rows per CTA of decode_adler_kernel
GATHER_THREADS = 256             # inflate_kernels.cu: threads (CRC segments) per chunk
LANES = 32                       # lanes of a warp: Adler-32 vectors of a row, inflate Adler lane ranges, CRC words per step
ADLER_MOD = 65521
VEC = 16                         # decode_adler_kernel: bytes per vector load
KERNEL_CONSTANTS = {
    "kCs2WarpWords": ("crc_stream_kernel.cu", CS2_WARP_WORDS),
    "kCs2Warps": ("crc_stream_kernel.cu", CS2_WARPS),
    "kAdlerRows": ("decode_kernels.cu", ADLER_ROWS),
    "kGatherThreads": ("inflate_kernels.cu", GATHER_THREADS),
    "kAdlerMod": ("common.cuh", ADLER_MOD),
}
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "fpng_b200", "csrc")

OK, CRC, INVALID_IDAT, ADLER = 0, 4, 8, 102
FPNG_MSG_START = 54              # "IDAT" of an fpng file without ancillary chunks: signature, IHDR, fdEC, the IDAT length field


def source_constants():
    """{name: value} of KERNEL_CONSTANTS as the .cu sources define them (`constexpr uint32_t name = value;`)"""
    out = {}
    for name, (fname, _) in KERNEL_CONSTANTS.items():
        with open(os.path.join(CSRC, fname)) as fh:
            m = re.findall(r"constexpr\s+uint32_t\s+" + name + r"\s*=\s*(\d+)u?\s*;", fh.read())
        out[name] = int(m[0]) if len(m) == 1 else None
    return out


# ---- models of the partitions ----------------------------------------------------------------------------------------------------
def crc_ctas(m0, L):
    """CTAs the message [m0, L) takes in idat_crc_stream_kernel"""
    return -(-((L >> 2) - (m0 >> 2)) // CS2_CTA_WORDS)


def crc_grid(max_file_size):
    """gridDim.x of the verify launch: crc_stream_ctas_for(max_file_size)"""
    return (max_file_size // 4 + CS2_CTA_WORDS - 1) // CS2_CTA_WORDS + 1


def crc_place(m0, L, b):
    """where file byte b (m0 <= b < L) of the message falls: the tail index, or the CTA / warp chunk (both from the end), the
    lane step and lane in the chunk, whether it is in the first (masked) word, and the exponent of the CTA's shift"""
    j, wend = b >> 2, L >> 2
    if j >= wend:
        return dict(tail=b - 4 * wend)
    cta, e = divmod(wend - 1 - j, CS2_CTA_WORDS)
    warp, r = divmod(e, CS2_WARP_WORDS)
    step, lane = divmod(CS2_WARP_WORDS - 1 - r, LANES)
    return dict(tail=None, cta=cta, warp=warp, step=step, lane=lane, first_word=j == m0 >> 2, cta_shift=32 * CS2_CTA_WORDS * cta)


def crc_spans(m0, L):
    """byte ranges [first, last] of CTA b, warp chunk (b, m) and lane step (b, m, s), as functions of the message (file bytes)"""
    wend = L >> 2

    def cta(b):
        return 4 * (wend - (b + 1) * CS2_CTA_WORDS), 4 * (wend - b * CS2_CTA_WORDS) - 1

    def chunk(b, m):
        end = wend - b * CS2_CTA_WORDS - m * CS2_WARP_WORDS
        return 4 * (end - CS2_WARP_WORDS), 4 * end - 1

    def step(b, m, s):
        first = chunk(b, m)[0] + 4 * LANES * s
        return first, first + 4 * LANES - 1
    return cta, chunk, step


def crc_first_chunk(m0, L):
    """(words of the first CTA's first warp chunk inside the message, lane of the message's first word in it)"""
    w0, wend = m0 >> 2, L >> 2
    nctas = crc_ctas(m0, L)
    begin = wend - nctas * CS2_CTA_WORDS                       # first word of the first CTA (may lie before w0)
    k = (w0 - begin) // CS2_WARP_WORDS                          # the first warp chunk that reaches w0
    chunk_begin = begin + k * CS2_WARP_WORDS
    return chunk_begin + CS2_WARP_WORDS - w0, (w0 - chunk_begin) % LANES


def adler_rows(h):
    """(CTAs, rows of the last CTA) of decode_adler_kernel for h rows"""
    n = -(-h // ADLER_ROWS)
    return n, h - ADLER_ROWS * (n - 1)


def adler_vectors(bpl):
    """(vectors per row, bytes of the masked last vector (0: none masked), most vectors of one lane, lane of the last vector)"""
    nvec = -(-bpl // VEC)
    return nvec, bpl % VEC, -(-nvec // LANES), (nvec - 1) % LANES


def adler_place(bpl, y, x):
    """CTA, warp, lane and vector of delta byte (y, x), and whether that vector is the masked last one of its row"""
    v = x // VEC
    nvec, rem, _, _ = adler_vectors(bpl)
    return dict(cta=y // ADLER_ROWS, warp=y % ADLER_ROWS, lane=v % LANES, vector=v, masked=bool(rem) and v == nvec - 1)


def gather_segments(length):
    """(m, segment bytes, threads with a non-empty segment, bytes of the last non-empty one) of an IDAT chunk of `length` bytes"""
    m = length + 4
    seg = -(-m // GATHER_THREADS)
    used = -(-m // seg)
    return m, seg, used, m - seg * (used - 1)


def gather_place(length, i):
    """thread of message byte i (0: the 'I' of the tag) of a chunk, and the shift m - b1 its segment gets"""
    m, seg, _, _ = gather_segments(length)
    t = i // seg
    return dict(thread=t, shift=m - min(m, t * seg + seg))


def inflate_lanes(n):
    """bytes per lane range, lanes with an empty range, lanes whose range crosses a multiple of 65521, and whether some non-empty
    range starts at or past 65521"""
    per = -(-n // LANES)
    b0 = [min(n, per * k) for k in range(LANES)]
    b1 = [min(n, b + per) for b in b0]
    empty = sum(1 for a, b in zip(b0, b1) if a == b)
    wraps = [k for k, (a, b) in enumerate(zip(b0, b1)) if (b - 1) // ADLER_MOD > a // ADLER_MOD and b > a]
    return dict(per=per, empty=empty, wrap_lanes=wraps, start_past_mod=any(a >= ADLER_MOD for a, b in zip(b0, b1) if b > a))


def inflate_place(n, p):
    per = -(-n // LANES)
    return dict(lane=p // per, lane_offset=p % per, mod_pos=p % ADLER_MOD)


# ---- the zlib model: expected statuses --------------------------------------------------------------------------------------------
def chunks(png):
    """[(offset, type, data, stored CRC)] of every chunk after the signature"""
    out, at = [], 8
    while at + 12 <= len(png):
        n = struct.unpack(">I", png[at:at + 4])[0]
        out.append((at, png[at + 4:at + 8], png[at + 8:at + 8 + n], struct.unpack(">I", png[at + 8 + n:at + 12 + n])[0]))
        at += 12 + n
    return out


def idat_run(png):
    """the chunks of the (first) run of IDAT chunks"""
    cs = chunks(png)
    first = [k for k, c in enumerate(cs) if c[1] == b"IDAT"][0]
    run = []
    for c in cs[first:]:
        if c[1] != b"IDAT":
            break
        run.append(c)
    return run


def inflate(z):
    """(raw bytes or None for a stream zlib rejects, the 4 bytes after the final block or None): zlib's header rules, then raw
    Deflate; the Adler-32 is read, not checked"""
    if len(z) < 2 or (z[0] & 15) != 8 or (z[0] >> 4) > 7 or ((z[0] << 8) | z[1]) % 31 or (z[1] & 0x20):
        return None, None
    d = zlib.decompressobj(-15)
    try:
        raw = d.decompress(z[2:]) + d.flush()
    except zlib.error:
        return None, None
    if not d.eof:
        return None, None
    tail = d.unused_data
    return raw, (struct.unpack(">I", tail[:4])[0] if len(tail) >= 4 else None)


def expected(png, raw_len, filter_at):
    """(status with verify on, status with verify off) of a file: every IDAT chunk's CRC with zlib.crc32, the stream with zlib
    (inflated size raw_len, filter bytes at positions filter_at at most 4), the Adler-32 with zlib.adler32"""
    run = idat_run(png)
    crc_ok = all(zlib.crc32(b"IDAT" + data) & 0xFFFFFFFF == crc for _, _, data, crc in run)
    raw, adler = inflate(b"".join(c[2] for c in run))
    stream_ok = raw is not None and len(raw) == raw_len and all(raw[p] <= 4 for p in filter_at)
    off = OK if stream_ok else INVALID_IDAT
    if not crc_ok:
        return CRC, off
    if not stream_ok:
        return INVALID_IDAT, off
    return (OK if adler == zlib.adler32(raw) & 0xFFFFFFFF else ADLER), off


def rows_filter_at(h, stride):
    return range(0, h * stride, stride)


def ext_filter_at(w, h, bits, interlace):
    out, at = [], 0
    for (_, _, _, _, pw, ph) in pf.passes(w, h, interlace):
        rb = (pw * bits + 7) // 8
        for _ in range(ph):
            out.append(at)
            at += rb + 1
    return out


# ---- cases ------------------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str                    # the construct the case exists to reach
    png: bytes = field(repr=False)
    kind: str                    # "fpng", "png" (8-bit general: any_png) or "ext" (all_formats only)
    want: int                    # status with verify on (zlib)
    want_off: int                # status with verify off for general files (zlib); fpng files: the reference decoder's
    reach: dict                  # the numbers that show the construct is reached
    raw_len: int = 0
    filter_at: object = field(default=(), repr=False)
    pixels: np.ndarray = field(default=None, repr=False)   # general files: the expected pixels [h, w, c] with verify off

    def recheck(self):
        """(verify on, verify off) from zlib, for the CPU test"""
        return expected(self.png, self.raw_len, self.filter_at)


def fpng_shape(png):
    """(w, h, c, m0, L, idat offset, idat length) of an fpng file, from its chunks"""
    w, h = struct.unpack(">II", png[16:24])
    c = {2: 3, 6: 4}[png[25]]
    ofs = [a for a, t, _, _ in chunks(png) if t == b"IDAT"][0]
    n = struct.unpack(">I", png[ofs:ofs + 4])[0]
    return w, h, c, ofs + 4, ofs + 8 + n, ofs, n


def fpng_case(name, png, reach):
    w, h, c, m0, L, _, _ = fpng_shape(png)
    raw_len = h * (w * c + 1)
    on, off = expected(png, raw_len, rows_filter_at(h, w * c + 1))
    r = dict(m0_mod4=m0 % 4, tail=L % 4, msg_len=L - m0, ctas=crc_ctas(m0, L))
    r.update(reach)
    return Case(name, png, "fpng", on, off, r, raw_len, rows_filter_at(h, w * c + 1))


def rewrite_crc(png, ofs):
    """png with the CRC of the chunk at ofs recomputed"""
    b = bytearray(png)
    n = struct.unpack(">I", b[ofs:ofs + 4])[0]
    b[ofs + 8 + n:ofs + 12 + n] = struct.pack(">I", zlib.crc32(bytes(b[ofs + 4:ofs + 8 + n])) & 0xFFFFFFFF)
    return bytes(b)


def stored_message_len(w, h, c):
    """len("IDAT" + stream) of an fpng stored-block file: zlib header, 5 bytes per 65535-byte block, raw rows, Adler-32"""
    n = h * (w * c + 1)
    return 4 + 2 + 5 * -(-n // 65535) + n + 4


def shape_for_message(t):
    """(w, h, c) of an fpng stored-block file whose message is t bytes, or None when no stored stream is that long (just past a
    whole number of 65535-byte blocks: 65551..65555 for one block)"""
    for h in range(1, 257):
        for c in (3, 4):
            for blocks in range(1, t // 65535 + 3):
                n = t - 10 - 5 * blocks
                if n > 0 and -(-n // 65535) == blocks and n % h == 0 and (n // h - 1) % c == 0 and n // h - 1 >= c:
                    return (n // h - 1) // c, h, c
    return None


def noise(w, h, c, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, c)).astype(np.uint8)


def stored_file(oracle, t, seed, text=None):
    """an fpng stored-block file of noise whose message is t bytes, with a tEXt chunk of `text` bytes in front of IDAT"""
    w, h, c = shape_for_message(t)
    png = oracle.encode(noise(w, h, c, seed), w, h, c, 2)
    png = png if text is None else with_text_chunk(png, text)
    assert fpng_shape(png)[4] - fpng_shape(png)[3] == t
    return png


def crc_tail_cases(oracle):
    """clean files: every message length mod 4 (0..3 tail bytes) at every IDAT alignment; the masked bytes of the first word are
    the IDAT length field's, which must not be zero for a kernel that reads them to be caught"""
    out = []
    for k, t in enumerate((1000, 1001, 1002, 1003)):
        base = stored_file(oracle, t, 40 + k)
        for text in range(4):
            png = with_text_chunk(base, text)
            m0 = fpng_shape(png)[3]
            masked = bytes(png[m0 & ~3:m0])
            out.append(fpng_case(f"crc_tail{t % 4}_align{m0 % 4}", png, dict(masked=masked.hex())))
    return out


SIZE_KS = ((CS2_WARP_WORDS, (1, 2, 3, 8, 9)), (CS2_CTA_WORDS, (1, 2, 5)))
WORD_DELTAS = (-4, -3, -2, -1, 0, 1, 2, 3, 4)


def crc_size_cases(oracle):
    """clean files whose message is 8 KiB k and 64 KiB k bytes and those +- 1..4 words: a first warp chunk partly inside the
    message, exactly 1, 2 and many CTAs (lengths no stored stream has are left out)"""
    out = []
    for unit, ks in SIZE_KS:
        for k in ks:
            for d in WORD_DELTAS:
                t = 4 * (unit * k + d)
                if shape_for_message(t) is None:
                    continue
                png = stored_file(oracle, t, k * 17 + d)
                m0, L = fpng_shape(png)[3:5]
                inside, lane = crc_first_chunk(m0, L)
                out.append(fpng_case(f"crc_size_{unit * 4 // 1024}KiBx{k}{d:+d}w", png,
                                     dict(words=(L >> 2) - (m0 >> 2), first_chunk_words=inside, first_lane=lane,
                                          grid=crc_grid(len(png)))))
    return out


DAMAGE_MSG = 4 * (5 * CS2_CTA_WORDS + 3 * CS2_WARP_WORDS + 77) + 1     # six CTAs, a partial first warp chunk, three tail bytes (m0 = 54)


def crc_damage_cases(oracle):
    """one bit flipped, CRC field left as written, in a file of six CTAs: the first data byte (in the first CTA's masked first
    warp chunk), the last whole word, each tail byte, the first and last byte of a CTA, a warp chunk and a lane step"""
    png = stored_file(oracle, DAMAGE_MSG, 7)
    m0, L = fpng_shape(png)[3:5]
    cta, chunk, step = crc_spans(m0, L)
    wend = L >> 2
    spots = [("first_data_byte", m0 + 4), ("last_whole_word", 4 * wend - 4), ("last_whole_word_last_byte", 4 * wend - 1)]
    spots += [(f"tail_byte{t}", 4 * wend + t) for t in range(L % 4)]
    for what, (a, b) in (("cta2", cta(2)), ("cta0", cta(0)), ("chunk1.3", chunk(1, 3)), ("chunk4.7", chunk(4, 7)),
                         ("step0.5.17", step(0, 5, 17)), ("step3.0.63", step(3, 0, 63))):
        spots += [(f"{what}_first", a), (f"{what}_last", b)]
    out = []
    for k, (what, at) in enumerate(spots):
        b = bytearray(png)
        b[at] ^= 1 << (k % 8)
        out.append(fpng_case(f"crc_damage_{what}", bytes(b), dict(byte=at, place=crc_place(m0, L, at))))
    return out


GRID_WORDS = 4 * CS2_CTA_WORDS + 1


def crc_grid_cases(oracle):
    """files whose CTA count is the most crc_stream_ctas_for(size) leaves room for (its grid - 1): one word past 4 CTAs, with
    and without an ancillary chunk in front of IDAT; decoded with max_file_size = the largest file's size"""
    out = []
    for text in (None, 3):
        m0 = FPNG_MSG_START + (0 if text is None else 12 + text)
        png = stored_file(oracle, 4 * ((m0 >> 2) + GRID_WORDS) - m0 + 1, 5 + (text or 0), text)
        m0, L = fpng_shape(png)[3:5]
        out.append(fpng_case(f"crc_grid_text{text}", png, dict(grid=crc_grid(len(png)), words=(L >> 2) - (m0 >> 2))))
    return out


# ---- fpng Adler-32 -----------------------------------------------------------------------------------------------------------------
def _bpl_shape(bpl):
    for c in (3, 4):
        if bpl % c == 0:
            return bpl // c, c
    return None


def adler_widths():
    """row widths w * c in bytes: 16 k - 1 .. 16 k + 1, 512 (one vector per lane) +- 1..16, and every vector remainder"""
    want = [16 * k + d for k in (1, 2, 4, 32, 64) for d in (-1, 0, 1)] + [512 + d for d in range(-16, 17)]
    out = [b for b in dict.fromkeys(want) if _bpl_shape(b)]
    have = {b % VEC for b in out}
    for r in range(VEC):
        if r not in have:
            out.append(next(b for b in range(1024 + r, 4096, VEC) if _bpl_shape(b)))
    return out


ADLER_HEIGHTS = (1, 2, 7, 8, 9, 41)
MODES = ((0, "1pass"), (1, "2pass"), (2, "stored"))


def adler_image(w, h, c, seed):
    return imagegen.gradient_noise(w, h, c, seed)


def adler_size_cases(oracle):
    """clean 1-pass, 2-pass and stored files at the widths of adler_widths (heights cycling through 1, 2, 7, 8, 9, 8k + 1),
    w * c + 1 = 65521 (21840 x 3, 16380 x 4), and 70000 rows (the closed-form filter term and row positions wrap)"""
    shapes = []
    for k, bpl in enumerate(adler_widths()):
        w, c = _bpl_shape(bpl)
        shapes.append((w, ADLER_HEIGHTS[k % len(ADLER_HEIGHTS)], c))
    shapes += [(21840, 2, 3), (16380, 9, 4), (1, 70000, 3), (1, 70000, 4)]
    out = []
    for j, (w, h, c) in enumerate(shapes):
        for flags, mode in MODES:
            png = oracle.encode(adler_image(w, h, c, j), w, h, c, flags)
            nvec, rem, per_lane, last_lane = adler_vectors(w * c)
            ctas, last_rows = adler_rows(h)
            raw, _ = inflate(b"".join(x[2] for x in idat_run(png)))
            out.append(fpng_case(f"adler_{mode}_{w}x{h}x{c}", png,
                                 dict(bpl=w * c, h=h, nvec=nvec, rem=rem, per_lane=per_lane, last_lane=last_lane, ctas=ctas,
                                      last_rows=last_rows, row_mod=(w * c + 1) % ADLER_MOD,
                                      filters=sorted({raw[y * (w * c + 1)] for y in range(h)}),
                                      stored_blocks=(raw is not None and ((idat_run(png)[0][2][2] >> 1) & 3) == 0))))
    return out


T_W, T_H, T_C = 171, 19, 3                 # 513-byte rows: 33 vectors, the last masked to 1 byte; 3 row CTAs, the last of 3 rows
T_SPOTS = (("first_row_first_col", 0, 0), ("first_row_last_col", 0, T_W * T_C - 1), ("last_row_first_col", T_H - 1, 0),
           ("last_row_last_col", T_H - 1, T_W * T_C - 1), ("last_cta_mid", 17, 256), ("masked_vector", 5, 512),
           ("lane_boundary", 9, 495))


def transplant_fpng(oracle, flags, y, x, seed):
    """(file of A' carrying A's Adler-32, reach): A and A' differ in delta byte (y, x) only, which is 0 in A"""
    stored = flags == 2
    rs = np.random.RandomState(seed)
    delta = adler_image(T_W, T_H, T_C, seed).reshape(T_H, T_W * T_C)
    if not stored:
        delta = delta.astype(np.int16)
        delta[1:] = (delta[1:] - delta[:-1]) & 255
        delta = delta.astype(np.uint8)
    d = delta.copy()
    d[y, x] = 0
    d2 = d.copy()
    d2[y, x] = 1 + rs.randint(0, 255)
    def image(dd):
        dd = dd.reshape(T_H, T_W, T_C)
        return dd.copy() if stored else imagegen.from_deltas(dd)
    a, a2 = image(d), image(d2)
    pa = oracle.encode(a, T_W, T_H, T_C, flags)
    pb = oracle.encode(a2, T_W, T_H, T_C, flags)
    ofs, n = fpng_shape(pb)[5:7]
    ao, an = fpng_shape(pa)[5:7]
    b = bytearray(pb)
    b[ofs + 8 + n - 4:ofs + 8 + n] = pa[ao + 8 + an - 4:ao + 8 + an]
    return rewrite_crc(bytes(b), ofs), a2


def adler_transplant_cases(oracle):
    out = []
    for flags, mode in MODES:
        for k, (what, y, x) in enumerate(T_SPOTS):
            png, a2 = transplant_fpng(oracle, flags, y, x, 100 + k)
            case = fpng_case(f"adler_transplant_{mode}_{what}", png, dict(y=y, x=x, place=adler_place(T_W * T_C, y, x),
                                                                            row_ctas=adler_rows(T_H)))
            case.pixels = a2
            out.append(case)
    return out


def fpng_cases(oracle):
    return (crc_tail_cases(oracle) + crc_size_cases(oracle) + crc_damage_cases(oracle) + crc_grid_cases(oracle) +
            adler_size_cases(oracle) + adler_transplant_cases(oracle))


# ---- general PNGs: the gather CRC ----------------------------------------------------------------------------------------------
GATHER_LENS = (0, 1, 3, 4, 255, 256, 257, 511, 8192, 65537)
GATHER_RUNS = {"zero_first": GATHER_LENS,
               "zero_mid": (1, 3, 4, 255, 0, 256, 257, 511, 8192, 65537),
               "zero_last": (65537, 8192, 511, 257, 256, 255, 4, 3, 1, None, 0)}   # None: the rest of the stream
GW, GH, GC = 140, 140, 4


def general_file(img, z, parts=None, ctype=None):
    h, w, c = img.shape
    parts = [z] if parts is None else parts
    return pngwrite.SIG + pngwrite.ihdr(w, h, ctype=pngwrite.COLOR_TYPE[c] if ctype is None else ctype) + \
        b"".join(pngwrite.chunk(b"IDAT", p) for p in parts) + pngwrite.IEND


def split_lengths(z, lens):
    """z cut into chunks of the given lengths (None: what the later lengths leave), the rest of z in one more chunk"""
    parts, at = [], 0
    for k, n in enumerate(lens):
        n = len(z) - at - sum(lens[k + 1:]) if n is None else n
        parts.append(z[at:at + n])
        at += n
    if at < len(z):
        parts.append(z[at:])
    return parts


def png_case(name, png, img, reach, raw_len=None, filter_at=None, kind="png", pixels=None):
    h, w, c = img.shape
    raw_len = h * (w * c + 1) if raw_len is None else raw_len
    filter_at = rows_filter_at(h, w * c + 1) if filter_at is None else filter_at
    on, off = expected(png, raw_len, filter_at)
    return Case(name, png, kind, on, off, reach, raw_len, filter_at, img if pixels is None else pixels)


def gather_cases():
    """IDAT runs of chunks 0, 1, 3, 4, 255, 256, 257, 511, 8192 and 65537 bytes long, a zero-length chunk first, in the middle and
    last: clean, then one bit flipped in the first, a middle and the last chunk's data and in a zero-length chunk's CRC field"""
    img = noise(GW, GH, GC, 11)
    raw = pngwrite.filter_rows(img, pngwrite.row_filters(GH, 0))
    z = zlib.compress(raw, 0)
    out = []
    for name, lens in GATHER_RUNS.items():
        parts = split_lengths(z, lens)
        segs = [gather_segments(len(p)) for p in parts]
        png = general_file(img, z, parts)
        out.append(png_case(f"gather_{name}", png, img, dict(lens=[len(p) for p in parts], segments=segs)))
        if name != "zero_mid":
            continue
        run = idat_run(png)
        mid = [len(p) for p in parts].index(8192)
        zero = [len(p) for p in parts].index(0)
        last = len(parts) - 1
        for what, k, i in (("first_chunk", 0, 4), ("mid_chunk_first_seg", mid, 4), ("mid_chunk_last_byte", mid, len(parts[mid]) + 3),
                           ("mid_chunk_seg_first", mid, gather_segments(8192)[1] * 100),
                           ("mid_chunk_seg_last", mid, gather_segments(8192)[1] * 100 - 1), ("last_chunk", last, len(parts[last]) // 2 + 4)):
            b = bytearray(png)
            b[run[k][0] + 4 + i] ^= 0x10
            out.append(png_case(f"gather_damage_{what}", bytes(b), img,
                                dict(chunk=k, len=len(parts[k]), place=gather_place(len(parts[k]), i))))
        b = bytearray(png)
        b[run[zero][0] + 8] ^= 0x01                                           # the zero-length chunk's CRC field
        out.append(png_case("gather_damage_zero_len_crc", bytes(b), img, dict(chunk=zero, len=0)))
    return out


# ---- general PNGs: the inflate Adler-32 -------------------------------------------------------------------------------------------
def shape_for_raw(n, chans=(3, 4, 1, 2)):
    """(w, h, c) of an 8-bit general PNG whose inflated stream is n bytes"""
    for h in range(1, 4097):
        for c in chans:
            if n % h == 0 and n // h - 1 >= c and (n // h - 1) % c == 0:
                return (n // h - 1) // c, h, c
    raise ValueError(n)


INFLATE_NS = (2, 9, 21, 26, 31, ADLER_MOD - 1, ADLER_MOD + 1, 2 * ADLER_MOD - 1, 2 * ADLER_MOD + 1, 1024 * 2049)


def inflate_image(w, h, c, seed):
    return pngwrite.source("g1", w, h, c, seed)


def inflate_size_cases():
    """clean files of N = h (w c + 1) inflated bytes: N < 32 (lanes with empty ranges), N = 65521 k +- 1 (a lane range across a
    wrap), N / 32 >= 65521 (lane ranges that start past the modulus); and an Adler-32 field split across two IDAT chunks"""
    out = []
    for j, n in enumerate(INFLATE_NS):
        w, h, c = shape_for_raw(n)
        img = inflate_image(w, h, c, j)
        z = pngwrite.compress(pngwrite.filter_rows(img, pngwrite.row_filters(h, "random", j)))
        out.append(png_case(f"inflate_N{n}", general_file(img, z), img, dict(N=n, shape=(w, h, c), lanes=inflate_lanes(n))))
    img = inflate_image(61, 17, 3, 99)
    z = pngwrite.compress(pngwrite.filter_rows(img, pngwrite.row_filters(17, "random", 99)))
    for k in (1, 2, 3):
        out.append(png_case(f"inflate_adler_split{k}", general_file(img, z, [z[:-k], z[-k:]]), img, dict(adler_bytes_in_last_chunk=k)))
    return out


def transplant_raw(raw, p, filter_at, seed):
    """(A, A'): raw streams equal but at byte p, which is 0 in A (a filter byte becomes 0 and 1: both valid)"""
    a, a2 = bytearray(raw), bytearray(raw)
    a[p] = 0
    a2[p] = 1 if p in set(filter_at) else 1 + np.random.RandomState(seed).randint(0, 255)
    return bytes(a), bytes(a2)


def with_adler(z, adler):
    return z[:-4] + struct.pack(">I", adler & 0xFFFFFFFF)


def inflate_transplant_cases():
    """general files of A' carrying A's Adler-32 (zlib.compress(A') + adler32(A)), the changed byte at lane-range boundaries, at
    positions = 65520 (mod 65521) and at the stream's first and last byte; the same for an Adam7 16-bit and a palette file (the
    ext path); and a bad filter byte with a bad Adler-32 in an 8-bit and a palette file, which must give INVALID_IDAT"""
    out = []
    for n in (ADLER_MOD + 1, 1024 * 2049):
        w, h, c = shape_for_raw(n)
        img = inflate_image(w, h, c, 7)
        raw = pngwrite.filter_rows(img, pngwrite.row_filters(h, 2))
        fa = rows_filter_at(h, w * c + 1)
        per = -(-n // LANES)
        spots = [0, per - 1, per, 16 * per, 31 * per - 1, 31 * per, ADLER_MOD - 1, n - 1]
        if n > 2 * ADLER_MOD:
            spots += [2 * ADLER_MOD - 1, 3 * per + 5]
        for k, p in enumerate(spots):
            a, a2 = transplant_raw(raw, p, fa, k)
            png = general_file(img, with_adler(zlib.compress(a2, 1), zlib.adler32(a)))
            px = pngwrite.unfilter(a2, w, h, c)
            out.append(png_case(f"inflate_transplant_N{n}_p{p}", png, img, dict(N=n, p=p, place=inflate_place(n, p)), pixels=px))
    rs = np.random.RandomState(21)
    for name, (w, h, ctype, depth, interlace) in (("adam7_16bit", (23, 19, 2, 16, 1)), ("palette", (37, 11, 3, 8, 0))):
        s = pf.random_samples(rs, w, h, ctype, depth)
        plte = rs.randint(0, 256, (256, 3)).astype(np.uint8) if ctype == 3 else None
        bits = depth * pf.SAMPLES[ctype]
        raw = pf.raw_stream(s, ctype, depth, interlace, filters=0)
        fa = ext_filter_at(w, h, bits, interlace)
        img = np.zeros((h, w, 1), np.uint8)
        for what, p in (("mid", len(raw) // 2 + 1), ("last", len(raw) - 1)):
            p = p + 1 if p in set(fa) else p
            a, a2 = transplant_raw(raw, p, fa, 3)
            png = pf.make_png(s, ctype, depth, interlace, plte=plte, z=with_adler(zlib.compress(a2), zlib.adler32(a)))
            out.append(png_case(f"ext_transplant_{name}_{what}", png, img, dict(p=p, N=len(raw)), raw_len=len(raw), filter_at=fa,
                                kind="ext"))
        bad = bytearray(raw)
        bad[fa[1]] = 7
        png = pf.make_png(s, ctype, depth, interlace, plte=plte, z=with_adler(zlib.compress(bytes(bad)), zlib.adler32(bytes(bad)) ^ 1))
        out.append(png_case(f"ext_bad_filter_and_adler_{name}", png, img, dict(filter_row=1), raw_len=len(raw), filter_at=fa, kind="ext"))
    img = inflate_image(29, 13, 3, 5)
    raw = bytearray(pngwrite.filter_rows(img, pngwrite.row_filters(13, 0)))
    raw[29 * 3 + 1] = 9                                                     # row 1's filter byte
    png = general_file(img, with_adler(zlib.compress(bytes(raw)), zlib.adler32(bytes(raw)) ^ 0x10000))
    out.append(png_case("inflate_bad_filter_and_adler", png, img, dict(filter_row=1)))
    return out


def general_cases():
    return gather_cases() + inflate_size_cases() + inflate_transplant_cases()


# ---- past 2^32 bits ---------------------------------------------------------------------------------------------------------------
BIG_W, BIG_H, BIG_C = 16384, 8448, 4        # RGBA noise: stored blocks, an IDAT of 553 MB (more than 2^29 bytes)


def big_message_len():
    return stored_message_len(BIG_W, BIG_H, BIG_C)


def big_damage_spots():
    """file bytes flipped in the big file (CRC field left as written): the first data byte and a byte in the first CTA (the
    shift of the CTA reaches exponents >= 2^32), and one at the middle"""
    m0 = FPNG_MSG_START
    L = m0 + big_message_len()
    return [m0 + 4, m0 + 4 + 4 * CS2_CTA_WORDS, (m0 + L) // 2]
