"""CPU model of the parallel fpng decoder the CUDA kernels implement (csrc/decode_kernels.cu: decode_prepare_kernel's tables,
decode_scan_kernel / scan_window, decode_link_kernel, decode_write_kernel / decode_write_range, unfilter_kernel), run on files
written by the oracle and by the unmodified reference and checked against the pixels that went in.

This is host logic (no GPU).  The reference decodes ONE serial bit string per file (fpng.cpp:2253-2557 / 2631-2873); the
format has no row index, so the kernels cut the token bit string into subsequences of kSubBits bits and rely on three facts
this model exercises with the kernels' own rules:
  1. SCAN: a decoder started kPreRoll bits before a subsequence almost always falls onto the true token grid before it
     reaches the subsequence (prefix codes self-synchronise), so every subsequence can guess its first token boundary, and
     from there its exit (first boundary in the next subsequence), its output byte count and its last four literals;
  2. LINK: the first subsequence starts exactly, so "start[i] == exit[i-1] for all i" makes the guessed parse THE parse;
     the rare wrong guesses are decoded again from the known boundary.  Prefix sums of the byte counts and the "last four
     literals" monoid (lit_combine) then give every subsequence its output offset and the delta pixel a leading RLE match
     replicates -- the result never depends on the speculation having succeeded (checked here with the pre-roll set to 0);
  3. WRITE: given (start, output offset, previous literals) a subsequence is decoded and written with no other context; the
     model writes them in shuffled order.
The multi-token table (up to three literals, or a whole match incl. extra bits and the distance bit, per 12 stream bits) and
its cut rule at a subsequence boundary (fast_tok) are restated from the kernels as well.
"""
import random

import numpy as np
import pytest

import imagegen
from common import with_text_chunk as _with_text_chunk

K_SUB_BITS = 1024          # csrc/decode.cuh
K_PRE_ROLL = 256
K_LINK_THREADS = 1024      # subsequences per step of decode_link_kernel
POS_END, POS_ERR = -1, -2  # exit flags (kPosEnd / kPosErr)

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_XBITS = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]


class Bits:
    """the file's bytes from the 4-byte boundary at or before the zlib stream (the kernels' `Stream`: aligned 32-bit words);
    positions are bit offsets from that boundary, reads beyond the buffer give zeros"""

    def __init__(self, file: bytes, zofs: int):
        self.base = zofs & ~3
        self.bit0 = (zofs & 3) * 8
        self.buf = file[self.base:] + bytes(8)

    def peek(self, pos: int, n: int) -> int:
        b = pos >> 3
        return (int.from_bytes(self.buf[b:b + 5], "little") >> (pos & 7)) & ((1 << n) - 1)


def canonical_table(sizes, bits):
    """single-token look-up table over `bits` stream bits: (symbol, length) or (0, 0); None unless the code is complete or has
    exactly one code word (build_lut_warp; fpng.cpp:1836-1895)"""
    cnt = [0] * 16
    for s in sizes:
        cnt[s] += 1
    nxt, total = [0] * 17, 0
    for l in range(1, 16):
        total = (total + cnt[l]) << 1
        nxt[l + 1] = total
    if total != 0x10000 and sum(cnt[1:]) != 1:
        return None
    tab = [(0, 0)] * (1 << bits)
    seen = [0] * 16
    for sym, l in enumerate(sizes):
        if not l:
            continue
        code = nxt[l] + seen[l]
        seen[l] += 1
        if l > bits:
            continue
        rev = int(format(code, "0%db" % l)[::-1], 2)
        for c in range(rev, 1 << bits, 1 << l):
            tab[c] = (sym, l)
    return tab


def prepare(file: bytes, idat_ofs: int, idat_len: int, chans: int):
    """decode_prepare_kernel: block header -> (token_start in zlib bits, single-token table, fast table, literal sizes)"""
    z = file[idat_ofs + 8:]
    assert idat_len >= 7 and z[0] == 0x78 and z[1] == 0x01
    if (z[2] & 6) == 0:
        return None                                      # stored blocks
    assert (z[2] & 7) == 5                               # BFINAL = 1, BTYPE = 2
    src = Bits(z, 0)
    pos = 16 + 3
    nlit = src.peek(pos, 5) + 257; ndist = src.peek(pos + 5, 5) + 1; nclen = src.peek(pos + 10, 4) + 4
    pos += 14
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    cl = [0] * 19
    for i in range(nclen):
        cl[order[i]] = src.peek(pos, 3); pos += 3
    cltab = canonical_table(cl, 7)
    assert cltab is not None and nlit + ndist <= 288 + 32
    sizes = []
    while len(sizes) < nlit + ndist:
        s, l = cltab[src.peek(pos, 7)]
        assert l
        pos += l
        if s <= 15:
            assert s <= 12                               # fpng.cpp:2007
            sizes.append(s)
        elif s == 16:
            rep = src.peek(pos, 2) + 3; pos += 2
            sizes += [sizes[-1]] * rep
        elif s == 17:
            rep = src.peek(pos, 3) + 3; pos += 3
            sizes += [0] * rep
        else:
            rep = src.peek(pos, 7) + 11; pos += 7
            sizes += [0] * rep
    assert len(sizes) == nlit + ndist
    dist = sizes[nlit:]
    ones = sum(1 for d in dist if d == 1)                # fpng.cpp:2058-2074
    assert 1 <= ones <= 2 and dist[chans - 1] == 1 and (ones == 1 or dist[chans] == 1)
    lit = sizes[:nlit] + [0] * (288 - nlit)
    base = canonical_table(lit, 12)
    assert base is not None
    fast = []
    for i in range(4096):
        sym0, len0 = base[i]
        fe = (0, 0, 0)                                   # (L, literal count, payload)
        if len0 and sym0 < 256:
            L, cnt, P = len0, 1, sym0
            for k in (1, 2):
                sym1, len1 = base[i >> L]
                if not len1 or sym1 >= 256 or L + len1 > 12:
                    break
                P |= sym1 << (8 * k); L += len1; cnt += 1
            fe = (L, cnt, P)
        elif len0 and 256 < sym0 <= 285:
            xb = LEN_XBITS[sym0 - 257]
            if len0 + xb + 1 <= 12:
                fe = (len0 + xb + 1, 0, LEN_BASE[sym0 - 257] + ((i >> len0) & ((1 << xb) - 1)))
        fast.append(fe)
    return pos, base, fast, lit


class Model:
    def __init__(self, file: bytes, info, pre_roll=K_PRE_ROLL):
        st, self.w, self.h, self.chans, idat_ofs, self.idat_len = info
        assert st == 0
        self.bits = Bits(file, idat_ofs + 8)
        self.pre_roll = pre_roll
        self.token_start, self.base, self.fast, self.lit_sizes = prepare(file, idat_ofs, self.idat_len, self.chans)
        self.tok0 = self.token_start + self.bits.bit0                      # file_span()
        endbit = (self.idat_len - 4) * 8 + self.bits.bit0
        self.g0 = self.tok0 // K_SUB_BITS
        self.g1 = max(self.g0, (endbit - 1) // K_SUB_BITS)
        self.repairs = 0

    # ---- one token at absolute position `pos`; tokens of a multi-literal entry that could start at or beyond `limit` are cut off
    def fast_tok(self, pos, limit):
        w = self.bits.peek(pos, 32)
        L, cnt, P = self.fast[w & 4095]
        if cnt >= 2 and pos + 12 > limit:
            P &= 0xFF; cnt = 1; L = self.lit_sizes[P]
        return L, cnt, P, w

    def slow_tok(self, w):
        sym, l0 = self.base[w & 4095]
        if not l0 or sym > 285:
            return 0, sym, 0
        if sym <= 256:
            return l0, sym, 0
        xb = LEN_XBITS[sym - 257]
        return l0 + xb + 1, sym, LEN_BASE[sym - 257] + ((w >> l0) & ((1 << xb) - 1))

    # ---- scan_window: tokens starting in [lo, hi), decoder started at `origin` <= lo
    def scan(self, origin, lo, hi):
        pos = origin
        while pos < lo:                                                    # pre-roll: lock on to the token grid
            L, cnt, P, w = self.fast_tok(pos, lo)
            if L:
                pos += L; continue
            l, sym, run = self.slow_tok(w)
            if not l or sym == 256:
                pos = lo; break                                            # not locked on
            pos += l
        first = pos
        lits = n_out = nlit = 0
        while pos < hi:
            L, cnt, P, w = self.fast_tok(pos, hi)
            if L:
                pos += L
                n_out += cnt if cnt else P
                nlit += cnt
                lits = ((lits | (P << 32)) >> (8 * cnt)) & 0xFFFFFFFF      # funnel shift: the new literals enter at the top
                continue
            l, sym, run = self.slow_tok(w)
            if not l:
                return dict(start=first, exit=POS_ERR, eob_end=0, n_out=n_out, nlit=min(nlit, 4), lits=lits)
            pos += l
            if sym == 256:
                return dict(start=first, exit=POS_END, eob_end=pos, n_out=n_out, nlit=min(nlit, 4), lits=lits)
            if sym < 256:
                n_out += 1; nlit += 1; lits = (lits >> 8) | (sym << 24)
            else:
                n_out += run
        return dict(start=first, exit=pos, eob_end=0, n_out=n_out, nlit=min(nlit, 4), lits=lits)

    def scan_all(self):
        subs = []
        for g in range(self.g0, self.g1 + 1):
            lo = g * K_SUB_BITS
            if g == self.g0:
                subs.append(self.scan(self.tok0, self.tok0, lo + K_SUB_BITS))     # the first subsequence starts exactly
            else:
                subs.append(self.scan(max(self.tok0, lo - self.pre_roll), lo, lo + K_SUB_BITS))
        return subs

    @staticmethod
    def lit_combine(n, v, nb, vb):
        """`a then b` of the keep-the-last-four-literals monoid (most recent literal in the top byte)"""
        if nb >= 4:
            return 4, vb
        if nb == 0:
            return n, v
        return min(n + nb, 4), ((v >> (8 * nb)) | (vb & (0xFFFFFFFF << (8 * (4 - nb))))) & 0xFFFFFFFF

    # ---- decode_link_kernel
    def link(self, subs):
        total_out = (self.w * self.chans + 1) * self.h
        want, out_pos, ln, lv = self.tok0, 0, 0, 0
        jobs, done, err, eob_end = [], False, False, 0
        for i, s in enumerate(subs):
            g = self.g0 + i
            if want != s["start"]:                                         # wrong guess: decode again from the known boundary
                self.repairs += 1
                hi = (g + 1) * K_SUB_BITS
                s = dict(start=want, exit=want, eob_end=0, n_out=0, nlit=0, lits=0) if want >= hi else self.scan(want, want, hi)
            if out_pos + s["n_out"] > total_out:
                err = True; break
            jobs.append(dict(g=g, start=s["start"], out_pos=out_pos, n_out=s["n_out"], tail=lv))
            out_pos += s["n_out"]
            ln, lv = self.lit_combine(ln, lv, s["nlit"], s["lits"])
            if s["exit"] == POS_END:
                done, eob_end = True, s["eob_end"]; break
            if s["exit"] == POS_ERR:
                err = True; break
            want = s["exit"]
        used = (eob_end - self.bits.bit0 + 7) >> 3 if eob_end >= self.bits.bit0 else 0
        ok = (not err) and done and out_pos == total_out and used + 4 == self.idat_len      # fpng.cpp:2559-2584
        return ok, jobs

    # ---- decode_link_kernel as the device runs it: chunks of K_LINK_THREADS subsequences; inside a chunk every iteration repairs
    # ALL mismatches at once against the exits of the previous iteration, until no start moves; the chunk's last exit is the
    # carry into the next chunk.  A subsequence whose predecessor is repaired in the same iteration may have to be repaired
    # again, so the repair count can exceed the number of subsequences (fpngb_debug_decode_repairs counts the same way).
    def link_parallel(self, subs, max_iters=None):
        """-> (ok, jobs, repairs, iterations per chunk); `max_iters` cuts the loop short (to show the tests discriminate)"""
        total_out = (self.w * self.chans + 1) * self.h
        carry_start, carry_out, ln, lv = self.tok0, 0, 0, 0
        jobs, done, err, eob_end, repairs, iters = [], False, False, 0, 0, []
        pos = lambda x: x >= 0                                             # a real position, not POS_END / POS_ERR
        for base in range(0, len(subs), K_LINK_THREADS):
            chunk = [dict(s) for s in subs[base:base + K_LINK_THREADS]]
            pad = K_LINK_THREADS - len(chunk)                              # threads without a subsequence: exit = kPosErr
            it = 0
            while max_iters is None or it < max_iters:
                exits = [s["exit"] for s in chunk]
                bad = [t for t, s in enumerate(chunk) if pos(carry_start if t == 0 else exits[t - 1])
                       and (carry_start if t == 0 else exits[t - 1]) != s["start"]]
                if not bad:
                    break
                it += 1
                for t in bad:
                    want = carry_start if t == 0 else exits[t - 1]
                    hi = (self.g0 + base + t + 1) * K_SUB_BITS
                    chunk[t] = dict(start=want, exit=want, eob_end=0, n_out=0, nlit=0, lits=0) if want >= hi else self.scan(want, want, hi)
                repairs += len(bad)
            iters.append(it)
            first_bad = next((t for t, s in enumerate(chunk) if not pos(s["exit"])), len(chunk) if pad else K_LINK_THREADS)
            for t, s in enumerate(chunk[:first_bad + 1]):
                if carry_out + s["n_out"] > total_out:
                    err = True
                jobs.append(dict(g=self.g0 + base + t, start=s["start"], out_pos=carry_out, n_out=s["n_out"], tail=lv))
                carry_out += s["n_out"]
                ln, lv = self.lit_combine(ln, lv, s["nlit"], s["lits"])
            if first_bad < len(chunk):
                if chunk[first_bad]["exit"] == POS_END:
                    done, eob_end = True, chunk[first_bad]["eob_end"]
                else:
                    err = True
            carry_start = chunk[-1]["exit"] if not pad else POS_ERR
            if carry_out > total_out:
                err = True
            if done or err:
                break
        used = (eob_end - self.bits.bit0 + 7) >> 3 if eob_end >= self.bits.bit0 else 0
        ok = (not err) and done and carry_out == total_out and used + 4 == self.idat_len      # fpng.cpp:2559-2584
        return ok, jobs, repairs, iters

    def decode_parallel(self, shuffle_seed=0, max_iters=None):
        """decode() with the link pass of the device (link_parallel) -> (pixels or None, repairs, iterations per chunk)"""
        ok, jobs, repairs, iters = self.link_parallel(self.scan_all(), max_iters)
        return (self.write_jobs(jobs, shuffle_seed) if ok else None), repairs, iters

    # ---- decode_write_range: one subsequence, no other context
    def write(self, job, stream: bytearray):
        chans, bpl, h = self.chans, self.w * self.chans, self.h
        hi = (job["g"] + 1) * K_SUB_BITS
        pos, lits, o = job["start"], job["tail"], job["out_pos"]
        while pos < hi:
            L, cnt, P, w = self.fast_tok(pos, hi)
            if L and cnt:
                pos += L
                for k in range(cnt):
                    v = (P >> (8 * k)) & 0xFF
                    lits = (lits >> 8) | (v << 24)
                    row, col = divmod(o, bpl + 1)
                    if row >= h or (col == 0 and v != (2 if row else 0)):   # fpng.cpp:2264, 2642: filter 0 on the first scanline, Up below
                        return False
                    stream[o] = v; o += 1
                continue
            if L:
                pos += L; run = P
            else:
                l, sym, run = self.slow_tok(w)
                if not l:
                    return False
                if sym == 256:
                    break
                pos += l
                assert sym > 256                                          # every literal is a fast entry
            row, col = divmod(o, bpl + 1)
            dcol = col - 1                                                 # fpng.cpp:2302-2315, 2681-2691, 2727
            if row >= h or col == 0 or dcol < chans or dcol % chans or run % chans or dcol + run > bpl:
                return False
            px = lits if chans == 4 else lits >> 8                         # the last `chans` literals, oldest in the low byte
            for k in range(run):
                stream[o + k] = (px >> (8 * (k % chans))) & 0xFF
            o += run
        return o == job["out_pos"] + job["n_out"]

    def decode(self, shuffle_seed=0):
        ok, jobs = self.link(self.scan_all())
        return self.write_jobs(jobs, shuffle_seed) if ok else None

    def write_jobs(self, jobs, shuffle_seed):
        bpl = self.w * self.chans
        stream = bytearray((bpl + 1) * self.h)
        order = list(range(len(jobs)))
        random.Random(shuffle_seed).shuffle(order)
        for j in order:
            if not self.write(jobs[j], stream):
                return None
        rows = np.frombuffer(bytes(stream), np.uint8).reshape(self.h, bpl + 1)
        assert np.array_equal(rows[:, 0], np.array([0] + [2] * (self.h - 1), np.uint8))
        # unfilter_kernel: running byte-wise sum down the columns (fpng.cpp:2439-2466)
        return np.cumsum(rows[:, 1:].astype(np.uint32), axis=0).astype(np.uint8).reshape(-1)


CASES = [("g1", 160, 24, 3, 0), ("g1", 97, 31, 4, 0), ("g0", 256, 40, 4, 0), ("g0", 333, 20, 3, 0), ("runs", 300, 17, 3, 0),
         ("g1", 128, 32, 3, 1), ("g1", 64, 48, 4, 1), ("runs", 301, 9, 4, 1), ("g0", 1100, 6, 3, 1),
         ("g1", 640, 200, 3, 0), ("g1", 512, 128, 4, 1)]        # > 900 subsequences each


@pytest.mark.parametrize("kind,w,h,chans,flags", CASES)
def test_parallel_decoder_model_recovers_pixels(oracle, kind, w, h, chans, flags):
    import fpng_b200
    img = imagegen.make(kind, w, h, chans, 5)
    png = oracle.encode(img, w, h, chans, flags)
    for pad in range(4):                                                   # all four alignments of the zlib stream inside its word
        f = png if pad == 0 else _with_text_chunk(png, pad)
        info = fpng_b200.get_info_ex(f)
        m = Model(f, info)
        assert m.bits.bit0 == 8 * ((info[4] + 8) & 3)
        px = m.decode(shuffle_seed=pad)
        assert px is not None and np.array_equal(px, np.asarray(img).reshape(-1)), (kind, w, h, chans, flags, pad)
        assert oracle.decode(f, chans)[0] == 0
    assert {8 * ((fpng_b200.get_info_ex(_with_text_chunk(png, p))[4] + 8) & 3) for p in range(4)} == {0, 8, 16, 24}


def test_result_does_not_depend_on_speculation(oracle):
    """pre-roll 0 = every guess is "my subsequence starts on a token boundary" (almost always wrong): the link pass repairs
    all of them and the pixels are the same"""
    import fpng_b200
    w, h, chans = 200, 12, 3
    img = imagegen.make("g1", w, h, chans, 9)
    png = oracle.encode(img, w, h, chans, 0)
    info = fpng_b200.get_info_ex(png)
    good, blind = Model(png, info), Model(png, info, pre_roll=0)
    a, b = good.decode(), blind.decode()
    assert np.array_equal(a, np.asarray(img).reshape(-1)) and np.array_equal(b, a)
    nsub = good.g1 - good.g0 + 1
    assert nsub > 20 and blind.repairs > nsub // 2                        # the blind guesses really were wrong
    assert good.repairs <= nsub // 10                                     # 256 bits of pre-roll lock on (almost) always


def test_reference_written_file_and_truncation(oracle, ref):
    import fpng_b200
    w, h, chans = 144, 20, 4
    img = imagegen.make("g1", w, h, chans, 3)
    for flags in (0, 1):
        png = ref.encode(img, w, h, chans, flags)
        m = Model(png, fpng_b200.get_info_ex(png))
        assert np.array_equal(m.decode(), np.asarray(img).reshape(-1))
    # a stream whose last token bytes are cut away (IDAT shortened, CRC not checked by the decoder): no EOB where the link pass
    # needs it -> rejected, like the reference (FPNG_DECODE_NOT_FPNG)
    st, ww, hh, cc, ofs, ln = fpng_b200.get_info_ex(png)
    cut = 40
    bad = png[:ofs] + (ln - cut).to_bytes(4, "big") + png[ofs + 4:ofs + 8 + ln - cut - 4] + png[ofs + 8 + ln - 4:]
    info = fpng_b200.get_info_ex(bad)
    assert info[0] == 0 and ref.decode(bad, chans)[0] == 1
    ok, _ = (lambda mm: mm.link(mm.scan_all()))(Model(bad, info))
    assert not ok


def model_repairs(file: bytes, pre_roll=K_PRE_ROLL):
    """subsequences decode_link_kernel decodes again for `file` (fpngb_debug_decode_repairs after one decode of it): 0 when the
    decoder never reaches the link pass (container or block header rejected, stored blocks)"""
    import fpng_b200
    info = fpng_b200.get_info_ex(file)
    if info[0] != 0:
        return 0
    try:
        m = Model(file, info, pre_roll=pre_roll)
    except (AssertionError, IndexError, TypeError):                         # prepare() rejected the header / stored blocks
        return 0
    return m.link_parallel(m.scan_all())[2]


# Slow-synchronising files: Up-filtered bytes uniform over k values (imagegen "u<k>").  Encoded 2-pass, the per-image table is
# close to a fixed-length code and wrong subsequence starts hardly ever fall back onto the token grid within the pre-roll; the
# link pass repairs most subsequences, in chains that take several iterations per chunk.  1-pass uses the shipped table (k = 128
# and 64 then fall back to stored blocks).  Floors: repairs per subsequence, and the most iterations any chunk needed.
U_CASES = [("u128", 640, 100, 3, 1, 1.2, 6), ("u128", 400, 100, 4, 1, 1.2, 6), ("u64", 520, 120, 3, 1, 0.6, 4),
           ("u16", 720, 100, 4, 1, 0.1, 2), ("u2", 700, 140, 4, 0, 0.1, 2)]


@pytest.mark.parametrize("kind,w,h,chans,flags,min_rate,min_iters", U_CASES)
def test_link_loop_recovers_slow_synchronising_files(oracle, kind, w, h, chans, flags, min_rate, min_iters):
    import fpng_b200
    img = imagegen.make(kind, w, h, chans, 1)
    png = oracle.encode(img, w, h, chans, flags)
    for pad in range(4):                                                   # all four alignments of the zlib stream inside its word
        f = png if pad == 0 else _with_text_chunk(png, pad)
        m = Model(f, fpng_b200.get_info_ex(f))
        nsub = m.g1 - m.g0 + 1
        px, repairs, iters = m.decode_parallel(shuffle_seed=pad)
        assert px is not None and np.array_equal(px, np.asarray(img).reshape(-1)), (kind, w, h, chans, flags, pad)
        assert nsub > K_LINK_THREADS and len(iters) >= 2, nsub                # the carry between chunks is exercised
        assert repairs >= min_rate * nsub and max(iters) >= min_iters, (kind, pad, nsub, repairs, iters)
        assert m.link(m.scan_all())[0]                                     # the serial restatement agrees
        if min_iters >= 2:                                                 # a loop cut after one iteration must not recover them
            assert Model(f, fpng_b200.get_info_ex(f)).decode_parallel(max_iters=1)[0] is None


def test_uniform_delta_files_match_reference(oracle, ref):
    """the u-kind files of the CPU and GPU tests are what the unmodified reference encoder writes"""
    shapes = [c[:5] for c in U_CASES] + [(k, w, h, c, f) for k in ("u128", "u64", "u16", "u2") for (w, h) in ((1024, 160), (1920, 200))
                                         for c in (3, 4) for f in (0, 1)]
    for kind, w, h, chans, flags in shapes:
        img = imagegen.make(kind, w, h, chans, 1)
        assert oracle.encode(img, w, h, chans, flags) == ref.encode(img, w, h, chans, flags), (kind, w, h, chans, flags)


def test_parallel_link_restates_serial_link_on_ordinary_files(oracle):
    """on files that lock on within the pre-roll the device loop and the serial chain agree, and pre-roll 0 forces repairs in
    both; the parallel count is never below the serial one (a repaired subsequence may be repaired again)"""
    import fpng_b200
    for kind, w, h, chans, flags in (("g1", 640, 200, 3, 0), ("runs", 300, 17, 3, 0), ("g0", 1100, 6, 3, 1)):
        img = imagegen.make(kind, w, h, chans, 5)
        png = oracle.encode(img, w, h, chans, flags)
        for pre_roll in (K_PRE_ROLL, 0, 13):
            m = Model(png, fpng_b200.get_info_ex(png), pre_roll=pre_roll)
            subs = m.scan_all()
            ok, jobs = m.link(subs)
            pok, pjobs, repairs, iters = m.link_parallel(subs)
            assert ok and pok and jobs == pjobs and repairs >= m.repairs, (kind, pre_roll)
            if pre_roll == 0:
                assert repairs > (m.g1 - m.g0) // 2
