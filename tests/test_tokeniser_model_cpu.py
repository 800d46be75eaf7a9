"""CPU model of the data-parallel tokeniser the 16-pixel CUDA kernels implement (csrc/row_walk16.cuh classify16 +
lane_info16, csrc/encode16_kernels.cu run_before16 / put_event16), checked against the serial restatement of the
reference's tokeniser (fpng.cpp:1182-1243 / 1468-1558; oracle/fpng_oracle.c tokenise_row) -- which is itself pinned to the
oracle here through the per-row token bit counts `oracle_encode_ex` reports.

This is host logic (no GPU): it documents WHY 32 lanes of 16 pixels can emit their tokens independently.  A run of pixels
equal to their left neighbour is cut into matches of M pixels from the run start; a token belongs to the pixel where it
ends (full match), or to the literal / row end that follows it (remainder).  Per lane the kernels need only
  eqm  -- 16-bit mask "pixel k equals its left neighbour",
  r_in -- the unfinished run entering the lane (from the nearest lower lane holding a literal: one ballot + one shuffle),
and derive from them (a) the literal pixels, (b) the "events": a pending run flushed before a literal, or the run
reaching M at a match pixel (at most one per lane since M > 16).

RGBA 1-pass under a table whose "one-pixel match vs four literals" rule can fire (fpng.cpp:1520-1528; the kernels' LIT1
instantiations) a flushed match of exactly one pixel is written as the four literals of the pixel it covers when the match
costs more bits.  The serial coder knows that pixel as the last literal; a lane knows it as its own pixel k - 1, or at lane
pixel 0 as the lane to the left's pixel 15 (one shuffle), or for lane 0 as lane 31's pixel 15 of the previous step."""
import json
import os
import numpy as np
import pytest

import imagegen
from common import HERE

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_XBITS = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]


def len_symbol(L):
    """RFC 1951 length code (symbol, extra bits) of a match of L bytes (fpng.cpp:498-512)."""
    if L == 258:
        return 285, 0
    s = max(i for i in range(28) if LEN_BASE[i] <= L)
    return 257 + s, LEN_XBITS[s]


def filtered_pixels(img, y):
    """PNG filter 0 on row 0, filter 2 (Up) below (fpng.cpp:1592-1660); returns (filter byte, [w] packed pixels)."""
    h, w, c = img.shape
    row = img[y].astype(np.int16)
    d = row if y == 0 else (row - img[y - 1].astype(np.int16)) & 255
    d = d.astype(np.uint32)
    px = d[:, 0] | (d[:, 1] << 8) | (d[:, 2] << 16)
    if c == 4:
        px = px | (d[:, 3] << 24)
    return (0 if y == 0 else 2), [int(v) for v in px]


def lit1_takes_literals(sizes, p):
    """The one-pixel-match rule (fpng.cpp:1520-1528): a one-pixel match covering the RGBA pixel p is written as p's four
    literals iff the match (length code + extra bits + the 1-bit distance) costs more bits than they do."""
    sym, xb = len_symbol(4)
    return int(sizes[sym]) + xb + 1 > sum(int(sizes[(p >> (8 * c)) & 255]) for c in range(4))


def flush(out, n, covered, lit1):
    """Appends the token of a pending run of n pixels whose last pixel is `covered` (lit1: the RGBA table's code sizes)."""
    if n == 1 and lit1 is not None and lit1_takes_literals(lit1, covered):
        out.append(("L", covered))
    elif n:
        out.append(("M", n))


def serial_tokens(filt, px, M, lit1=None):
    out = [("F", filt)]
    prev, run = None, 0
    for x, p in enumerate(px):
        if x and p == prev:
            run += 1
            if run == M:
                out.append(("M", M)); run = 0
        else:
            flush(out, run, prev, lit1); run = 0
            out.append(("L", p)); prev = p
    flush(out, run, prev, lit1)
    return out


def run_before(eqm, r_in, kk, M):
    """Pending run length before pixel kk of a lane (encode16_kernels.cu run_before16)."""
    t = ~eqm & ((1 << kk) - 1)
    if t == 0:
        r = kk + r_in
        return r - M if r >= M else r
    return kk - 1 - (t.bit_length() - 1)


def parallel_tokens(filt, px, M, lit1=None, sites=None):
    """Tokens of one scanline as 32 lanes x 16 pixels per warp step produce them, lanes concatenated in order.  lit1: the RGBA
    table's code sizes, applying the one-pixel-match rule; sites (a Counter) counts where the rule took the literals."""
    w = len(px)
    out = [("F", filt)]
    carry_prev, carry_run = 0, 0
    for s0 in range(0, w, 512):
        lanes = []
        for lane in range(32):
            p0 = s0 + lane * 16
            nvp = min(16, w - p0) if p0 < w else 0
            lpx = [px[p0 + k] if k < nvp else 0 for k in range(16)]   # the lane's filtered pixels, zero beyond the row
            eqm = 0
            for k in range(nvp):
                x = p0 + k
                left = px[x - 1] if x > 0 else None
                if x > 0 and px[x] == left:
                    eqm |= 1 << k
            valid = (1 << nvp) - 1
            litm = valid & ~eqm
            trail = (nvp - 1 - (litm.bit_length() - 1)) if litm else nvp
            lanes.append(dict(p0=p0, nvp=nvp, eqm=eqm, litm=litm, trail=trail, px=lpx))
        # run phase entering each lane: the nearest lower lane with a literal decides (ballot + shuffle in classify16)
        for lane, t in enumerate(lanes):
            src = max((l for l in range(lane) if lanes[l]["litm"]), default=None)
            run = (lanes[src]["trail"] + 16 * (lane - src - 1)) if src is not None else (carry_run + 16 * lane)
            t["run"] = run % M
        last = lanes[31]
        carry_run = last["trail"] if last["litm"] else (last["run"] + last["nvp"]) % M
        # per-lane emission from (eqm, r_in) alone: literals + events; under the rule also the pixel left of the lane
        for lane, t in enumerate(lanes):
            eqm, litm, nvp, r_in, lpx = t["eqm"], t["litm"], t["nvp"], t["run"], t["px"]
            left = lanes[lane - 1]["px"][15] if lane else carry_prev
            lead = ((~eqm) & -(~eqm)).bit_length() - 1            # leading match pixels (ffs(~eqm) - 1)
            kM = M - 1 - r_in
            evm = (litm & ((eqm << 1) | (1 if r_in else 0))) | ((1 << kM) if kM < lead else 0)
            for k in range(nvp + 1):
                tail = k == nvp
                if tail and not (nvp and t["p0"] + nvp == w):     # the lane holding the scanline's last pixel flushes its run
                    break
                if tail or evm >> k & 1:
                    n = M if not tail and eqm >> k & 1 else run_before(eqm, r_in, k, M)
                    covered = lpx[k - 1] if k else left
                    if sites is not None and n == 1 and lit1 is not None and lit1_takes_literals(lit1, covered):
                        sites["row end" if tail else "mid-lane" if k else "lane 0, previous step" if lane == 0 else "lane pixel 0"] += 1
                    flush(out, n, covered, lit1)
                if not tail and litm >> k & 1:
                    out.append(("L", lpx[k]))
        carry_prev = last["px"][15]
    return out


def token_bits(tokens, sizes, chans):
    bits = 0
    for kind, v in tokens:
        if kind == "F":
            bits += int(sizes[v])
        elif kind == "L":
            bits += sum(int(sizes[(v >> (8 * c)) & 255]) for c in range(chans))
        else:
            sym, xb = len_symbol(v * chans)
            bits += int(sizes[sym]) + xb + 1                       # + the 1-bit distance code (fpng.cpp:1135)
    return bits


@pytest.mark.parametrize("chans", [3, 4])
@pytest.mark.parametrize("kind", ["g1", "g0", "runs", "mut", "zero"])
def test_lane_parallel_tokeniser_equals_serial_and_oracle(oracle, kind, chans):
    M = 85 if chans == 3 else 63
    sizes, _, _ = oracle.static_table(chans)
    for i, (w, h) in enumerate([(1, 3), (17, 2), (85, 3), (512, 4), (513, 3), (700, 5), (1100, 3), (2049, 2)]):
        img = imagegen.make(kind, w, h, chans, 7 + i)
        _, row_bits, stored = oracle.encode(img, w, h, chans, 0, want_rows=True)
        for y in range(h):
            filt, px = filtered_pixels(img, y)
            ser = serial_tokens(filt, px, M)
            par = parallel_tokens(filt, px, M)
            assert par == ser, (kind, chans, w, h, y)
            if not stored:   # the oracle reports each row's token bits of the compressed attempt
                assert token_bits(ser, sizes, chans) == int(row_bits[y]), (kind, chans, w, h, y)


def test_run_boundaries_at_max_match():
    """Runs that cross lanes, steps and the maximum match length M (255/3 and 252/4 pixels)."""
    for chans, M in ((3, 85), (4, 63)):
        for run_len in (M - 1, M, M + 1, 2 * M, 2 * M + 5, 511, 512, 513, 1030):
            for lead_in in (0, 1, 15, 16, 17, 500):
                px = list(range(1, lead_in + 1)) + [777] * run_len + [5, 5, 6]
                assert parallel_tokens(2, px, M) == serial_tokens(2, px, M), (chans, run_len, lead_in)


def test_one_pixel_match_rule_under_trained_rgba_table(oracle):
    """RGBA 1-pass under the fixture table of tests/golden/trained_tables.json, whose one-pixel-match rule fires: the lane-parallel
    tokens equal the serial ones and their bits equal the oracle's per-row counts, at widths on both sides of the 16-pixel lane
    and the 512-pixel step, with the rule taking the literals at every kind of site the kernels handle."""
    from collections import Counter
    with open(os.path.join(HERE, "golden", "trained_tables.json")) as f:
        t = json.load(f)["tables"]["4"]
    assert oracle.set_static_table(4, bytes.fromhex(t["prefix"]), t["bit_buf"], t["bit_buf_size"])
    try:
        sizes, _, _ = oracle.static_table(4)
        order = np.argsort(sizes[:256], kind="stable")
        cheap = [int(v) for v in order[:5]]
        pals = (cheap[:2], cheap + [int(order[40]), int(order[200])])   # the rule fires mostly / rarely
        images = [(name, img) for name, _, _, img in imagegen.trained_table_images(4, sizes)]
        for i, w in enumerate((15, 16, 17, 31, 33, 511, 512, 513, 527, 1023, 1024, 1025, 1553)):
            for j, pal in enumerate(pals):
                images.append((f"short_runs w={w} palette {j}", imagegen.short_runs(w, 24, 4, 300 + i, pal)))
            images.append((f"runs w={w}", imagegen.make("runs", w, 4, 4, 300 + i)))
        sites = Counter()
        for name, img in images:
            h, w, _ = img.shape
            _, row_bits, stored = oracle.encode(img, w, h, 4, 0, want_rows=True)
            assert not stored, name
            for y in range(h):
                filt, px = filtered_pixels(img, y)
                ser = serial_tokens(filt, px, 63, sizes)
                assert parallel_tokens(filt, px, 63, sizes, sites) == ser, (name, y)
                assert token_bits(ser, sizes, 4) == int(row_bits[y]), (name, y)
        for site in ("mid-lane", "lane pixel 0", "lane 0, previous step", "row end"):
            assert sites[site] > 0, (site, sites)
    finally:
        oracle.set_static_table(4)


def test_one_pixel_remainder_of_max_match_under_rule(oracle):
    """A run of M + 1 pixels ends in a one-pixel match: the rule applies to it, wherever the run sits in lanes and steps."""
    with open(os.path.join(HERE, "golden", "trained_tables.json")) as f:
        sizes = np.array(json.load(f)["tables"]["4"]["sizes"], np.uint8)
    cheap = int(np.argmin(sizes[:256]))
    assert lit1_takes_literals(sizes, cheap * 0x01010101)
    for lead_in in (0, 1, 15, 16, 17, 448, 449, 500):
        for tail in ([5, 5, 6], [], [cheap * 0x01010101 + 1]):
            px = list(range(1, lead_in + 1)) + [cheap * 0x01010101] * 65 + tail
            ser = serial_tokens(2, px, 63, sizes)
            assert ser.count(("L", cheap * 0x01010101)) == 2 and parallel_tokens(2, px, 63, sizes) == ser, (lead_in, tail)
