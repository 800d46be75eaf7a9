"""CPU budget of the pack kernel (pack_rows16_kernel, csrc/encode16_kernels.cu) on bench.py's g1 workloads.

Counts, from the real inputs, what the kernel's time depends on and what no CUDA-event time shows:
  * how many 8-pixel halves (32 lanes x 8 pixels) take each of the four warp-uniform emission paths
    (1) all literal, no run pending  (2) no literal  (3) mixed, >= 16 literals  (4) sparse literals;
  * output (code) words per warp step, which the flush loop stores and folds into the scanline CRC;
  * shared-memory wavefronts of the literal look-ups of path (1) (64-bit (code, size) entries: two half-warp passes, each
    as many wavefronts as the most distinct words any one bank holds) and of the scanline-CRC look-ups (byte tables
    [4][256] against nibble tables [8][16]), simulated from the actual table indices: the filtered bytes, and the CRC
    register of each lane of the lane-strided Horner run over the scanline's code words of the reference file.

The lane records follow the CPU model of tests/test_tokeniser_model_cpu.py (checked there against the serial tokeniser and the
oracle).  For every sampled scanline the tokens rebuilt from the records here must equal the model's serial tokens, so the
counts rest on the same classification the kernels use.  Host only, no GPU.

    python tools/pack_budget.py [--workload c2] [--images 4] [--rows 24]
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (WORKLOADS, workload_image: the benchmark's own generator)
import test_tokeniser_model_cpu as model  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402

CRC_POLY = 0xEDB88320


def advance_tables() -> np.ndarray:
    """[4][256] tables of the kernel's Horner step: byte k of the register advanced over 128 bytes (linear in the byte)."""
    t0 = np.zeros(256, np.uint32)
    for n in range(256):
        c = n
        for _ in range(8):
            c = (CRC_POLY ^ (c >> 1)) if c & 1 else (c >> 1)
        t0[n] = c
    reg = (np.arange(256, dtype=np.uint32)[None, :] << (8 * np.arange(4, dtype=np.uint32)[:, None])).astype(np.uint32)
    for _ in range(128):                                  # raw CRC of 128 zero bytes from register `reg`
        reg = (reg >> np.uint32(8)) ^ t0[reg & np.uint32(0xFF)]
    return reg


def lane_records(px: list[int], M: int):
    """Per warp step and lane: (eqm, litm, r_in, evm, nvp), as classify16 / the pack kernel derive them (the model's formulas;
    tokens_from_records() turns them back into the token list, which main() checks against the serial tokeniser)."""
    w = len(px)
    a = np.asarray(px, dtype=np.int64)
    eq = np.zeros(w, bool)
    eq[1:] = a[1:] == a[:-1]
    carry_run, steps = 0, []
    for s0 in range(0, w, 512):
        lanes = []
        for lane in range(32):
            p0 = s0 + 16 * lane
            nvp = min(16, w - p0) if p0 < w else 0
            eqm = int(sum(1 << k for k in range(nvp) if eq[p0 + k]))
            litm = ((1 << nvp) - 1) & ~eqm
            trail = (nvp - 1 - (litm.bit_length() - 1)) if litm else nvp
            lanes.append([eqm, litm, trail, nvp, 0])
        for lane, t in enumerate(lanes):
            src = max((q for q in range(lane) if lanes[q][1]), default=None)
            t[4] = ((lanes[src][2] + 16 * (lane - src - 1)) if src is not None else (carry_run + 16 * lane)) % M
        last = lanes[31]
        carry_run = last[2] if last[1] else (last[4] + last[3]) % M
        recs = []
        for eqm, litm, _, nvp, r_in in lanes:
            lead = ((~eqm) & -(~eqm)).bit_length() - 1
            kM = M - 1 - r_in
            evm = (litm & ((eqm << 1) | (1 if r_in else 0))) | ((1 << kM) if kM < lead else 0)
            recs.append((eqm, litm, r_in, evm, nvp))
        steps.append(recs)
    return steps


def tokens_from_records(filt: int, px: list[int], steps, M: int):
    """The scanline's tokens as the lanes emit them from their records alone: per pixel an event (a pending run flushed, or the
    run reaching M) before its literal; the lane holding the last pixel flushes the trailing run."""
    out = [("F", filt)]
    for s, recs in enumerate(steps):
        for lane, (eqm, litm, r_in, evm, nvp) in enumerate(recs):
            p0 = 512 * s + 16 * lane
            for k in range(nvp):
                if evm >> k & 1:
                    n = M if eqm >> k & 1 else model.run_before(eqm, r_in, k, M)
                    if n:
                        out.append(("M", n))
                if litm >> k & 1:
                    out.append(("L", px[p0 + k]))
            if nvp and p0 + nvp == len(px):
                n = model.run_before(eqm, r_in, nvp, M)
                if n:
                    out.append(("M", n))
    return out


def lds64_wavefronts(idx: np.ndarray) -> int:
    """32 lanes' 64-bit loads of entries idx (8 bytes each): two half-warp passes."""
    total = 0
    for half in (idx[:16], idx[16:]):
        words = np.unique(np.concatenate([2 * half, 2 * half + 1]))
        total += int(np.bincount(words % 32, minlength=32).max())
    return total


def lds32_wavefronts(words: np.ndarray) -> int:
    return int(np.bincount(np.unique(words) % 32, minlength=32).max()) if words.size else 0


def split_wavefronts(idx: np.ndarray, copies: int) -> int:
    """The same 32-bit look-ups into a table replicated `copies` times, copy g confined to banks [g * 32 / copies, (g + 1) * 32 /
    copies) and read by lanes [g * 32 / copies, (g + 1) * 32 / copies): a lane group's indices only collide among themselves."""
    nb = 32 // copies
    g = np.arange(idx.size) // nb
    banks = g * nb + idx % nb
    addr = g * 4096 + idx                                  # distinct words: (copy, entry)
    _, first = np.unique(addr, return_index=True)
    return int(np.bincount(banks[first], minlength=32).max())


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--rows", type=int, default=24, help="scanlines sampled per image (evenly spaced, row 0 excluded)")
    args = ap.parse_args()
    wl = bench.WORKLOADS[args.workload]
    w, h, c = wl["w"], wl["h"], wl["chans"]
    M = 85 if c == 3 else 63
    o = Oracle()
    f128 = advance_tables()
    paths = np.zeros(5, np.int64)
    lit_wf = lit_lds = 0
    crc_byte_wf = crc_byte_lds = crc_nib_lds = 0
    crc_split_wf = {2: 0, 4: 0}
    words_total = steps_total = 0
    mixed_event_words = mixed_words = 0
    for i in range(args.images):
        img = bench.workload_image(wl, "g1", i)
        data, row_bits, stored = o.encode(img, w, h, c, wl["flags"], want_rows=True)
        assert not stored
        stream = np.frombuffer(data + b"\0" * 8, dtype=np.uint8)
        _, _, hb = o.static_table(c)
        G = 8 * (41 + 2) + hb + np.concatenate([[0], np.cumsum(row_bits.astype(np.int64))])   # row start bits in the file
        for y in np.linspace(1, h - 1, args.rows).astype(int):
            filt, px = model.filtered_pixels(img, y)
            steps = lane_records(px, M)
            assert tokens_from_records(filt, px, steps, M) == model.serial_tokens(filt, px, M), (i, y)
            d = ((img[y].astype(np.int16) - img[y - 1].astype(np.int16)) & 255).astype(np.uint8).reshape(-1)
            steps_total += len(steps)
            for s, recs in enumerate(steps):
                for hh in range(2):
                    lit8 = [(r[1] >> (8 * hh)) & 0xFF for r in recs]
                    ev8 = [(r[3] >> (8 * hh)) & 0xFF for r in recs]
                    if all(l == 0xFF and e == 0 for l, e in zip(lit8, ev8)):
                        paths[1] += 1
                        base = s * 512 * c + np.arange(32) * 16 * c + hh * 8 * c
                        for b in range(8 * c):
                            idx = d[np.minimum(base + b, d.size - 1)].astype(np.int64)
                            lit_wf += lds64_wavefronts(idx)
                            lit_lds += 1
                    elif all(l == 0 for l in lit8):
                        paths[2] += 1
                    elif sum(bin(l).count("1") for l in lit8) >= 16:
                        paths[3] += 1
                        for e in ev8:                    # words of a lane's half that hold an event pixel other than at byte 0
                            for j in range(2 * c):
                                k0, k3 = 4 * j // c, (4 * j + 3) // c
                                mixed_words += 1
                                mixed_event_words += bool(k3 != k0 and (e >> k3) & 1)
                    else:
                        paths[4] += 1
            # scanline CRC: the row's code words (first / last masked to the row's bits), lane j % 32 folds word j
            g0, g1 = int(G[y]), int(G[y + 1])
            nw = (g1 + 31) // 32 - g0 // 32
            wv = np.frombuffer(stream[4 * (g0 // 32): 4 * (g0 // 32) + 4 * nw].tobytes(), "<u4").astype(np.uint64)
            wv[0] &= (0xFFFFFFFF << (g0 & 31)) & 0xFFFFFFFF
            if g1 & 31:
                wv[-1] &= (1 << (g1 & 31)) - 1
            words_total += nw
            cx = np.zeros(32, np.uint64)
            for j0 in range(0, nw, 32):
                v = wv[j0:j0 + 32]
                n = v.size
                reg = cx[:n]
                for k in range(4):
                    b = ((reg >> np.uint64(8 * k)) & np.uint64(0xFF)).astype(np.int64)
                    crc_byte_wf += lds32_wavefronts(256 * k + b)
                    for r in crc_split_wf:
                        crc_split_wf[r] += split_wavefronts(b, r)
                    crc_byte_lds += 1
                crc_nib_lds += 8                          # 16 entries in 16 distinct banks: one wavefront each
                nxt = v.copy()
                for k in range(4):
                    nxt ^= f128[k][((reg >> np.uint64(8 * k)) & np.uint64(0xFF)).astype(np.int64)].astype(np.uint64)
                cx[:n] = nxt
    halves = paths[1:].sum()
    print(f"workload {wl['name']}: {args.images} images x {args.rows} scanlines, {steps_total} warp steps, {halves} halves")
    for p, name in ((1, "all literal"), (2, "no literal"), (3, "mixed"), (4, "sparse")):
        print(f"  path ({p}) {name:12s} {paths[p]:8d} halves  {paths[p] / halves:6.2%}")
    print(f"  mixed halves: {mixed_event_words / max(mixed_words, 1):.2%} of (lane, word) pairs split by an event inside the word")
    print(f"  output words per warp step: {words_total / steps_total:.1f} ({words_total / steps_total / 32:.2f} per lane)")
    print(f"  path (1) literal LDS.64: {lit_wf / lit_lds:.2f} wavefronts per load (2 = conflict free)")
    print(f"  CRC byte tables: {crc_byte_wf / crc_byte_lds:.2f} wavefronts per LDS, {crc_byte_wf / steps_total:.1f} per warp step;"
          f" nibble tables: 1.00 per LDS, {crc_nib_lds / steps_total:.1f} per warp step")
    for r, wf in crc_split_wf.items():
        print(f"  CRC byte tables in {r} bank-disjoint copies (lane group g reads copy g): {wf / crc_byte_lds:.2f} wavefronts per LDS")


if __name__ == "__main__":
    main()
